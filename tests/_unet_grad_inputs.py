"""Cases and inputs of the UNet gradient golden vectors (tests/golden/make_unet_grad_golden.py): gradients of loss = sum(G * eps),
eps = denoise_fn(x, noise_level), with respect to x, the noise level and every parameter, for a fixed seeded upstream gradient G.  Inputs
come from seeded CPU generators, so the fixture only holds the reference's results.  Shared by the generator,
tests/test_oracle_unet_grad.py and tests/test_gpu_unet_grad.py.

Weights come from torch.manual_seed(SEED) in the reference's construction order (orthogonal, train-phase init)."""
import torch

from _lowres_inputs import TINY4
from _sizes_inputs import SR16_64, TINY

SEED = 11
UNCOND = dict(TINY, in_channel=3)

# name -> (unet, image_size, conditional, batch, height, width)
CASES = {
    "tiny_32x32": (TINY, 32, True, 2, 32, 32),              # attention on the 16x16 level: 256 tokens
    "tiny_32x64": (TINY, 32, True, 2, 32, 64),              # 16x32: 512 tokens (the training plan's unfused attention)
    "tiny4_b3": (TINY4, 16, True, 3, 16, 16),               # lowest level 4x4: the batch is padded to 8 images
    "uncond_32x32": (UNCOND, 32, False, 2, 32, 32),         # unconditional: x is x_t alone (3 channels)
}
# a train-mode (Dropout) forward of TINY with the reference's own masks: (case, p, torch seed that drives nn.Dropout)
DROPOUT_CASE = ("tiny_32x32", 0.2, 777)
# checked on the GPU against the oracle only (no reference fixture): the 16->64 config at 64x64, batch 2
GPU_ONLY = {"sr16_64_64x64": (SR16_64, 64, True, 2, 64, 64)}
ALL = dict(CASES, **GPU_ONLY)


def inputs(name):
    """x [B,in_channel,H,W], noise level [B,1] and the upstream gradient G [B,3,H,W] of a case."""
    unet, _, _, b, h, w = ALL[name]
    gen = torch.Generator().manual_seed(2000 + sorted(ALL).index(name))
    x = torch.randn(b, unet["in_channel"], h, w, generator=gen)
    nl = torch.tensor([[0.7], [0.05], [0.4]])[:b]
    g = torch.randn(b, unet["out_channel"], h, w, generator=gen)
    return x, nl, g


def signature(t):
    """norm, sum and 16 strided samples of a gradient (the fixture never stores a whole parameter gradient)."""
    f = t.detach().flatten()
    stride = max(1, f.numel() // 16)
    return {"norm": f.norm().item(), "sum": f.double().sum().item(), "samples": f[::stride][:16].clone(), "numel": f.numel()}

"""Cases and inputs of the training golden vectors at image sizes other than a net's image_size (tests/golden/make_train_sizes_golden.py),
drawn from seeded CPU generators so that the fixture only holds the reference's results.  Shared by the generator,
tests/test_oracle_train_sizes.py and tests/test_gpu_train_sizes.py.

Every case trains a net built for `image_size` (which places the attention layers) on (height, width) images, with the draws of p_losses
injected: gamma from np.random.RandomState(NP_SEED) through oracle.draw_gamma (the reference's own two numpy draws), noise from
`batch`.  Weights come from torch.manual_seed(SEED) in the reference's construction order (orthogonal, train-phase init)."""
import torch

from _sizes_inputs import SR16_64, TINY

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}      # = tests/_train_util.SCHED
SEED = 5
NP_SEED = 7
FULL = SR16_64           # sr_sr3_16_128.json's UNet; at image_size 128 its attention sits on the 16x16 level

# name -> (unet, image_size, batch, height, width)
CASES = {
    "tiny_32x64": (TINY, 32, 2, 32, 64),                  # attention level 16x32: 512 tokens
    "tiny_64x32": (TINY, 32, 2, 64, 32),
    "tiny_64x64": (TINY, 32, 2, 64, 64),                  # 32x32: 1024 tokens
    "sr16_64_128x128": (SR16_64, 64, 2, 128, 128),        # 32x32 attention (1024 tokens); lowest level 8x8 instead of 4x4
    "full_128x256": (FULL, 128, 2, 128, 256),             # 16x32 attention (512 tokens), 8x16 in the middle block
}
# a training-mode (Dropout) step of TINY at a non-square size with the reference's own masks
DROPOUT_CASE = ("tiny_32x64", 0.2, 4242)                   # (case, p, torch seed that drives nn.Dropout)


def batch(B, H, W, seed):
    gen = torch.Generator().manual_seed(seed)
    hr = torch.rand(B, 3, H, W, generator=gen) * 2 - 1
    sr = torch.rand(B, 3, H, W, generator=gen) * 2 - 1
    noise = torch.randn(B, 3, H, W, generator=gen)
    return hr, sr, noise


def case_batch(name):
    _, _, b, h, w = CASES[name]
    return batch(b, h, w, 1000 + sorted(CASES).index(name))


def signature(t):
    """norm, sum and 16 strided samples of a gradient (the fixture never stores a whole tensor)."""
    f = t.detach().flatten()
    stride = max(1, f.numel() // 16)
    return {"norm": f.norm().item(), "sum": f.double().sum().item(), "samples": f[::stride][:16].clone(), "numel": f.numel()}

"""Cases and inputs of the golden vectors for images of another size than the net's image_size (tests/golden/make_sizes_golden.py), drawn
from seeded CPU generators so that the fixture only has to hold the reference's outputs.  Shared by the generator,
tests/test_oracle_sizes.py and tests/test_gpu_sizes.py.

Every case runs a net built for `image_size` (which places the attention layers) on `(height, width)` images.  Outputs are compared on
fixed crops (`crop`) to keep the fixture small (about 200 KB); per-layer outputs ("taps") are kept for image 0 over a crop of the layer's own grid."""
import torch

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
SCHED10 = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
T_EVAL = (1999, 1000, 1)

# image_size 32, two levels, attention at the construction-time 16x16 level: at 32x64 / 64x32 it attends over 512 tokens, at 64x64 over 1024
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)
# the 16->64 config: lowest level 4x4 at 64x64, 8x8 at 128x128 (its attention level then holds 32x32 = 1024 tokens)
SR16_64 = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
# sr_sr3_16_128 (config/sr_sr3_16_128.json): the same UNet options at image_size 128; at 128x256 its attention level is 16x32 = 512 tokens
FULL = SR16_64


def _c(r0, r1, c0, c1):
    return (slice(r0, r1), slice(c0, c1))


ALL = (slice(None), slice(None))
# name -> (unet, image_size, seed, batch, height, width, eps crop (rows, cols), taps {layer: (rows, cols) crop of that layer's grid})
CASES = {
    # 32x64 -> 16x32 (attention, 512 tokens); downs.3 / mid.0 carry attention
    "tiny_32x64": (TINY, 32, 0, 2, 32, 64, _c(8, 24, 24, 40), {"downs.3": _c(4, 8, 8, 12), "mid.0": _c(8, 12, 20, 24), "ups.4": _c(8, 12, 40, 44)}),
    "tiny_64x32": (TINY, 32, 0, 2, 64, 32, _c(24, 40, 8, 24), {"downs.3": _c(8, 12, 4, 8), "mid.0": _c(20, 24, 8, 12), "ups.4": _c(40, 44, 8, 12)}),
    # 64x64 -> 32x32 (attention, 1024 tokens)
    "tiny_64x64": (TINY, 32, 0, 2, 64, 64, _c(24, 40, 24, 40), {"downs.3": _c(8, 12, 8, 12), "mid.0": _c(20, 24, 16, 20),
                                                                 "ups.4": _c(40, 44, 16, 20)}),
    # 128 -> 64 -> 32 (attention, 1024 tokens) -> 16 -> 8 (lowest)
    "sr16_64_128x128": (SR16_64, 64, 0, 2, 128, 128, _c(56, 72, 56, 72),
                        {"downs.8": _c(8, 10, 8, 12), "mid.0": _c(2, 4, 2, 4), "ups.7": _c(12, 14, 8, 10), "ups.18": _c(56, 60, 56, 64)}),
    # 128x256 -> 64x128 -> 32x64 -> 16x32 (attention, 512 tokens) -> 8x16 (mid.0 attention, 128 tokens)
    "full_128x256": (FULL, 128, 0, 2, 128, 256, _c(56, 72, 120, 136),
                     {"downs.11": _c(4, 6, 8, 10), "mid.0": _c(2, 4, 6, 8), "ups.5": _c(8, 10, 16, 18), "ups.18": _c(56, 60, 120, 128)}),
}
LOOP_CASE = "full_128x256"          # p_mean_variance at T_EVAL and a 10-step loop with injected noise


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def inputs(name):
    """x [B,6,H,W] and noise levels of the forward with taps; cond / x_t of the eps and p_mean_variance evaluations at T_EVAL."""
    _, _, _, b, h, w, _, _ = CASES[name]
    g = _gen(500 + sorted(CASES).index(name))
    x = torch.randn(b, 6, h, w, generator=g)
    cond = torch.rand(b, 3, h, w, generator=g) * 2 - 1
    x_t = torch.randn(b, 3, h, w, generator=g)
    nl = torch.tensor([[0.7], [0.05]])[:b]
    return {"x": x, "noise_level": nl, "cond": cond, "x_t": x_t}


def loop_inputs():
    """x_T and noises[i] (used at step i) of the 10-step loop of LOOP_CASE."""
    _, _, _, b, h, w, _, _ = CASES[LOOP_CASE]
    g = _gen(4322)
    return {"x_T": torch.randn(b, 3, h, w, generator=g), "noises": torch.randn(10, b, 3, h, w, generator=g)}


def tap_crop(name, layer, t):
    """Image 0 of a layer output [B,C,h,w] over the case's crop of that layer."""
    rows, cols = CASES[name][7][layer]
    return t[:1, :, rows, cols]


def eps_crop(name, t):
    rows, cols = CASES[name][6]
    return t[:, :, rows, cols]

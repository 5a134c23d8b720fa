"""Inputs of the 4x4-level golden vectors (tests/golden/make_lowres_golden.py), drawn from seeded CPU generators so that the fixture only
has to hold the reference's outputs.  Shared by the generator, tests/test_oracle_lowres.py and tests/test_gpu_lowres.py."""
import torch

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
SCHED10 = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
# 16 -> 8 -> 4 (middle block with attention at 4x4); 32 -> 16 -> 8 -> 4 unconditional; the 16->64 config (64 -> ... -> 4)
TINY4 = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 2], attn_res=[], res_blocks=1, dropout=0.0)
UNCOND32 = dict(in_channel=3, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8], attn_res=[], res_blocks=1, dropout=0.0)
SR16_64 = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
# per-layer outputs kept in the fixture: the layers at and next to the 4x4 level, image 0
TAPS = ("downs.4", "downs.5", "mid.0", "mid.1", "ups.0", "ups.1")
CROP = (slice(None), slice(None), slice(24, 40), slice(24, 40))      # 16x16 centre of a 64x64 output
T_EVAL = (1999, 1000, 1)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def tiny4():
    g = _gen(100)
    x = torch.randn(3, 6, 16, 16, generator=g)
    cond = torch.rand(3, 3, 16, 16, generator=g) * 2 - 1
    x_t = torch.randn(3, 3, 16, 16, generator=g)
    return {"x": x, "noise_level": torch.tensor([[0.7], [0.05], [0.4]]), "cond": cond, "x_t": x_t}


def tiny4_diffusion():
    g = _gen(4321)
    x_T = torch.randn(3, 3, 16, 16, generator=g)
    noises = torch.randn(10, 3, 3, 16, 16, generator=g)        # noises[i] is used at step i
    hr = torch.rand(3, 3, 16, 16, generator=g) * 2 - 1
    noise = torch.randn(3, 3, 16, 16, generator=g)
    return {"x_T": x_T, "noises": noises, "hr": hr, "noise": noise, "np_seed": 7}


def uncond32():
    return {"x_t": torch.randn(2, 3, 32, 32, generator=_gen(102))}


def sr16_64():
    g = _gen(103)
    cond = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    return {"cond": cond, "x_t": torch.randn(2, 3, 64, 64, generator=g)}

"""Windowed sampling without a GPU: the window grid and blend weights (the host arithmetic `_native.window_grid` / `window_weights` shares
with the native side) and the CPU oracle's merged step (oracle/windowed_oracle.py)."""
import itertools

import pytest
import torch

from oracle import sr3_oracle as orc
from oracle import windowed_oracle as worc
from sr3_b200 import _native

LENGTHS = (64, 65, 96, 127, 128, 129, 160, 200, 255, 256, 312, 720, 1280)


def cases():
    for side in (64, 128):
        for overlap in (0, 1, 32, side - 1):
            for L in LENGTHS:
                if L >= side:
                    yield L, side, overlap


@pytest.mark.parametrize("L,side,overlap", list(cases()))
def test_window_grid_and_weights(L, side, overlap):
    o = _native.window_grid(L, side, overlap)
    assert o == worc.window_grid(L, side, overlap)
    assert o[0] == 0 and o[-1] == L - side and o == sorted(set(o))
    assert (len(o) == 1) == (L == side)
    for a, b in zip(o, o[1:]):
        assert a + side - b >= overlap, (a, b)
    w = _native.window_weights(len(o), side, overlap)
    assert w.dtype == torch.float32 and torch.equal(w, worc.window_weights(len(o), side, overlap))
    assert (w > 0).all() and (w <= 1).all()
    total, cover = torch.zeros(L), torch.zeros(L)
    for k, a in enumerate(o):
        total[a:a + side] += w[k]
        cover[a:a + side] += 1
    assert (total > 0).all() and (cover >= 1).all()
    assert torch.equal(w[0][:1], torch.ones(1)) and torch.equal(w[-1][-1:], torch.ones(1))      # no ramp towards the canvas border
    for k, a in enumerate(o):                      # where one window covers, its weight is 1
        alone = cover[a:a + side] == 1
        assert torch.equal(w[k][alone], torch.ones(int(alone.sum())))


def test_grid_refuses_small_canvas_and_bad_overlap():
    with pytest.raises(ValueError, match="smaller than the window"):
        _native.window_grid(100, 128, 32)
    for ov in (-1, 128, 200):
        with pytest.raises(ValueError, match="overlap"):
            _native.window_grid(256, 128, ov)


TINY = orc.UNetConfig(6, 3, 64, 32, (1, 2), (16,), 1, 0.0, 32)
SCHED4 = {"schedule": "linear", "n_timestep": 4, "linear_start": 1e-4, "linear_end": 2e-2}


def test_one_window_is_the_plain_loop_exactly():
    sd = orc.init_state_dict(TINY, 0)
    sch = orc.make_schedule(SCHED4)
    g = torch.Generator().manual_seed(1)
    cond, x_T = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1, torch.randn(2, 3, 32, 32, generator=g)
    noises = torch.randn(4, 2, 3, 32, 32, generator=g)
    with torch.no_grad():
        plain = orc.p_sample_loop(sd, TINY, sch, cond, x_T, noises, True, continous=True)
        win = worc.p_sample_loop_windowed(sd, TINY, sch, cond, x_T, noises, True, (32, 32), (8, 8), continous=True)
    assert plain.shape == win.shape and torch.equal(plain, win)


@pytest.mark.parametrize("H,W,overlap", [(32, 48, (8, 16)), (40, 32, (3, 0)), (50, 70, (8, 8))])
def test_blend_is_an_affine_average(H, W, overlap):
    """A 'UNet' whose posterior mean is a function of the pixel's canvas position alone: every window reports the same value for a canvas
    pixel, and the blend returns it."""
    f = (torch.arange(H, dtype=torch.float32)[:, None] * 0.37 - torch.arange(W, dtype=torch.float32)[None, :] * 0.11).sin()
    sch = orc.make_schedule(SCHED4)
    oy, ox = worc.window_grid(H, 32, overlap[0]), worc.window_grid(W, 32, overlap[1])
    origins = list(itertools.product(oy, ox)) * 2

    def mean_fn(x, c, t):
        assert x.shape[0] == len(origins)
        return torch.stack([f[y0:y0 + 32, x0:x0 + 32].expand(3, 32, 32) for y0, x0 in origins])

    x_t = torch.zeros(2, 3, H, W)
    out = worc.windowed_step(mean_fn, sch, x_t, None, 0, None, (32, 32), overlap)
    assert (out - f.expand(2, 3, H, W)).abs().max() < 1e-6
    noise = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(2))
    out2 = worc.windowed_step(mean_fn, sch, x_t, None, 2, noise, (32, 32), overlap)
    sigma = (0.5 * sch.buffers["posterior_log_variance_clipped"][2]).exp()
    assert (out2 - (f.expand(2, 3, H, W) + sigma * noise)).abs().max() < 1e-6

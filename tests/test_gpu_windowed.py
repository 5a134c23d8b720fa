"""Windowed sampling on the device (GaussianDiffusion.super_resolution_windowed, sr3_windowed_*): canvases of any size denoised by
overlapping windows whose posterior means are merged inside every reverse step (DESIGN.md 3.9).

What is pinned: one window is the plain sampler bit for bit; one merged step equals its definition evaluated by the test from the device's
own window means and the documented Philox stream at canvas pixel indices; ten steps agree with the CPU oracle (oracle/windowed_oracle.py);
the result does not depend on how many windows run per engine pass, on repetition or on batching; there is no seam; bad arguments are
refused on the host before anything is allocated; sharding by image does not change the images."""
import numpy as np
import pytest
import torch

import _philox
import _sizes_inputs as si
from oracle import sr3_oracle as orc
from oracle import windowed_oracle as worc

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
TINY_CFG = orc.UNetConfig(6, 3, 64, 32, (1, 2), (16,), 1, 0.0, 32)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def build(monkeypatch, unet, image_size, seed=0, sched=si.SCHED10, precision="bf16"):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet, precision=precision),
                     "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}
    torch.manual_seed(seed)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


def draws(B, H, W, seed, T=None):
    g = torch.Generator().manual_seed(seed)
    cond, x_T = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.randn(B, 3, H, W, generator=g)
    noises = None if T is None else torch.randn(T, B, 3, H, W, generator=g)
    return cond.cuda(), x_T.cuda(), None if noises is None else noises.cuda()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("config", ["tiny_32x64", "full_128"])
def test_one_window_is_the_plain_sampler_bit_for_bit(monkeypatch, config, precision):
    unet, image_size, (H, W) = (si.TINY, 32, (32, 64)) if config == "tiny_32x64" else (si.FULL, 128, (128, 128))
    net = build(monkeypatch, unet, image_size, precision=precision)
    cond, x_T, noises = draws(2, H, W, 3, T=10)
    for kw in ({"seed": 7}, {"seed": 7, "continous": True}, {"noises": noises, "continous": True}, {"seed": 2 ** 40 + 5, "first_index": 3}):
        plain = net.super_resolution(cond, x_T=x_T, **kw)
        win = net.super_resolution_windowed(cond, window=(H, W), x_T=x_T, **kw)
        assert plain.shape == win.shape and torch.isfinite(win).all()
        assert torch.equal(win, plain), kw


def device_window_means(sampler, cond, x_t, t):
    """The device's own p_mean_variance means of every window of the canvas, run in the passes the sampler runs (the engine's batch, the
    last pass padded with its last window)."""
    oy, ox, _, _ = sampler.grid()
    eng = sampler.engine
    wh, ww = eng.height, eng.width
    crops = [(slice(b, b + 1), slice(None), slice(y0, y0 + wh), slice(x0, x0 + ww)) for b in range(x_t.shape[0]) for y0 in oy for x0 in ox]
    means = []
    for first in range(0, len(crops), eng.batch):
        idx = [min(first + s, len(crops) - 1) for s in range(eng.batch)]
        m, _ = eng.p_mean_variance(torch.cat([x_t[crops[i]] for i in idx]), t, True, torch.cat([cond[crops[i]] for i in idx]))
        means += list(m[: min(eng.batch, len(crops) - first)])
    return means, crops


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,H,W,overlap", [("tiny", 96, 160, (16, 16)), ("tiny", 70, 99, (5, 0)), ("full", 200, 312, None)])
def test_one_merged_step_is_its_definition(monkeypatch, config, H, W, overlap):
    unet, image_size, window = (si.TINY, 32, (64, 64)) if config == "tiny" else (si.FULL, 128, (128, 128))
    net = build(monkeypatch, unet, image_size, sched=si.SCHED)
    B, seed, first = 2, 2 ** 35 + 11, 2 ** 32 - 1
    cond, x_t, _ = draws(B, H, W, 5)
    sampler = net._windowed_sampler(B, H, W, window, overlap)
    oy, ox, wy, wx = sampler.grid()
    ov = sampler.overlap
    from sr3_b200 import _native
    assert oy == _native.window_grid(H, window[0], ov[0]) and ox == _native.window_grid(W, window[1], ov[1])
    assert torch.equal(wy, _native.window_weights(len(oy), window[0], ov[0])) and torch.equal(wx, _native.window_weights(len(ox), window[1], ov[1]))
    for t in (1500, 1, 0):
        means, crops = device_window_means(sampler, cond, x_t, t)
        num, den = torch.zeros_like(x_t), torch.zeros(B, 1, H, W, device="cuda")
        n = 0
        for b in range(B):                                         # ascending window index, separately rounded fp32 products and sums
            for iy in range(len(oy)):
                for ix in range(len(ox)):
                    w = (wy[iy][:, None] * wx[ix][None, :]).cuda()
                    c = crops[n]
                    num[c] = num[c] + w * means[n]
                    den[c] = den[c] + w
                    n += 1
        assert (den > 0).all()
        mean = (num / den).double().cpu()
        sampler.begin(cond, x_t, seed, first)
        sampler.steps(t, 1)
        got = sampler.read_state().double().cpu()
        if t == 0:
            assert (got - mean).abs().max() <= 1e-6 * mean.abs().max(), t
            continue
        sigma = float(np.exp(0.5 * float(net.posterior_log_variance_clipped[t].double())))
        z = torch.from_numpy(_philox.sampling_noise(seed, [first + b for b in range(B)], t, H, W))
        bound = 1e-6 * (mean.abs() + sigma * z.abs()) + 1e-9
        assert ((got - (mean + sigma * z)).abs() <= bound).all(), t
        # a counter word off by one misses by orders of magnitude
        zb = torch.from_numpy(_philox.sampling_noise(seed, [first + b for b in range(B)], t, H, W,
                                                     words=lambda c0, c1, c2, c3, k0, k1: ((c0 + np.uint64(1)) & np.uint64(0xFFFFFFFF), c1, c2, c3, k0, k1)))
        assert ((got - (mean + sigma * zb)).abs() / bound).median() > 1e3, t


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision,tol", [("bf16", 1e-2), ("fp32", 1e-3)])
def test_ten_steps_match_the_cpu_oracle(monkeypatch, precision, tol):
    net = build(monkeypatch, si.TINY, 32, precision=precision)
    H, W, window, overlap = 40, 72, (32, 32), (8, 8)
    cond, x_T, noises = draws(1, H, W, 9, T=10)
    got = net.super_resolution_windowed(cond, window=window, overlap=overlap, continous=True, x_T=x_T, noises=noises).cpu()
    sd = {k[len("denoise_fn."):]: v.detach().cpu() for k, v in net.state_dict().items() if k.startswith("denoise_fn.")}
    with torch.no_grad():
        ref = worc.p_sample_loop_windowed(sd, TINY_CFG, orc.make_schedule(si.SCHED10), cond.cpu(), x_T.cpu(), noises.cpu(), True, window, overlap,
                                          continous=True)
    assert got.shape == ref.shape == (11, 3, H, W)
    assert torch.equal(got[:1], cond.cpu())
    assert rel(got[5:6], ref[5:6]) < tol and rel(got[-1:], ref[-1:]) < tol, (rel(got[5:6], ref[5:6]), rel(got[-1:], ref[-1:]))


# (B, H, W) with window 32x32 and overlap 8: 1, 3, 6 and 7 windows
COUNTS = {1: (1, 32, 32), 3: (1, 32, 80), 6: (2, 80, 32), 7: (1, 32, 160)}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("count", sorted(COUNTS))
def test_result_does_not_depend_on_windows_per_pass(monkeypatch, count):
    net = build(monkeypatch, si.TINY, 32)
    B, H, W = COUNTS[count]
    cond, x_T, _ = draws(B, H, W, 20 + count)
    outs = {}
    for bw in (1, 2, 4, 2):
        monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (bw,))
        sampler = net._windowed_sampler(B, H, W, (32, 32), 8)
        oy, ox, _, _ = sampler.grid()
        assert B * len(oy) * len(ox) == count and sampler.engine.batch == bw
        out = net.super_resolution_windowed(cond, window=(32, 32), overlap=8, continous=True, x_T=x_T, seed=13).cpu()
        assert torch.isfinite(out).all()
        if bw in outs:
            assert torch.equal(out, outs[bw]), "repeat run"
        outs[bw] = out
    assert torch.equal(outs[1], outs[2]) and torch.equal(outs[1], outs[4])


def test_batched_images_equal_the_images_alone(monkeypatch):
    net = build(monkeypatch, si.TINY, 32)
    monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (2,))
    cond, x_T, _ = draws(2, 48, 80, 31)
    both = net.super_resolution_windowed(cond, window=(32, 32), continous=True, x_T=x_T, seed=17, first_index=4)[-2:].cpu()
    for b in range(2):
        alone = net.super_resolution_windowed(cond[b:b + 1], window=(32, 32), continous=True, x_T=x_T[b:b + 1], seed=17, first_index=4 + b)[-1:]
        assert torch.equal(alone.cpu(), both[b:b + 1]), b


def _hdiff(img, lo, hi):
    """Mean absolute horizontal difference over the column pairs (j, j + 1), j in [lo, hi), and over all the other pairs."""
    d = (img[..., 1:] - img[..., :-1]).abs().double()
    inside = torch.zeros(d.shape[-1], dtype=torch.bool)
    inside[lo:hi] = True
    return d[..., inside].mean().item(), d[..., ~inside].mean().item()


@pytest.mark.timeout(900)
def test_no_seam_across_the_overlap(monkeypatch):
    net = build(monkeypatch, si.TINY, 32)
    H, W, side, ov = 64, 96, 64, 32
    cond, x_T, _ = draws(1, H, W, 41)
    out = net.super_resolution_windowed(cond, window=(side, side), overlap=ov, continous=True, x_T=x_T, seed=23)[-1:].cpu()
    seam, rest = _hdiff(out, W - side - 1, side)
    # the contrast: each window sampled alone (its own noise in the overlap), pasted at the middle of the overlap
    parts = [net.super_resolution(cond[..., x0:x0 + side], continous=True, x_T=x_T[..., x0:x0 + side], seed=23)[-1:].cpu() for x0 in (0, W - side)]
    cut = W // 2
    pasted = torch.cat([parts[0][..., :cut], parts[1][..., cut - (W - side):]], dim=-1)
    p_seam, p_rest = _hdiff(pasted, cut - 1, cut)
    msg = "merged per step: overlap %.4f vs rest %.4f; sampled alone and pasted: cut %.4f vs rest %.4f" % (seam, rest, p_seam, p_rest)
    print(msg)
    assert seam <= 1.5 * rest and rest <= 1.5 * seam, msg


@pytest.mark.parametrize("kw,exc,msg", [
    ({"window": (96, 96)}, "UnsupportedSizeError", "powers of two"),
    ({"window": (64, 64), "overlap": 64}, "ValueError", "overlap"),
    ({"window": (64, 64), "overlap": (8, -1)}, "ValueError", "overlap"),
    ({"window": (256, 256)}, "ValueError", "smaller than the window"),
])
def test_bad_arguments_are_refused_before_allocating(monkeypatch, kw, exc, msg):
    from sr3_b200 import _native
    net = build(monkeypatch, si.SR16_64, 64)
    unet = net.denoise_fn
    cond = torch.zeros(1, 3, 200, 136).cuda()
    unet(torch.zeros(1, 6, 64, 64).cuda(), torch.full((1, 1), 0.5).cuda())
    keys = list(unet._engines)
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    with pytest.raises(getattr(_native, exc, ValueError) if exc != "ValueError" else ValueError, match=msg):
        net.super_resolution_windowed(cond, **kw)
    torch.cuda.synchronize()
    assert list(unet._engines) == keys and getattr(net, "_windowed", None) is None
    assert torch.cuda.mem_get_info()[0] >= free - (2 << 20)


@pytest.mark.timeout(900)
def test_sharded_windowed_super_resolution(monkeypatch):
    """On one rank the sharded call is the unsharded one bit for bit; the shards of a two-rank group (two images, then one) are the images
    the whole batch gives: the noise is keyed by the global sample index and the canvas pixel, and a window's mean does not depend on
    the windows that share its pass."""
    from sr3_b200 import parallel
    net = build(monkeypatch, si.TINY, 32)
    monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (2,))
    cond, x_T, _ = draws(3, 40, 72, 51)
    ref = net.super_resolution_windowed(cond, window=(32, 32), overlap=8, continous=True, x_T=x_T, seed=11)[-3:].cpu()
    whole = parallel.sharded_super_resolution(net, cond.cpu(), x_T=x_T.cpu(), seed=11, window=(32, 32), overlap=8).cpu()
    assert whole.shape == (3, 3, 40, 72) and torch.equal(whole, ref)
    parts = []
    for rank in (0, 1):
        monkeypatch.setattr(parallel.dist, "is_initialized", lambda: True)
        monkeypatch.setattr(parallel.dist, "get_world_size", lambda group=None: 2)
        monkeypatch.setattr(parallel.dist, "get_rank", lambda group=None, r=rank: r)
        monkeypatch.setattr(parallel, "gather_shards", lambda local, n, group=None: local)
        parts.append(parallel.sharded_super_resolution(net, cond.cpu(), x_T=x_T.cpu(), seed=11, window=(32, 32), overlap=8).cpu())
    assert [p.shape[0] for p in parts] == [2, 1]
    assert torch.equal(torch.cat(parts), whole)

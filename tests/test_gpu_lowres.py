"""UNets whose lowest level is 4x4: the tile kernel's padded 4x4 patch, 16-token attention, the 4x4 weight gradient and whole UNets.

A 4x4 image has 16 pixels, half a warp's 32 rows.  pick_image_box (engine.cu) gives it a 4 x 8 patch: rows 4..7 lie outside the image,
TMA loads them as zeros and the epilogue masks them, so every warp still holds one image (its FiLM bias, GroupNorm run and TMA boxes) and
a 128-row tile holds four images.  The weight-gradient kernel contracts a 4x4 image as one 8x8 patch whose other pixels are zero.

Kernel-level cases compare against fp64 on the same bf16 operands, with the bounds of test_gpu_tile_variants.py.  UNet-level cases compare
against the reference's outputs in tests/golden/sr3_lowres_golden.pt, and the gradients against the oracle's fp32 CPU autograd
(oracle/sr3_oracle.py, pinned to the same fixture by tests/test_oracle_lowres.py), at the project's bf16 and precise-mode tolerances.
"""
import math
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _lowres_inputs as li
import _train_util as tu
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

TALL_ENV = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_MAX_CTAS")
BF16_TOL, FP32_TOL, GRAD_TOL = 1e-2, 1e-3, 2e-2
SCHED, TINY4, UNCOND32, SR16_64 = li.SCHED, li.TINY4, li.UNCOND32, li.SR16_64


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def clear_knobs(monkeypatch):
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)


# ------------------------------------------------------------------------------------------------ kernel level
def nchw(t):
    return t.permute(0, 3, 1, 2)


def check_close(y, ref, what, rtol_l2=2e-5, elem=None):
    r = rel(y, ref)
    assert r < rtol_l2, f"{what}: relative L2 {r:.3e} >= {rtol_l2:.1e}"
    err = (y.double() - ref).abs()
    bound = elem if elem is not None else 1e-4 * (ref.abs() + ref.pow(2).mean().sqrt())
    bad = (err > bound).nonzero()
    if bad.numel():
        b, h, w, c = bad[0].tolist()
        pytest.fail(f"{what}: {bad.shape[0]} elements out of bound, first at (image {b}, row {h}, column {w}, channel {c}): "
                    f"got {y[b, h, w, c].item():.7g}, want {ref[b, h, w, c].item():.7g}")


def check_stats(stats, ref):
    st, refc = stats.cpu(), nchw(ref)
    assert torch.allclose(st[..., 0], refc.sum(dim=(2, 3)), rtol=1e-4, atol=1e-3), "GroupNorm sums"
    assert torch.allclose(st[..., 1], (refc ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=1e-3), "GroupNorm sums of squares"


def conv_ref(x, w, stride, bias=None, bias2=None, resid=None):
    k = w.shape[-1]
    y = F.conv2d(nchw(x.double()), w.bfloat16().double(), stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.double()
    if bias2 is not None:
        y = y + bias2.double()[:, None, None, :]
    if resid is not None:
        y = y + resid.double()
    return y


def check_geometry(geo, bn=None, split=None):
    assert geo["tall"] == 0 and geo["mh"] == 1 and geo["h_box"] == 8 and geo["b_box"] == 4, geo
    if bn is not None:
        assert geo["block_n"] == bn, geo
    if split is not None:
        assert geo["ksplit"] == split, geo


# (name, input side, Cin, k, stride): every output is 4x4
CONV_FORMS = [("3x3", 4, 128, 3, 1), ("1x1", 4, 768, 1, 1), ("stride2_from_8x8", 8, 128, 3, 2)]
CONV_CASES = [(f"{n}-bn{bn}-split{sp}-B{B}", H, Cin, k, s, bn, sp, B)
              for n, H, Cin, k, s in CONV_FORMS for bn in (32, 64, 128, 256) for sp in (1, 2) for B in (1, 3, 8, 9)]


@pytest.mark.parametrize("cid,H,Cin,k,s,bn,split,B", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_at_4x4(monkeypatch, cid, H, Cin, k, s, bn, split, B):
    """Per-image FiLM bias, residual, GroupNorm sums and the bf16 copy of a 4x4 conv, every forced BLOCK_N, unsplit and split-K, with
    batches that leave the last tile's image slots empty (1, 3, 9) or fill them (8)."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    monkeypatch.setenv("SR3_BLOCK_N", str(bn))
    monkeypatch.setenv("SR3_KSPLIT", str(split))
    g = torch.Generator().manual_seed(zlib.crc32(cid.encode()))
    Cout = 256
    x = torch.randn(B, H, H, Cin, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k)
    bias, bias2 = torch.randn(Cout, generator=g), torch.randn(B, Cout, generator=g)
    resid = split > 1 or bn < 256           # an unsplit 128 x 256 stage and the staged residual do not fit in shared memory together
    res = torch.randn(B, 4, 4, Cout, generator=g) if resid else None
    y, yb, stats, geo = _native.test_conv_ex(x.cuda(), w.cuda(), k, s, bias=bias.cuda(), bias2=bias2.cuda(),
                                             resid=res.cuda() if resid else None, want_bf16=True, want_stats=True)
    check_geometry(geo, bn, split)
    y = y.cpu()
    ref = conv_ref(x, w, s, bias, bias2, res)
    check_close(y, ref, cid)
    check_stats(stats, ref)
    assert torch.equal(yb.cpu(), y.bfloat16()), "bf16 copy differs from bf16(fp32 output)"


@pytest.mark.parametrize("B", [1, 3, 9])
def test_block2_with_shortcut_at_4x4(monkeypatch, B):
    """block2 of a 4x4 ResnetBlock whose channel count changes: the 1x1 res_conv over the block input as extra K columns of the same GEMM."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    cin, cout = 256, 128
    g = torch.Generator().manual_seed(B)
    a = torch.randn(B, 4, 4, cout, generator=g).bfloat16()
    raw = torch.randn(B, 4, 4, cin, generator=g).bfloat16()
    w = torch.randn(cout, cout, 3, 3, generator=g) / math.sqrt(cout * 9)
    wr = torch.randn(cout, cin, 1, 1, generator=g) / math.sqrt(cin)
    b2, br, bias2 = torch.randn(cout, generator=g), torch.randn(cout, generator=g), torch.randn(B, cout, generator=g)
    y, yb, stats, geo = _native.test_conv_ex(a.cuda(), w.cuda(), 3, 1, bias=(b2 + br).cuda(), bias2=bias2.cuda(), x2=raw.cuda(),
                                             w2=wr.cuda(), want_bf16=True, want_stats=True)
    check_geometry(geo)
    y = y.cpu()
    ref = conv_ref(a, w, 1, b2, bias2) + conv_ref(raw, wr, 1, br)
    check_close(y, ref, f"block2 + shortcut B={B}")
    check_stats(stats, ref)
    assert torch.equal(yb.cpu(), y.bfloat16())


@pytest.mark.parametrize("B", [1, 3, 9])
def test_folded_upsample_from_4x4(monkeypatch, B):
    """Upsample 4 -> 8 as the engine runs it: the four output phases of nearest-2x -> conv3x3 folded onto the 4x4 grid, one launch."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    C = 128
    g = torch.Generator().manual_seed(100 + B)
    x = torch.randn(B, 4, 4, C, generator=g).bfloat16()
    w = torch.randn(C, C, 3, 3, generator=g) / math.sqrt(C * 9)
    bias = torch.randn(C, generator=g)
    y, _, stats, geo = _native.test_conv_ex(x.cuda(), w.cuda(), 3, 1, bias=bias.cuda(), fold_up=True, want_stats=True)
    check_geometry(geo)
    assert geo["tiles"] % 4 == 0, geo
    y = y.cpu()
    # the fold sums aliased taps before the bf16 rounding: against the unfolded weights that is one extra rounding (2^-9 relative)
    up = F.interpolate(nchw(x.double()), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, w.bfloat16().double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    assert y.shape == (B, 8, 8, C)
    assert rel(y, ref) < 4e-3, rel(y, ref)
    check_stats(stats, y.double())


@pytest.mark.parametrize("B", [3, 9])
def test_precise_mode_at_4x4(monkeypatch, B):
    """Precise mode's three passes in the 4x4 form, on unrounded fp32 operands; bound derived in test_gpu_tile_variants.py."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    Cin = Cout = 128
    g = torch.Generator().manual_seed(200 + B)
    x = torch.randn(B, 4, 4, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (3.0 / math.sqrt(Cin * 9))
    bias, res = torch.randn(Cout, generator=g), torch.randn(B, 4, 4, Cout, generator=g)
    hi = x.bfloat16()
    xin = torch.cat([hi, (x - hi.float()).bfloat16()], dim=-1)
    y, yb, _, geo = _native.test_conv_ex(xin.cuda(), w.cuda(), 3, 1, bias=bias.cuda(), resid=res.cuda(), want_bf16=True, precise=True)
    check_geometry(geo)
    y = y.cpu()
    ref = F.conv2d(nchw(x.double()), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1) + res.double()
    absdot = F.conv2d(nchw(x.double().abs()), w.double().abs(), padding=1).permute(0, 2, 3, 1)
    check_close(y, ref, "precise mode 4x4", elem=2.0 ** -15 * absdot + 2.0 ** -22 * ref.abs())
    yb = yb.cpu()
    yh = y.bfloat16()
    assert torch.equal(yb[..., :Cout], yh) and torch.equal(yb[..., Cout:], (y - yh.float()).bfloat16())


@pytest.mark.parametrize("nz,C", [(1, 128), (2, 512)])
def test_attention_16_tokens_per_image(nz, C):
    """Eight 4x4 images (16 tokens each) share a 128-token attention batch under the block-diagonal mask (reference and bound:
    tests/_attention_ref.py)."""
    from _attention_ref import check_fused
    from sr3_b200 import _native
    Lt, HW = 128, 16
    g = torch.Generator().manual_seed(nz + C)
    q, k, v = (torch.randn(nz, Lt, C, generator=g) for _ in range(3))
    qk = torch.cat([2.0 * q, k], dim=2).bfloat16()
    vb = v.bfloat16()
    out = _native.test_attention(qk.reshape(nz * Lt, 2 * C).cuda(), vb.transpose(1, 2).contiguous().reshape(nz * C, Lt).cuda(),
                                 nz, Lt, HW, C).float().cpu().reshape(nz, Lt, C)
    check_fused(out, qk, vb, Lt, HW, C)


@pytest.mark.parametrize("B,k,stride", [(1, 3, 1), (3, 3, 1), (5, 1, 1), (3, 3, 2), (5, 3, 2)])
def test_wgrad_at_4x4(B, k, stride):
    """Weight gradient with a 4x4 output (stride 2: from an 8x8 input): one 8x8 patch per image, zero outside it."""
    from sr3_b200 import _native
    CY, Cin = 128, 128
    g = torch.Generator().manual_seed(300 + 10 * B + k + stride)
    dy = torch.randn(B, 4, 4, CY, generator=g).bfloat16()
    x = torch.randn(B, 4 * stride, 4 * stride, Cin, generator=g).bfloat16()
    got, used = _native.test_wgrad(dy.cuda(), x.cuda(), k, stride)
    assert 1 <= used <= B
    ref = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (CY, Cin, k, k), dy.double().permute(0, 3, 1, 2),
                                      stride=stride, padding=k // 2)
    got = got.cpu().double()
    assert rel(got, ref) < 2e-5, rel(got, ref)
    assert ((got - ref).abs() <= 1e-4 * (ref.abs() + ref.pow(2).mean().sqrt())).all()


# ------------------------------------------------------------------------------------------------ UNet level
def make_opt(unet, image_size, conditional=True, phase="val", sched=SCHED):
    return {"phase": phase, "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}


def build(unet, image_size, seed, conditional=True, sched=SCHED, precision="bf16"):
    import sr3_b200
    torch.manual_seed(seed)
    net = sr3_b200.define_G(make_opt(dict(unet, precision=precision), image_size, conditional, sched=sched)).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


def inputs(B, R, cin, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cin, R, R, generator=g), torch.rand(B, 1, generator=g) * 0.9 + 0.05


@pytest.fixture(scope="module")
def lowres():
    """Outputs of the unmodified reference for these nets (tests/golden/make_lowres_golden.py; weights from the same seeded init, inputs
    from tests/_lowres_inputs.py)."""
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sr3_lowres_golden.pt"), map_location="cpu",
                      weights_only=False)


@pytest.mark.parametrize("precision,B", [("bf16", 1), ("bf16", 3), ("bf16", 16), ("fp32", 1), ("fp32", 3), ("fp32", 16)])
def test_tiny_4x4_net_layers_and_eps(monkeypatch, lowres, precision, B):
    """Per-layer outputs around the 4x4 level and eps of the 16 -> 8 -> 4 net against the reference; batches beyond the golden's three
    repeat its images, and every copy of image 0 is checked layer by layer."""
    clear_knobs(monkeypatch)
    g, inp = lowres["tiny4"], li.tiny4()
    idx = [i % 3 for i in range(B)]
    net = build(TINY4, 16, g["seed"], precision=precision)
    eps = net.denoise_fn(inp["x"][idx].cuda(), inp["noise_level"][idx].cuda())
    tol = BF16_TOL if precision == "bf16" else FP32_TOL
    eng = net.denoise_fn.engine(B)
    first = [i for i in range(B) if idx[i] == 0]
    for name, ref in g["taps"].items():
        act = eng.read_activation(name).cpu()[first]
        e = rel(act, ref.expand_as(act))
        assert e < tol, (name, e)
    assert rel(eps, g["eps"][idx]) < tol, rel(eps, g["eps"][idx])


def test_tiny_4x4_eps_and_pmv_over_t(monkeypatch, lowres):
    clear_knobs(monkeypatch)
    g, inp = lowres["tiny4"], li.tiny4()
    net = build(TINY4, 16, g["seed"])
    sch = orc.make_schedule(SCHED)
    for t, ref in g["eps_t"].items():
        eps = net.denoise_fn(torch.cat([inp["cond"], inp["x_t"]], 1).cuda(), orc.noise_level_for_t(sch, t, 3).cuda())
        assert rel(eps, ref) < BF16_TOL, (t, rel(eps, ref))
        mean, lv = net.p_mean_variance(inp["x_t"].cuda(), t, True, condition_x=inp["cond"].cuda())
        assert rel(mean, g["pmv"][t][0]) < BF16_TOL and float(lv) == float(g["pmv"][t][1]), t


def test_tiny_4x4_loop_and_p_losses(monkeypatch, lowres):
    """The reference's 10-step loop with the same draws injected (super_resolution, continous=True), and p_losses."""
    clear_knobs(monkeypatch)
    g, inp, d = lowres["tiny4_diffusion"], li.tiny4(), li.tiny4_diffusion()
    net = build(TINY4, 16, 0, sched=li.SCHED10)
    out = net.super_resolution(inp["cond"].cuda(), continous=True, x_T=d["x_T"].cuda(), noises=d["noises"].cuda())
    assert out.shape == (3 * 11, 3, 16, 16)
    assert torch.equal(out[:3].cpu(), inp["cond"])
    assert rel(out[15:18], g["loop_mid"]) < BF16_TOL, rel(out[15:18], g["loop_mid"])
    assert rel(out[-3:], g["loop_last"]) < BF16_TOL, rel(out[-3:], g["loop_last"])
    np.random.seed(d["np_seed"])
    net.set_loss("cuda")
    with torch.no_grad():
        loss = net.p_losses({"HR": d["hr"].cuda(), "SR": inp["cond"].cuda()}, noise=d["noise"].cuda())
    assert abs(loss.item() - g["loss"].item()) / g["loss"].item() < BF16_TOL


def test_unconditional_32_net_eps(monkeypatch, lowres):
    clear_knobs(monkeypatch)
    g, x_t = lowres["uncond32"], li.uncond32()["x_t"]
    net = build(UNCOND32, 32, g["seed"], conditional=False)
    sch = orc.make_schedule(SCHED)
    for t, ref in g["eps"].items():
        eps = net.denoise_fn(x_t.cuda(), orc.noise_level_for_t(sch, t, x_t.shape[0]).cuda())
        assert rel(eps, ref) < BF16_TOL, rel(eps, ref)


@pytest.mark.timeout(900)
def test_16_64_config_eps_and_pmv(monkeypatch, lowres):
    """eps and p_mean_variance of the 16->64 config at batch 2 against the reference's 16x16 centre crop."""
    clear_knobs(monkeypatch)
    g, s = lowres["sr16_64"], li.sr16_64()
    net = build(SR16_64, 64, g["seed"])
    sch = orc.make_schedule(SCHED)
    for t, ref in g["eps"].items():
        eps = net.denoise_fn(torch.cat([s["cond"], s["x_t"]], 1).cuda(), orc.noise_level_for_t(sch, t, 2).cuda())
        assert torch.isfinite(eps).all()
        assert rel(eps[li.CROP], ref) < BF16_TOL, (t, rel(eps[li.CROP], ref))
        mean, lv = net.p_mean_variance(s["x_t"].cuda(), t, True, condition_x=s["cond"].cuda())
        assert rel(mean[li.CROP], g["pmv"][t][0]) < BF16_TOL and float(lv) == float(g["pmv"][t][1]), t


@pytest.mark.parametrize("B", [3, 16])
def test_4x4_net_is_bit_reproducible(monkeypatch, B):
    """Repeat runs give the same bits (exact GroupNorm sums, fixed-order split-K)."""
    sched = {"schedule": "linear", "n_timestep": 6, "linear_start": 1e-4, "linear_end": 2e-2}
    g = torch.Generator().manual_seed(B)
    cond, x_T = torch.rand(B, 3, 16, 16, generator=g) * 2 - 1, torch.randn(B, 3, 16, 16, generator=g)
    clear_knobs(monkeypatch)
    net = build(TINY4, 16, 0, sched=sched)
    a = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=5).cpu()
    b = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=5).cpu()
    assert torch.equal(a, b) and torch.isfinite(a).all()


def test_sharded_super_resolution_single_rank_4x4(monkeypatch):
    from sr3_b200 import parallel
    clear_knobs(monkeypatch)
    sched = {"schedule": "linear", "n_timestep": 6, "linear_start": 1e-4, "linear_end": 2e-2}
    net = build(TINY4, 16, 0, sched=sched)
    g = torch.Generator().manual_seed(8)
    cond, x_T = torch.rand(3, 3, 16, 16, generator=g) * 2 - 1, torch.randn(3, 3, 16, 16, generator=g)
    a = parallel.sharded_super_resolution(net, cond, x_T=x_T, seed=11)
    b = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=11, first_index=0)[-3:]
    assert a.shape == (3, 3, 16, 16) and torch.equal(a.cpu(), b.cpu())


def test_gradients_of_4x4_net_match_oracle(monkeypatch):
    """Every parameter gradient of the tiny 4x4 net at an odd batch (forward, data gradients in the 4x4 form, 4x4 weight gradients, the
    16-token attention backward) against the oracle's fp32 autograd."""
    clear_knobs(monkeypatch)
    unet = dict(TINY4)
    net = tu.build_train_net(unet, 16, 5, "l2")
    hr, sr, noise = tu.batch(3, 16, 1000)
    gamma = tu.draw_gamma(3, 7)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    lr_, gr = tu.oracle_loss_and_grads(net, unet, 16, hr, sr, gamma, noise, "l2")
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    assert set(go) == set(gr)
    for n, e, c, _ in tu.compare(go, gr):
        assert e < GRAD_TOL, (n, e, c)


def test_batch_of_one_does_not_compute_the_padded_images(monkeypatch):
    """A net with a 4x4 level allocates 8 image slots at batch 1, but a layer whose tiles hold one image launches tiles for the real image
    only.  Had the padded slots been computed, the 64x64 launches at batch 1 would be the same launches as at batch 8 (same tiles, same
    time); they take clearly less."""
    clear_knobs(monkeypatch)
    net = build(SR16_64, 64, 0)
    times = {}
    for B in (1, 8):
        x, nl = inputs(B, 64, 6, seed=B)
        net.denoise_fn(x.cuda(), nl.cuda())
        times[B] = [ms for k, ms, _, _ in net.denoise_fn.engine(B).profile_step(500, reps=20) if k == 0]
    assert len(times[1]) == len(times[8])
    # plan order: the first conv and the two ResnetBlocks of the 64x64 level are the first five tile-kernel launches
    t1, t8 = sum(times[1][:5]), sum(times[8][:5])
    print(f"64x64 tile-kernel launches: B=1 {t1:.4f} ms, B=8 {t8:.4f} ms")
    assert t1 < 0.8 * t8, (t1, t8)


def test_levels_below_4x4_are_refused(monkeypatch):
    clear_knobs(monkeypatch)
    net = build(dict(TINY4, channel_multiplier=[1, 2, 2, 2]), 16, 0)           # 16 -> 8 -> 4 -> 2
    with pytest.raises(RuntimeError, match="< 4"):
        net.denoise_fn(torch.zeros(1, 6, 16, 16).cuda(), torch.full((1, 1), 0.5).cuda())

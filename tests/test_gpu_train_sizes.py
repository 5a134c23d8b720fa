"""Training at image sizes other than a net's image_size (non-square included) on the GPU: sr3_engine_create_train_sized and everything
above it (GaussianDiffusion.p_losses, DataParallelTrainer.step, the reference's DDPM.optimize_parameters over our define_G).

Gradients are held to the bounds of tests/test_gpu_train.py against the oracle's fp32 autograd on the CPU; the L1 loss and the reference's
Dropout masks against tests/golden/sr3_train_sizes_golden.pt.  The kernels whose geometry changes with the size (the attention backward on
segments of 512 to 4096 tokens, weight and data gradients with OH != OW, the loss gradient) are checked alone against fp64."""
import ctypes

import numpy as np
import pytest
import torch

import _philox
import _train_sizes_inputs as ti
import _train_util as tu
from oracle import sr3_oracle as orc
from test_gpu_backward import attention_operands, check, gen, upsample_dgrad_kernel
from test_gpu_wgrad import operands as wgrad_operands, wgrad_ref
from test_oracle_train_sizes import golden, unpack_masks  # noqa: F401  (golden: module fixture)
from test_reference_wrapper import make_opt as wrapper_opt, ref_model_pkg  # noqa: F401  (ref_model_pkg: fixture)

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-2          # relative L2 per parameter tensor, as tests/test_gpu_train.py
FIVE_LEVEL_TOL = 3e-2    # the 362 tensors of the five-level 16->64 / 16->128 UNet (test_gradients_full_16_128_config)


def build(name, loss_type="l2", dropout=0.0, conditional=True):
    unet, image_size, b, h, w = ti.CASES[name]
    unet = dict(unet, dropout=dropout)
    if not conditional:
        unet["in_channel"] = 3
    return tu.build_train_net(unet, image_size, ti.SEED, loss_type, ti.SCHED, conditional), unet


def compare_with_oracle(name, loss_type="l2", conditional=True):
    _, image_size, b, h, w = ti.CASES[name]
    net, unet = build(name, loss_type, conditional=conditional)
    hr, sr, noise = ti.case_batch(name)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    eng = net.denoise_fn._engines[(b, h, w, "cuda:0", conditional, 3, "bf16", 0.0)]
    assert (eng.height, eng.width) == (h, w)
    torch.set_num_threads(min(16, torch.get_num_threads()))
    lr_, gr = tu.oracle_loss_and_grads(net, unet, image_size, hr, sr, gamma, noise, loss_type)
    return lo, go, lr_, gr


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", sorted(ti.CASES))
def test_gradients_match_oracle_l2(name):
    """Every parameter gradient of one training step at h x w against the oracle: the tiny net at 32x64 / 64x32 (512-token attention) and
    64x64 (1024), the 16->64 net at 128x128 (1024-token attention, lowest level 8x8 so no batch padding to 8), the 16->128 net at 128x256."""
    lo, go, lr_, gr = compare_with_oracle(name)
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    rows = tu.compare(go, gr)
    assert set(go) == set(gr)
    five = len(ti.CASES[name][0]["channel_multiplier"]) == 5
    if five:
        assert len(rows) == 362
    worst = sorted(rows, key=lambda r: -r[1])[:5]
    print(name, "worst:", [(n, f"{e:.2e}") for n, e, _, _ in worst])
    bad = [(n, e, c) for n, e, c, _ in rows if e >= (FIVE_LEVEL_TOL if five else GRAD_TOL)]
    assert not bad, bad[:10]


SR64_512 = dict(in_channel=6, out_channel=3, inner_channel=64, norm_groups=16, channel_multiplier=[1, 2, 4, 8, 16], attn_res=[], res_blocks=1,
                dropout=0.0)     # sr_sr3_64_512.json's UNet


@pytest.mark.timeout(1800)
def test_gradients_64_512_config_match_oracle_l2():
    """sr_sr3_64_512's UNet (16 GroupNorm groups, concats up to 2048 channels, the C = 1024 middle attention) trained on a 128x128 batch of
    2: the loss within 1e-2 and every one of its parameter gradients within GRAD_TOL of the oracle's fp32 autograd.  (Its 16-group
    forward is pinned to the reference by the big_64_512 golden, tests/test_oracle.py.)"""
    b, h = 2, 128
    net = tu.build_train_net(SR64_512, 512, ti.SEED, "l2", ti.SCHED)
    hr, sr, noise = ti.batch(b, h, h, 2000)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    assert (b, h, h, "cuda:0", True, 3, "bf16", 0.0) in net.denoise_fn._engines
    torch.set_num_threads(min(16, torch.get_num_threads()))
    lr_, gr = tu.oracle_loss_and_grads(net, SR64_512, 512, hr, sr, gamma, noise, "l2")
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    assert set(go) == set(gr)
    rows = tu.compare(go, gr)
    worst = sorted(rows, key=lambda r: -r[1])[:5]
    print(f"sr64_512 at {h}x{h}, {len(rows)} parameter tensors, loss {lo:.6g} vs {lr_:.6g}; worst:", [(n, f"{e:.2e}") for n, e, _, _ in worst])
    bad = [(n, e, c) for n, e, c, _ in rows if e >= GRAD_TOL]
    assert not bad, bad[:10]


def test_gradients_unconditional_model_non_square():
    lo, go, lr_, gr = compare_with_oracle("tiny_64x32", conditional=False)
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    for n, e, c, _ in tu.compare(go, gr):
        assert e < GRAD_TOL, (n, e, c)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", ["tiny_32x64", "tiny_64x32"])
def test_l1_loss_against_the_reference(golden, name):  # noqa: F811
    """The loss the reference trains with (L1, sum / (b c h w)): within 1e-2 of the golden loss, gradient norms within 15 % of the golden
    ones, and the gradients close in direction to the reference's: cosine similarity above 0.95 per tensor against the oracle, and over the
    golden's sampled entries of all tensors together (each tensor's samples scaled by its norm)."""
    _, _, b, h, w = ti.CASES[name]
    rec = golden["cases"][name]
    net, unet = build(name, "l1")
    hr, sr, noise = ti.case_batch(name)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    assert abs(lo / (b * 3 * h * w) - rec["loss"]) < 1e-2 * abs(rec["loss"]), (lo / (b * 3 * h * w), rec["loss"])
    ours, ref = [], []
    for k, sig in rec["grads"].items():
        f = go[k].flatten().cpu()
        assert f.numel() == sig["numel"]
        assert abs(f.norm().item() - sig["norm"]) <= 0.15 * sig["norm"] + 1e-12, (k, f.norm().item(), sig["norm"])
        if sig["norm"] > 0:
            stride = max(1, f.numel() // 16)
            ours.append(f[::stride][:16] / sig["norm"])
            ref.append(sig["samples"] / sig["norm"])
    assert tu.cosine(torch.cat(ours), torch.cat(ref)) > 0.95
    _, gr = tu.oracle_loss_and_grads(net, unet, ti.CASES[name][1], hr, sr, gamma, noise, "l1")
    for n, e, cs, _ in tu.compare(go, gr):
        assert cs > 0.95, (n, e, cs)


def test_reference_dropout_masks_at_a_non_square_size(golden):  # noqa: F811
    """The reference's own nn.Dropout masks of one step, [B, C, h, w] with h != w, injected through sr3_train_set_dropout_mask: the loss
    within 1e-2 of the reference's, and different from the eval-mode loss."""
    d = golden["dropout"]
    name = d["case"]
    _, _, b, h, w = ti.CASES[name]
    net, _ = build(name, "l1", dropout=d["p"])
    hr, sr, noise = ti.case_batch(name)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    net.train(True)
    eng = net.denoise_fn.engine(b, conditional=True, channels=3, train_dropout=float(d["p"]), height=h, width=w)
    masks = unpack_masks(d)
    assert sorted(eng.dropout_layers()) == sorted(masks)
    for k, keep in masks.items():
        eng.set_dropout_mask(k, keep.cuda().contiguous())
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True)
    assert abs(lo / (b * 3 * h * w) - d["loss"]) < 1e-2 * abs(d["loss"]), (lo / (b * 3 * h * w), d["loss"])
    for k, sig in d["grads"].items():
        f = go[k].flatten().cpu()
        assert abs(f.norm().item() - sig["norm"]) <= 0.15 * sig["norm"] + 1e-12, (k, f.norm().item(), sig["norm"])
    with torch.no_grad():
        net.eval()
        ev = net.p_losses({"HR": hr.cuda(), "SR": sr.cuda()}, noise=noise.cuda(), gamma=gamma).item()
    assert abs(ev - lo) / lo > 1e-4


def dropout_shapes(name, B):
    """{"downs.1.res_block.block2": (B, C, h, w)}: the activation each block2 Dropout masks, at the case's h x w."""
    unet, image_size, _, h, w = ti.CASES[name]
    downs, mid, ups = orc.unet_topology(tu.oracle_cfg(unet, image_size))
    return {s.name + ".res_block.block2": (B, s.cout, s.res * h // image_size, s.res * w // image_size)
            for s in downs + mid + ups if s.kind == "res"}


@pytest.mark.parametrize("name", ["tiny_32x64", "tiny_64x32"])
def test_philox_dropout_at_a_non_square_size(name):
    """The device's Philox masks at h != w are the numpy restatement's (tests/_philox.py: vector index (b * h w + pixel) * C/4 + c/4): every
    gradient against the oracle on those masks.  A repeated step with the same seed gives the same loss bits (the backward's fp32 atomics
    leave the gradients within the run-to-run bound of test_philox_dropout_is_deterministic)."""
    p, seed = 0.2, 0x5EED0000C0FFEE
    unet, image_size, b, h, w = ti.CASES[name]
    net, unet = build(name, "l2", dropout=p)
    hr, sr, noise = ti.case_batch(name)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    net.train(True)
    eng = net.denoise_fn.engine(b, conditional=True, channels=3, train_dropout=p, height=h, width=w)
    shapes = dropout_shapes(name, b)
    masks = {}
    for layer, k in enumerate(eng.dropout_layers()):
        bb, c, hh, ww = shapes[k]
        keep = _philox.keep_mask(bb, c, hh * ww, p, seed, layer).reshape(bb, c, hh, ww)
        masks[k] = _philox.scale_mask(keep, p)
    l1, g1 = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=seed)
    l2, g2 = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=seed)
    assert l1 == l2
    assert max(tu.rel(g1[k], g2[k]) for k in g1) < 2e-2
    lr_, gr = tu.oracle_loss_and_grads(net, unet, image_size, hr, sr, gamma, noise, "l2", dropout_masks=masks)
    assert abs(l1 - lr_) / abs(lr_) < 1e-2, (l1, lr_)
    for n, e, c, _ in tu.compare(g1, gr):
        assert e < GRAD_TOL, (n, e, c)


# ------------------------------------------------------------------------------------------------ kernels at the new geometries
@pytest.mark.timeout(600)
@pytest.mark.parametrize("nz,Lt,HW,C", [(1, 512, 512, 256), (1, 1024, 1024, 128), (2, 512, 512, 512), (1, 4096, 4096, 128),
                                        (1, 1024, 1024, 1024)])
def test_attention_backward_long_segments_match_fp64(nz, Lt, HW, C):
    """bwd_attention on one image per attention batch of 512 to 4096 tokens (the 16->128 net's attention level at 128x256, 256x256 and
    512x512; the 64->512 net's C = 1024 middle block at 512x512): the bounds of test_attention_backward_matches_fp64.  The row dot of
    the softmax backward and the dK / dV contractions now run over up to 4096 terms in fp32, ~2^-24 sqrt(n) each: still far inside
    2e-5."""
    from sr3_b200 import _native
    g = gen("attn", nz, Lt, HW, C)
    qk, vT, P, dO, inside = attention_operands(nz, Lt, HW, C, g)
    dS, dSb, dqkv, dqkvb = (t.cpu() for t in _native.test_attention_bwd(qk.cuda(), vT.cuda(), P.cuda(), dO.cuda(), nz, Lt, HW, C))
    Q = qk[:, :C].double().view(nz, Lt, C)
    K = qk[:, C:].double().view(nz, Lt, C)
    V = vT.double().view(nz, C, Lt).transpose(1, 2)
    Pd = P.double().view(nz, Lt, Lt)
    dP = dO.double().view(nz, Lt, C) @ V.transpose(1, 2)
    scale = float(np.float32(1.0) / np.sqrt(np.float32(C), dtype=np.float32))
    dS_ref = Pd * (dP - (Pd * dP).sum(-1, keepdim=True)) * scale
    what = f"nz={nz} Lt={Lt} HW={HW} C={C}"
    check(dS.view(nz, Lt, Lt), dS_ref, "dS " + what)
    assert torch.equal(dSb, dS.bfloat16()), "dS_b is not bf16(dS): " + what
    dSk = dSb.double().view(nz, Lt, Lt)
    check(dqkv[:, :C].reshape(nz, Lt, C), dSk @ K, "dQ " + what)
    check(dqkv[:, C:2 * C].reshape(nz, Lt, C), dSk.transpose(1, 2) @ Q, "dK " + what)
    check(dqkv[:, 2 * C:].reshape(nz, Lt, C), Pd.transpose(1, 2) @ dO.double().view(nz, Lt, C), "dV " + what)
    assert torch.equal(dqkvb, dqkv.bfloat16()), "d(qkv) bf16 copy: " + what


NON_SQUARE = [(8, 16), (16, 8), (32, 64)]


@pytest.mark.parametrize("OH,OW", NON_SQUARE)
@pytest.mark.parametrize("k,stride", [(3, 1), (3, 2), (1, 1)])
def test_wgrad_non_square_matches_fp64(OH, OW, k, stride):
    """wgrad_kernel's patch grid per side (OH / 8 x OW / 8 patches): fp32 accumulation of exact bf16 products, 2e-5 against fp64."""
    from sr3_b200 import _native
    import test_gpu_wgrad
    dy, x = wgrad_operands(2, OH, OW, 128, 64, stride, seed=OH * 100 + OW + k + stride)
    got, _ = _native.test_wgrad(dy.cuda(), x.cuda(), k, stride)
    test_gpu_wgrad.check(got.cpu(), wgrad_ref(dy, x, k, stride, 128, 64, 1.0), f"wgrad {OH}x{OW} k={k} s={stride}")


@pytest.mark.parametrize("H,W", NON_SQUARE)
@pytest.mark.parametrize("form", ["conv", "down", "up"])
def test_dgrad_non_square_matches_fp64(H, W, form):
    """The three data-gradient forms at H != W (H x W: the conv's input): stride 1 (mirrored taps), the Downsample's four parity phases on
    the H/2 x W/2 dY grid, and the Upsample's 4x4 stride-2 conv over the 2H x 2W dY; bounds of tests/test_gpu_backward.py."""
    import torch.nn.functional as F
    from sr3_b200 import _native
    B, C = 2, 128
    g = gen("dgrad_ns", H, W, form)
    w = torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5
    oh, ow = {"conv": (H, W), "down": (H // 2, W // 2), "up": (2 * H, 2 * W)}[form]
    dy = torch.randn(B, oh, ow, C, generator=g).bfloat16()
    got = _native.test_dgrad(dy.cuda(), w.cuda(), form, H, W).cpu()
    dyd = dy.double().permute(0, 3, 1, 2)
    if form == "up":
        ref = F.conv2d(dyd, upsample_dgrad_kernel(w).double().permute(2, 3, 0, 1), stride=2, padding=1)
    else:
        ref = torch.nn.grad.conv2d_input((B, C, H, W), w.bfloat16().double(), dyd, stride=1 if form == "conv" else 2, padding=1)
    check(got, ref.permute(0, 2, 3, 1), f"dgrad {form} {H}x{W}")


@pytest.mark.parametrize("H,W", [(4, 4), (8, 16), (16, 8)])
@pytest.mark.parametrize("l2", [False, True])
def test_loss_grad_at_small_and_non_square_images(H, W, l2):
    """loss_grad_kernel at the image's own H x W: the loss, bf16 d loss / d eps and the final-conv bias sum.  A 4x4 image (16 pixels) puts
    two channels in one warp, so the bias sum cannot be a warp reduction there."""
    from sr3_b200 import _native
    B = 3
    g = gen("loss_ns", H, W, l2)
    noise, eps = torch.randn(B, 3, H, W, generator=g), torch.randn(B, 3, H, W, generator=g)
    loss, deps, bias = _native.test_loss_grad(noise.cuda(), eps.cuda(), l2)
    d = eps - noise
    ref = (d.double() ** 2).sum().item() if l2 else d.double().abs().sum().item()
    assert abs(loss - ref) <= 1e-12 * ref, (loss, ref)
    gd = 2 * d if l2 else torch.sign(d)
    assert torch.equal(deps.cpu()[..., :3], gd.permute(0, 2, 3, 1).bfloat16())
    bsum = gd.double().sum((0, 2, 3))
    assert ((bias.cpu().double() - bsum).abs() <= 1e-5 * gd.double().abs().sum((0, 2, 3)) + 1e-6).all(), (bias, bsum)


# ------------------------------------------------------------------------------------------------ plan and wrappers
def test_create_train_sized_at_image_size_is_create_train(monkeypatch):
    """create_train_sized(image_size, image_size) builds the plan create_train builds: the same launches, backward blocks and device bytes,
    and the same loss bits.  (Gradients of two runs differ at the bf16 noise floor: the backward accumulates with fp32 atomics.)"""
    from sr3_b200 import _native
    net, _ = build("tiny_32x64")
    hr, sr, noise = tu.batch(2, 32, 1000)
    gamma = tu.draw_gamma(2, ti.NP_SEED)
    runs = []
    for sized in (True, False):
        net.denoise_fn._engines.clear(); net.denoise_fn._engine_versions.clear()
        if not sized:
            lib = _native.lib()
            plain = lib.sr3_engine_create_train
            monkeypatch.setattr(lib, "sr3_engine_create_train_sized",
                                lambda c, b, h, w, dev, p, out: plain(c, b, dev, p, out) if (h, w) == (32, 32) else 1)
        loss, grads = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
        eng = next(iter(net.denoise_fn._engines.values()))
        runs.append((loss, grads, eng.ops_per_step(), eng.num_backward_blocks(), eng.workspace_bytes()))
    (la, ga, *pa), (lb, gb, *pb) = runs
    assert pa == pb and la == lb
    assert max(tu.rel(ga[k], gb[k]) for k in ga) < 2e-2


def test_p_losses_without_grad_matches_with_grad():
    """The no-grad branch (inference plan) and the autograd branch (training plan) take the size from x_in['HR'] alike."""
    name = "tiny_32x64"
    _, _, b, h, w = ti.CASES[name]
    net, _ = build(name)
    net.eval()
    hr, sr, noise = ti.case_batch(name)
    gamma = tu.draw_gamma(b, ti.NP_SEED)
    x_in = {"HR": hr.cuda(), "SR": sr.cuda()}
    with torch.no_grad():
        a = net.p_losses(x_in, noise=noise.cuda(), gamma=gamma).item()
    l = net.p_losses(x_in, noise=noise.cuda(), gamma=gamma)
    assert l.requires_grad
    assert abs(l.item() - a) <= 2e-3 * abs(a), (l.item(), a)
    assert {k[1:3] for k in net.denoise_fn._engines} == {(h, w)}


def test_weight_update_reaches_the_training_engines_of_two_sizes():
    """Two cached training engines (32x64 and 64x32); an optimizer-style in-place update; both engines then compute the loss of a net built
    with the updated weights, bit for bit."""
    net, _ = build("tiny_32x64")
    gamma = tu.draw_gamma(2, ti.NP_SEED)
    batches = {n: ti.case_batch(n) for n in ("tiny_32x64", "tiny_64x32")}
    for n, (hr, sr, noise) in batches.items():
        tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    assert len([k for k in net.denoise_fn._engines if k[-1] is not None]) == 2
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(1.01)
    after = {n: tu.ours_loss_and_grads(net, *batches[n][:2], gamma, batches[n][2])[0] for n in batches}
    fresh, _ = build("tiny_32x64")
    fresh.load_state_dict(net.state_dict())
    for n in batches:
        assert tu.ours_loss_and_grads(fresh, *batches[n][:2], gamma, batches[n][2])[0] == after[n], n


@pytest.mark.timeout(900)
def test_reference_optimize_parameters_trains_at_128x256(ref_model_pkg, tmp_path):  # noqa: F811
    """model/model.py:48-58 UNMODIFIED over sr3_b200.define_G with the sr_sr3_16_128 UNet on a 128x256 batch: every parameter receives a
    finite, non-zero gradient, and the loss of a fixed batch goes down over three iterations."""
    ref_model, _, _ = ref_model_pkg
    opt = wrapper_opt("train", str(tmp_path))
    opt["gpu_ids"] = [0]
    opt["model"]["unet"] = dict(ti.FULL)
    opt["model"]["diffusion"]["image_size"] = 128
    torch.manual_seed(0)
    np.random.seed(0)
    m = ref_model.create_model(opt)
    losses = []
    for it in range(3):
        data = {"HR": torch.rand(2, 3, 128, 256, generator=torch.Generator().manual_seed(3)) * 2 - 1,
                "SR": torch.rand(2, 3, 128, 256, generator=torch.Generator().manual_seed(4)) * 2 - 1, "Index": torch.arange(2)}
        m.feed_data(data)
        np.random.seed(1)
        torch.manual_seed(1)
        m.optimize_parameters()
        losses.append(m.get_current_log()["l_pix"])
        if it == 0:
            missing = [k for k, p in m.netG.named_parameters() if p.grad is None or not torch.isfinite(p.grad).all() or p.grad.abs().sum() == 0]
            assert not missing, missing[:5]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


def test_refusals_allocate_nothing_and_release_no_engine():
    """An unsupported size, an SR image of another size than HR, and a plan larger than the device: each raises before anything is
    allocated (free device memory unchanged) and leaves the cached engines alone."""
    from sr3_b200 import _native
    net, _ = build("tiny_32x64")
    hr, sr, noise = ti.case_batch("tiny_32x64")
    gamma = tu.draw_gamma(2, ti.NP_SEED)
    tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    cached = dict(net.denoise_fn._engines)
    bad = torch.zeros(2, 3, 8, 16, device="cuda")                # lowest level 4x8
    hr, sr_half, noise = hr.cuda(), sr[..., :32].contiguous().cuda(), noise.cuda()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(_native.UnsupportedSizeError, match="8x16"):
        net.p_losses({"HR": bad, "SR": bad}, noise=bad, gamma=gamma)
    with pytest.raises(ValueError, match="x_in\\['SR'\\] is 32x32 but x_in\\['HR'\\] is 32x64"):
        net.p_losses({"HR": hr, "SR": sr_half}, noise=noise, gamma=gamma)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    assert net.denoise_fn._engines == cached
    # a plan that cannot fit: the 16->128 net, batch 64 at 512x512 (hundreds of GB of kept intermediates)
    c = _native.UNetConfigC()
    c.in_channel, c.out_channel, c.inner_channel, c.norm_groups, c.n_mults = 6, 3, 64, 32, 5
    for i, m in enumerate([1, 2, 4, 8, 8]):
        c.channel_mults[i] = m
    c.n_attn_res, c.attn_res[0] = 1, 16
    c.res_blocks, c.image_size, c.channels, c.conditional = 2, 128, 3, 1
    h_ = ctypes.c_void_p()
    assert _native.lib().sr3_engine_create_train_sized(ctypes.byref(c), 64, 512, 512, torch.cuda.current_device(), 0.0, ctypes.byref(h_)) != 0
    err = _native.lib().sr3_last_error().decode()
    assert "512x512" in err and "batch 64" in err and "bytes" in err, err
    assert not h_.value
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


# ------------------------------------------------------------------------------------------------ two ranks
def _rank_step(rank, world, port, path):
    import os
    import torch.distributed as dist
    from sr3_b200 import parallel
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        out = _trainer_step(dev, *parallel.shard_bounds(4, world, rank))
        torch.save(out, f"{path}.rank{rank}")
    finally:
        dist.destroy_process_group()


def _trainer_step(dev, lo, hi):
    from sr3_b200 import parallel
    net, _ = build("tiny_64x32")
    net = net.to(dev)
    net.eval()
    hr, sr, noise = ti.batch(4, 64, 32, 55)
    gamma = tu.draw_gamma(4, ti.NP_SEED)
    tr = parallel.DataParallelTrainer(net, lr=1e-4, bucket_mb=0.25)
    loss = tr.step(hr[lo:hi].to(dev), sr[lo:hi].to(dev), gamma=gamma[lo:hi], noise=noise[lo:hi].to(dev), global_batch=4)
    torch.cuda.synchronize()
    return {"loss": loss, "grad": tr.buckets.flat.cpu()}


@pytest.mark.timeout(600)
def test_two_rank_training_step_at_64x32_matches_single_process(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from test_gpu_multi import _free_port
    path = str(tmp_path / "tr")
    mp.spawn(_rank_step, args=(2, _free_port(), path), nprocs=2, join=True)
    outs = [torch.load(f"{path}.rank{r}") for r in range(2)]
    assert torch.equal(outs[0]["grad"], outs[1]["grad"])
    one = _trainer_step(torch.device("cuda", 0), 0, 4)
    assert abs(outs[0]["loss"] + outs[1]["loss"] - one["loss"]) < 1e-3 * abs(one["loss"])
    assert ((one["grad"] - outs[0]["grad"]).norm() / one["grad"].norm()).item() < 1e-2


def test_single_process_trainer_step_at_64x32():
    """DataParallelTrainer without a process group at a non-square size: the gradient arena is the p_losses gradient (1 / (b c h w) with
    the real h, w)."""
    one = _trainer_step(torch.device("cuda", 0), 0, 4)
    net, _ = build("tiny_64x32")
    net.eval()
    hr, sr, noise = ti.batch(4, 64, 32, 55)
    _, grads = tu.ours_loss_and_grads(net, hr, sr, tu.draw_gamma(4, ti.NP_SEED), noise)
    flat = torch.cat([grads[k].flatten() for k in grads]).norm()
    assert abs(one["grad"].norm().item() - flat.item()) <= 2e-2 * flat.item()

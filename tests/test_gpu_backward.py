"""Kernel-level tests of the training backward (csrc/train_kernels.cuh, csrc/train_plan.inc) against fp64 references on the CPU, through
hooks that build their launches with the training plan's own helpers (engine.cu: gn_op / prep_launch / gn_bwd_launch, combine_launch,
dgrad_pack_desc and the data-gradient ConvArgs, the attention-backward GemmDescs and WgradOut views, launch_film_bwd / launch_embed_bwd,
launch_loss_grad).  Shapes follow the configs the project ships: channels 64 .. 2048 (the skip concats of the 16->128 config make 192, 384,
768 and 1024, those of the 64->512 config up to 2048 at 16 groups), 4x4 .. 512x512 pixels, batches 1, 3 and 16.

Unless a test says otherwise a result is held to a relative L2 error and, element-wise, to 1e-4 (|ref| + rms(ref)); the first element out of
bound is reported by its index ((image, pixel, channel) for activations).
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _philox

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def check(got, ref, what, bound=2e-5, elem=1e-4):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    r = rel(got, ref)
    assert r < bound, f"{what}: relative L2 {r:.3e} (bound {bound:.1e})"
    bad = ((got - ref).abs() > elem * (ref.abs() + ref.pow(2).mean().sqrt())).nonzero()
    if bad.numel():
        idx = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} elements out of bound, first at {idx}: got {got[idx].item():.7g}, want {ref[idx].item():.7g}")


def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ------------------------------------------------------------------------------------------------ GroupNorm (+SiLU, +Dropout) layer
def channel_sums(x):
    """fp64 (sum, sum of squares) per (image, channel) of x [B, HW, C]: what the producing conv epilogues accumulate."""
    xd = x.double()
    return torch.stack([xd.sum(1), (xd * xd).sum(1)], -1).contiguous()


def gn_reference(x, gamma, beta, groups, silu, dA, mask):
    """fp64 autograd of a = drop(silu(GN(x))): returns (a, dx, dgamma, dbeta); x, dA [B, HW, C]; mask: scaled keep-mask [B, C, HW] or None."""
    B, HW, C = x.shape
    xn = x.double().permute(0, 2, 1).contiguous().requires_grad_(True)
    g = gamma.double().requires_grad_(True)
    b = beta.double().requires_grad_(True)
    y = F.group_norm(xn, groups, g, b, eps=1e-5)
    if silu:
        y = F.silu(y)
    if mask is not None:
        y = y * mask.double()
    y.backward(dA.double().permute(0, 2, 1))
    return y.detach().permute(0, 2, 1), xn.grad.permute(0, 2, 1), g.grad, b.grad


GN_CASES = [
    # B, H, W, C0, C1, groups, silu, acc0, add, ratio, drop
    (2, 16, 16, 128, 64, 32, True, True, True, 0.0, None),        # 192 = 128 + 64: group size 6, group 21 = channels 126..131 spans both
    (2, 16, 16, 128, 64, 32, False, False, False, 0.0, None),
    (1, 128, 128, 64, 0, 32, True, False, True, 0.0, None),       # largest image, group size 2
    (3, 12, 12, 256, 0, 32, False, True, True, 0.0, None),        # 144 pixels: the blocks do not divide the image
    (16, 8, 8, 256, 128, 32, True, True, True, 0.0, None),        # 384, batch 16
    (3, 8, 8, 512, 256, 32, True, False, True, 0.0, None),        # 768: group size 24
    (2, 8, 8, 512, 512, 32, True, True, True, 0.0, None),         # 1024: one pixel per thread column
    (3, 4, 4, 256, 0, 32, True, True, False, 0.0, None),          # 4x4 level
    (3, 4, 4, 384, 0, 16, True, False, True, 0.0, None),          # 16 groups of 24
    (2, 32, 32, 128, 0, 32, True, True, True, 60.0, None),        # |mean| / std ~ 60
    (3, 12, 12, 128, 64, 32, False, False, True, 100.0, None),    # ~100, two sources
    (2, 16, 16, 256, 0, 32, True, False, False, 0.0, ("philox", 0.2, 0x123456789ABCDEF, 3)),
    (3, 12, 12, 128, 0, 32, True, False, False, 0.0, ("philox", 0.5, 7, 0)),
    (3, 8, 8, 512, 0, 32, True, False, False, 0.0, ("mask", 0.1)),
    (1, 32, 32, 64, 0, 32, True, False, False, 0.0, ("mask", 0.3)),
    # 16 groups (sr_sr3_64_512)
    (2, 32, 32, 1024, 1024, 16, True, True, True, 0.0, None),     # 2048: 512-thread blocks, 128-channel groups
    (2, 32, 32, 1024, 512, 16, True, True, True, 0.0, None),      # 1536: 384 threads, group 10 = channels 960..1055 spans both
    (2, 64, 64, 512, 256, 16, True, False, True, 0.0, None),      # 768: group 10 = channels 480..527 spans both
    (1, 512, 512, 64, 0, 16, True, False, True, 0.0, None),       # 262 144 pixels, group size 4
    (2, 32, 32, 256, 0, 16, True, True, True, 60.0, None),        # |mean| / std ~ 60
    (2, 8, 8, 1024, 1024, 16, True, False, False, 0.0, ("philox", 0.2, 0x5EED0000C0FFEE, 9)),   # Philox at 2048 channels
]


@pytest.mark.parametrize("B,H,W,C0,C1,groups,silu,acc0,add,ratio,drop", GN_CASES)
def test_groupnorm_layer_matches_fp64(B, H, W, C0, C1, groups, silu, acc0, add, ratio, drop):
    """prep_kernel (forward apply, (mean, rstd) saved) then both passes of gn_bwd_kernel, launched as the training plan launches them.

    Reference: fp64 autograd of drop(silu(GN(cat(x0, x1)))) with the same keep-mask, plus `add`, plus the old dst0 when accumulating.
    Every step of the kernels is fp32 on operands that are exact: the group statistics are fp64 rounded once to fp32, the per-channel
    sums S1 = sum d, S2 = sum d xh run over <= 64 pixels per thread and then a few hundred block partials.  With |mean| / std = r the fp32
    mean moves xh by ~r 2^-24 (6e-6 at r = 100) and the fp32 x - mean adds as much; the other rounding errors are a few 2^-24 of the terms.
    So the input gradient is held to 5e-5 relative L2 and 1e-4 (|ref| + rms) element-wise.  dgamma / dbeta are sums of B * HW products of
    random sign (|sum| ~ sqrt(n) * term while the rounding grows with n * term): 1e-4 relative L2 and the same element bound.
    Exact: dst0_b == bf16(dst0) bit for bit; a dropped element of `a` is exactly 0.  gsum0 is checked against the sum over pixels of the
    kernel's own dst0 (which includes the accumulated skip part) within 1e-5 of sum |dst0|.  `a` (bf16) is within one bf16 rounding
    (2^-8 |ref|) of the fp64 forward, plus 1e-4 rms for the fp32 arithmetic before the rounding."""
    from sr3_b200 import _native
    g = gen("gn", B, H, W, C0, C1, groups, silu, acc0, add, ratio, str(drop))
    HW, C = H * W, C0 + C1
    x = torch.randn(B, HW, C, generator=g) * (0.5 + torch.rand(C, generator=g))
    if ratio:
        x = x + ratio * (torch.randint(0, 2, (1, 1, C), generator=g) * 2 - 1).float() * (1.0 + 0.1 * torch.rand(C, generator=g))
    gamma = 0.5 + torch.rand(C, generator=g)
    beta = torch.randn(C, generator=g)
    dA = torch.randn(B, HW, C, generator=g)
    addt = torch.randn(B, HW, C + 64, generator=g) if add else None          # a wider row, as the shortcut conv's gradient of a concat
    dst0 = torch.randn(B, HW, C0, generator=g) if acc0 else None
    x0, x1 = x[..., :C0].contiguous(), (x[..., C0:].contiguous() if C1 else None)
    mask, dspec = None, None
    if drop is not None:
        p = drop[1]
        if drop[0] == "philox":
            keep = torch.from_numpy(_philox.keep_mask(B, C, HW, p, drop[2], drop[3]))
            dspec = drop
        else:
            keep = (torch.rand(B, C, HW, generator=g) >= p).to(torch.uint8)
            dspec = ("mask", p, keep.cuda().contiguous())
        mask = _philox.scale_mask(keep, p)
    gscale = 0.37
    cu = lambda t: None if t is None else t.cuda().contiguous()
    out = _native.test_groupnorm_layer(cu(x0), cu(channel_sums(x0)), cu(gamma), cu(beta), groups, silu, cu(dA), x1=cu(x1),
                                       st1=cu(channel_sums(x1)) if C1 else None, add=cu(addt), dst0=cu(dst0), acc0=acc0, drop=dspec, gscale=gscale)
    a_ref, dx, dg, db = gn_reference(x, gamma, beta, groups, silu, dA, mask)
    if add:
        dx = dx + addt[..., :C].double()
    d0 = dx[..., :C0] + (dst0.double() if acc0 else 0)
    what = f"B={B} {H}x{W} C={C0}+{C1} G={groups} silu={silu} acc={acc0} add={add} r={ratio} drop={drop and drop[:2]}"
    check(out["dst0"], d0, "dst0 " + what, bound=5e-5)
    if C1:
        check(out["dst1"], dx[..., C0:], "dst1 " + what, bound=5e-5)
    dst0_dev = out["dst0"].cpu()
    assert torch.equal(out["dst0_b"].cpu(), dst0_dev.bfloat16()), "dst0_b is not bf16(dst0): " + what
    gs_ref = dst0_dev.double().sum(1)
    gs_err = (out["gsum0"].cpu().double() - gs_ref).abs()
    assert (gs_err <= 1e-5 * dst0_dev.double().abs().sum(1)).all(), ("gsum0", gs_err.max().item(), what)
    check(out["dgamma"], gscale * dg, "dgamma " + what, bound=1e-4)
    check(out["dbeta"], gscale * db, "dbeta " + what, bound=1e-4)
    a = out["a"].cpu().double()
    tol = 2.0 ** -8 * a_ref.abs() + 1e-4 * a_ref.pow(2).mean().sqrt()
    bad = ((a - a_ref).abs() > tol).nonzero()
    assert bad.numel() == 0, ("a", tuple(bad[0].tolist()), a[tuple(bad[0].tolist())].item(), a_ref[tuple(bad[0].tolist())].item(), what)
    if mask is not None:
        dropped = (mask == 0).permute(0, 2, 1)
        assert (a[dropped] == 0).all(), "a dropped element of the forward is not 0: " + what
        assert dropped.any() and (~dropped).any()
    xd = x.double().reshape(B, HW, groups, C // groups)
    mean = xd.mean((1, 3))
    rstd = 1.0 / (xd.var((1, 3), unbiased=False) + 1e-5).sqrt()
    check(out["mr"], torch.stack([mean, rstd], -1), "(mean, rstd) " + what, bound=1e-6, elem=1e-5)


@pytest.mark.parametrize("B,C,HW,p,seed,layer", [(2, 256, 256, 0.2, 11, 0), (3, 128, 144, 0.1, 2 ** 40 + 5, 7), (16, 64, 1024, 0.5, 12345, 255)])
def test_philox_keep_rate(B, C, HW, p, seed, layer):
    """The keep-mask reproduced by the numpy Philox (the one test_groupnorm_layer_matches_fp64 proves bit-identical to the device's) keeps a
    fraction 1 - p of the elements, within 4 sigma of a binomial draw; different layers and seeds give different masks."""
    keep = _philox.keep_mask(B, C, HW, p, seed, layer)
    n = keep.size
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(keep.mean() - (1 - p)) < 4 * sigma, (keep.mean(), 1 - p, sigma)
    assert (keep != _philox.keep_mask(B, C, HW, p, seed, (layer + 1) % 256)).any()
    assert (keep != _philox.keep_mask(B, C, HW, p, seed + 1, layer)).any()


def test_philox_known_answer():
    """Philox4x32-10 known-answer vectors of the Random123 distribution (counter, key) -> output."""
    out = _philox.philox4x32_10(0, 0, 0, 0, 0, 0)
    assert [int(w) for w in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    out = _philox.philox4x32_10(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(w) for w in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


# ------------------------------------------------------------------------------------------------ grad_combine + bias gradient
@pytest.mark.parametrize("B,HW,C,two,acc", [(1, 128 * 128, 64, False, True), (3, 16 * 16, 192, True, True), (16, 8 * 8, 512, True, False),
                                           (3, 4 * 4, 1024, False, False), (2, 12 * 12, 384, True, True), (3, 64 * 64, 128, False, True)])
def test_grad_combine_and_bias(B, HW, C, two, acc):
    """grad_combine_kernel is elementwise fp32: dst and dst_b are bit-equal to torch fp32 evaluated in the kernel's order, (a + b) + old.
    gsum (fp32 partial sums over <= 32 pixels per thread, then block and grid atomics) is within 1e-5 of sum |out| of the fp64 column sum
    of the kernel's own output.  bias_grad_kernel sums gsum over images in image order and scales: bit-equal to that fp32 sum, written to
    both destinations."""
    from sr3_b200 import _native
    g = gen("combine", B, HW, C, two, acc)
    a = torch.randn(B, HW, C, generator=g)
    b = torch.randn(B, HW, C, generator=g) if two else None
    old = torch.randn(B, HW, C, generator=g)
    dst = old.clone().cuda()
    db, gs, bias = _native.test_grad_combine(a.cuda(), b.cuda() if two else None, dst, acc=acc, bias_outputs=2, gscale=0.37)
    want = a + b if two else a.clone()
    if acc:
        want = want + old
    assert torch.equal(dst.cpu(), want)
    assert torch.equal(db.cpu(), want.bfloat16())
    gsum = gs.cpu()
    err = (gsum.double() - want.double().sum(1)).abs()
    assert (err <= 1e-5 * want.double().abs().sum(1)).all(), err.max().item()
    s = torch.zeros(C)
    for i in range(B):
        s = s + gsum[i]
    assert torch.equal(bias[0].cpu(), s * torch.tensor(0.37)) and torch.equal(bias[1].cpu(), bias[0].cpu())


# ------------------------------------------------------------------------------------------------ data gradients on the tile kernel
@pytest.mark.parametrize("B,H,W,Cout,Cin,k", [(2, 16, 16, 128, 192, 3), (1, 128, 128, 64, 64, 3), (3, 8, 8, 256, 384, 1), (16, 4, 4, 256, 256, 3),
                                             (2, 16, 16, 1536, 512, 1), (3, 4, 4, 128, 256, 1), (2, 32, 32, 3, 64, 3)])
def test_dgrad_stride1_matches_fp64(B, H, W, Cout, Cin, k):
    """dX of a stride-1 conv: the forward tile kernel on the weights packed by pack_entry type 2 (mirrored taps).  Products of bf16 operands
    are exact and accumulate in fp32 over k*k*Cout terms: 2e-5 relative L2 against fp64 autograd on bf16(W).  The final conv (Cout 3)
    reads its dY from a 64-channel buffer: the 61 padding channels are filled with finite non-zero values and must change nothing."""
    from sr3_b200 import _native
    g = gen("dgrad", B, H, W, Cout, Cin, k)
    CY = (Cout + 63) // 64 * 64
    dy = torch.randn(B, H, W, CY, generator=g).bfloat16()
    if CY != Cout:
        dy[..., Cout:] = 0
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cout * k * k) ** 0.5
    got = _native.test_dgrad(dy.cuda(), w.cuda(), "conv", H, W).cpu()
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w.bfloat16().double(), dy[..., :Cout].double().permute(0, 3, 1, 2), padding=k // 2)
    check(got, ref.permute(0, 2, 3, 1), f"dgrad k={k} {Cout}->{Cin} {H}x{W} B={B}")
    if CY != Cout:
        dy2 = dy.clone()
        dy2[..., Cout:] = (torch.rand(B, H, W, CY - Cout, generator=g) + 0.5).bfloat16() * 1000
        assert torch.equal(_native.test_dgrad(dy2.cuda(), w.cuda(), "conv", H, W).cpu(), got)


@pytest.mark.parametrize("B,H,C", [(3, 8, 128), (16, 8, 256), (1, 128, 64), (2, 32, 192)])
def test_dgrad_downsample_matches_fp64(B, H, C):
    """Downsample (conv3x3 stride 2): four input-parity phases on the low-resolution dY grid, weights packed by pack_entry type 3.  fp32
    accumulation over <= 4C exact products: 2e-5 relative L2 against fp64 autograd on bf16(W)."""
    from sr3_b200 import _native
    g = gen("down", B, H, C)
    dy = torch.randn(B, H // 2, H // 2, C, generator=g).bfloat16()
    w = torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5
    got = _native.test_dgrad(dy.cuda(), w.cuda(), "down", H, H).cpu()
    ref = torch.nn.grad.conv2d_input((B, C, H, H), w.bfloat16().double(), dy.double().permute(0, 3, 1, 2), stride=2, padding=1)
    check(got, ref.permute(0, 2, 3, 1), f"Downsample dgrad {H}->{H // 2} C={C} B={B}")


def upsample_dgrad_kernel(w):
    """pack_entry type 4 restated: K[u][v][ci][co] = sum of the 3x3 taps W[co][ci][r][s] with r = e + 2 - u, s = f + 2 - v (e, f in {0, 1}),
    summed in fp32 in the kernel's order and rounded to bf16 once."""
    C = w.shape[0]
    K = torch.zeros(4, 4, C, C)
    for u in range(4):
        for v in range(4):
            acc = torch.zeros(C, C)                     # [co][ci]
            for e in range(2):
                r = e + 2 - u
                if not 0 <= r <= 2:
                    continue
                for f in range(2):
                    s = f + 2 - v
                    if 0 <= s <= 2:
                        acc = acc + w[:, :, r, s]
            K[u, v] = acc.t()
    return K.bfloat16()


@pytest.mark.parametrize("B,H,C", [(3, 4, 128), (16, 4, 256), (1, 64, 64), (2, 16, 192)])
def test_dgrad_upsample(B, H, C):
    """Upsample (nearest 2x then conv3x3): one 4x4 stride-2 conv over dY, weights packed by pack_entry type 4.
    (1) Against that 4x4 conv restated on the CPU (taps summed in fp32, rounded once) in fp64: 2e-5 relative L2 (exact products, fp32
    accumulation over 16C terms).  (2) Against fp64 autograd of conv3x3(nearest2x(x)) on bf16(W): folding up to four taps before the bf16
    rounding differs from rounding each tap by ~2^-9 relative per weight, so 4e-3 relative L2 and 2^-6 (|ref| + rms) element-wise."""
    from sr3_b200 import _native
    g = gen("up", B, H, C)
    dy = torch.randn(B, 2 * H, 2 * H, C, generator=g).bfloat16()
    w = torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5
    got = _native.test_dgrad(dy.cuda(), w.cuda(), "up", H, H).cpu()
    K = upsample_dgrad_kernel(w).double().permute(2, 3, 0, 1)                # [ci][co][u][v]
    ref = F.conv2d(dy.double().permute(0, 3, 1, 2), K, stride=2, padding=1)
    check(got, ref.permute(0, 2, 3, 1), f"Upsample dgrad (4x4 kernel) {H}->{2 * H} C={C} B={B}")
    x = torch.zeros(B, C, H, H, dtype=torch.float64, requires_grad=True)
    F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w.bfloat16().double(), padding=1).backward(dy.double().permute(0, 3, 1, 2))
    check(got, x.grad.permute(0, 2, 3, 1), f"Upsample dgrad (autograd) {H}->{2 * H} C={C} B={B}", bound=4e-3, elem=2.0 ** -6)


# ------------------------------------------------------------------------------------------------ attention backward
def attention_operands(nz, Lt, HW, C, g):
    qk = (torch.randn(nz * Lt, 2 * C, generator=g) * 0.5).bfloat16()
    vT = torch.randn(nz * C, Lt, generator=g).bfloat16()
    dO = torch.randn(nz * Lt, C, generator=g).bfloat16()
    logits = torch.randn(nz * Lt, Lt, generator=g) * 2
    seg = torch.arange(Lt) // HW
    inside = seg.view(1, Lt) == seg.repeat(nz).view(nz * Lt, 1)
    P = torch.softmax(logits.masked_fill(~inside, float("-inf")), -1).bfloat16()
    return qk, vT, P, dO, inside


@pytest.mark.parametrize("nz,Lt,HW,C", [(2, 256, 256, 512), (2, 128, 64, 256), (1, 128, 16, 128), (3, 128, 16, 256), (2, 128, 64, 1024),
                                        (1, 128, 16, 1024)])
def test_attention_backward_matches_fp64(nz, Lt, HW, C):
    """bwd_attention from the transposes to the bf16 copy of d(qkv): dP = dO V^T and dQ = dS K on the tile kernel, softmax_bwd_kernel over
    HW-token segments, dK = dS^T Q (Q read through the 16-wide view inside the q|k rows) and dV = P^T dO on the weight-gradient kernel.

    dS = P (dP - sum_seg P dP) / sqrt(C) against that formula in fp64 on the bf16 P: dP accumulates C exact products in fp32 and the row
    dot another <= 256 in fp32, each ~2^-24 sqrt(n) of its terms, so 2e-5 relative L2 and 1e-4 (|ref| + rms).  dS is exactly 0 outside a
    row's segment and dS_b == bf16(dS).  dQ and dK against fp64 products on the kernel's own dS_b, dV against fp64 P^T dO: exact bf16
    products, fp32 accumulation over Lt terms, 2e-5.  The bf16 copy of d(qkv) is bit-exact."""
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
    assert (dS[~inside] == 0).all(), "dS outside its segment: " + what
    assert torch.equal(dSb, dS.bfloat16()), "dS_b is not bf16(dS): " + what
    dSk = dSb.double().view(nz, Lt, Lt)
    check(dqkv[:, :C].reshape(nz, Lt, C), dSk @ K, "dQ " + what)
    check(dqkv[:, C:2 * C].reshape(nz, Lt, C), dSk.transpose(1, 2) @ Q, "dK " + what)
    check(dqkv[:, 2 * C:].reshape(nz, Lt, C), Pd.transpose(1, 2) @ dO.double().view(nz, Lt, C), "dV " + what)
    assert torch.equal(dqkvb, dqkv.bfloat16()), "d(qkv) bf16 copy: " + what


# ------------------------------------------------------------------------------------------------ FiLM + noise-level MLP
def film_reference(wf, tau, dfilm, nl, w1, b1, w2, gscale):
    """fp64 autograd of film = W_f tau + b_f + cb (loss = sum dfilm * film) with tau = W2 swish(W1 PE(nl) + b1) + b2 recomputed from nl."""
    inner = wf.shape[1]
    d = lambda t: t.double().clone().requires_grad_(True)
    Wf, Bf, Cb, W1, B1, W2, B2 = d(wf), d(torch.zeros(wf.shape[0])), d(torch.zeros(wf.shape[0])), d(w1), d(b1), d(w2), d(torch.zeros(inner))
    count = inner // 2
    e = nl.double().view(-1, 1) * torch.exp(-np.log(10000.0) * torch.arange(count, dtype=torch.float64) / count).view(1, -1)
    pe = torch.cat([e.sin(), e.cos()], 1)
    pre = pe @ W1.t() + B1
    tau_r = F.silu(pre) @ W2.t() + B2
    t_in = tau.double().clone().requires_grad_(True)            # the forward's tau (W_f's gradient reads it as given)
    film = t_in @ Wf.t() + Bf + Cb
    film.backward(dfilm.double())
    tau_r.backward(t_in.grad)
    return {"dwf": gscale * Wf.grad, "dbf": gscale * Bf.grad, "dcb": gscale * Cb.grad, "dtau": t_in.grad, "dw1": gscale * W1.grad,
            "db1": gscale * B1.grad, "dw2": gscale * W2.grad, "db2": gscale * B2.grad}


@pytest.mark.parametrize("B,inner", [(1, 64), (3, 64), (16, 64), (80, 64), (3, 128), (40, 128)])
def test_film_and_mlp_backward(B, inner):
    """film_bwd_kernel (into a zeroed dtau, atomics) then embed_bwd_kernel (the MLP recomputed in shared memory).  fp32 sums over B
    images, F film channels (dtau) and inner / 4 inner hidden units, each ~2^-24 sqrt(n) of its terms; PE recomputed with fp32 expf / sinf
    (a few ulp): 2e-5 relative L2 and 1e-4 (|ref| + rms).  B = 80 (inner 64) and 40 (inner 128) are the largest batches the shared memory
    of one block admits."""
    from sr3_b200 import _native
    g = gen("film", B, inner)
    F_ = 1000                                                   # not a multiple of the 64-channel blocks
    wf = torch.randn(F_, inner, generator=g) / inner ** 0.5
    tau = torch.randn(B, inner, generator=g)
    dfilm = torch.randn(B, F_, generator=g)
    nl = torch.rand(B, generator=g)
    w1 = torch.randn(4 * inner, inner, generator=g) / inner ** 0.5
    b1 = torch.randn(4 * inner, generator=g) * 0.1
    w2 = torch.randn(inner, 4 * inner, generator=g) / (4 * inner) ** 0.5
    got = _native.test_film_embed_bwd(*(t.cuda() for t in (wf, tau, dfilm, nl, w1, b1, w2)), gscale=0.37)
    ref = film_reference(wf, tau, dfilm, nl, w1, b1, w2, 0.37)
    for k in ref:
        check(got[k], ref[k], f"{k} B={B} inner={inner}")


@pytest.mark.parametrize("B,inner", [(81, 64), (41, 128)])
def test_film_and_mlp_backward_refuses_a_batch_past_shared_memory(B, inner):
    from sr3_b200 import _native
    z = lambda *s: torch.zeros(*s, device="cuda")
    with pytest.raises(RuntimeError, match="too large"):
        _native.test_film_embed_bwd(z(64, inner), z(B, inner), z(B, 64), z(B), z(4 * inner, inner), z(4 * inner), z(inner, 4 * inner))


# ------------------------------------------------------------------------------------------------ loss gradient
@pytest.mark.parametrize("B,H", [(1, 32), (3, 16), (16, 128)])
@pytest.mark.parametrize("l2", [False, True])
def test_loss_grad(B, H, l2):
    """loss_grad_kernel: the summed L1 / L2 loss (fp64 accumulation of the fp32 differences: within 1e-12 of fp64), d loss / d eps written
    bit-exactly as bf16 into channels 0..2 of a 64-channel buffer (sign(d) for L1, exact zeros included; bf16(2 d) for L2), the 61 padding
    channels untouched, and the final-conv bias sum (exact for L1: a sum of small integers; 1e-5 of sum |2 d| for L2)."""
    from sr3_b200 import _native
    g = gen("loss", B, H, l2)
    noise = torch.randn(B, 3, H, H, generator=g)
    eps = torch.randn(B, 3, H, H, generator=g)
    tie = torch.rand(B, 3, H, H, generator=g) < 0.05
    eps[tie] = noise[tie]                                        # d == 0: sign 0
    deps = torch.full((B, H, H, 64), 7.0).bfloat16()
    loss, deps, bias = _native.test_loss_grad(noise.cuda(), eps.cuda(), l2, deps=deps.cuda())
    d = eps - noise                                              # fp32, as the kernel forms it
    ref = (d.double() ** 2).sum().item() if l2 else d.double().abs().sum().item()
    assert abs(loss - ref) <= 1e-12 * ref, (loss, ref)
    gd = 2 * d if l2 else torch.sign(d)
    deps = deps.cpu()
    assert torch.equal(deps[..., :3], gd.permute(0, 2, 3, 1).bfloat16())
    assert (deps[..., 3:] == 7.0).all()
    bsum = gd.double().sum((0, 2, 3))
    if l2:
        assert ((bias.cpu().double() - bsum).abs() <= 1e-5 * gd.double().abs().sum((0, 2, 3))).all(), (bias, bsum)
    else:
        assert torch.equal(bias.cpu().double(), bsum)

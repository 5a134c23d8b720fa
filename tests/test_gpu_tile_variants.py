"""Every variant of the implicit-GEMM tile kernel (gemm_wgmma.cuh) in the forms the UNet builds, against fp64 references on the CPU.

The host picks the tile shape, split-K factor and pipeline depth from a byte model of the device (conv_geometry / pick_stages in
engine.cu), so a test shape alone does not say which variant runs.  These tests force each one with the SR3_* knobs the host reads on
every call, run it through sr3_test_conv_ex (the layer builders' own descriptor code) and check the geometry the hook reports: a variant
the host replaced or capped fails the case, and the last test fails if any intended (tall, MH, BLOCK_N, one stage, split) cell did not run.

References are computed in fp64 from the same bf16-rounded operands: F.conv2d in double, bias / per-image bias / residual added in double.
The kernel multiplies bf16 exactly and accumulates in fp32 over K <= 2304 products, an error of order sqrt(K) 2^-24 of the partial sums
(~3e-6 of the output rms): relative L2 below 2e-5, and element-wise within 1e-4 (|ref| + rms(ref)).
"""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TALL_ENV = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_MAX_CTAS")
REPORTS = {}          # case id -> (intended cell, reported geometry)


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def check_close(y, ref, what, rtol_l2=2e-5, elem=None):
    """y fp32 NHWC (CPU), ref fp64 NHWC.  elem: element-wise bound tensor (default 1e-4 (|ref| + rms(ref)))."""
    r = rel(y.double(), ref)
    assert r < rtol_l2, f"{what}: relative L2 {r:.3e} >= {rtol_l2:.1e}"
    err = (y.double() - ref).abs()
    bound = elem if elem is not None else 1e-4 * (ref.abs() + ref.pow(2).mean().sqrt())
    bad = (err > bound).nonzero()
    if bad.numel():
        b, h, w, c = bad[0].tolist()
        pytest.fail(f"{what}: {bad.shape[0]} elements out of bound, first at (image {b}, row {h}, column {w}, channel {c}): "
                    f"got {y[b, h, w, c].item():.7g}, want {ref[b, h, w, c].item():.7g}")


def check_stats(stats, ref):
    st = stats.cpu()
    refc = nchw(ref)
    assert torch.allclose(st[..., 0], refc.sum(dim=(2, 3)), rtol=1e-4, atol=1e-3), "GroupNorm sums"
    assert torch.allclose(st[..., 1], (refc ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=1e-3), "GroupNorm sums of squares"


def check_bf16_copy(yb, y):
    assert torch.equal(yb.cpu(), y.bfloat16()), "bf16 copy differs from bf16(fp32 output)"


def conv_ref(x, w, stride, bias=None, bias2=None, resid=None):
    """fp64 NHWC reference of the tile kernel's image conv: x bf16 NHWC, w fp32 OIHW (rounded to bf16 like the packer)."""
    k = w.shape[-1]
    y = F.conv2d(nchw(x.double()), w.bfloat16().double(), stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.double()
    if bias2 is not None:
        y = y + bias2.double()[:, None, None, :]
    if resid is not None:
        y = y + resid.double()
    return y


# ------------------------------------------------------------------------------------------------ variant sweep
class Form:
    def __init__(self, name, tall, mh, bn, B, H, W, Cin, Cout, k, s, h_box=None, b_box=None, max_one_resid=False, max_one_split=False,
                 two_fits_resid=True, two_fits=True, split_ok=True, resid_ok=True):
        self.name, self.tall, self.mh, self.bn = name, tall, mh, bn
        self.B, self.H, self.W, self.Cin, self.Cout, self.k, self.s = B, H, W, Cin, Cout, k, s
        self.h_box, self.b_box = h_box, b_box
        self.max_one_resid, self.max_one_split = max_one_resid, max_one_split
        self.two_fits_resid, self.two_fits, self.split_ok, self.resid_ok = two_fits_resid, two_fits, split_ok, resid_ok

    def env(self, split, stages, max_ctas=None):
        e = {"SR3_KSPLIT": str(split)}
        if self.tall:
            e.update(SR3_TALL_BN=str(self.bn), SR3_TALL_MH=str(self.mh))
        else:
            e["SR3_BLOCK_N"] = str(self.bn)
        if stages is not None:
            e["SR3_STAGES"] = str(stages)
        if max_ctas is not None:
            e["SR3_MAX_CTAS"] = str(max_ctas)
        return e


# Shared-memory budget on sm_90 (232 448 B per CTA): a stage holds the A box(es) and up to three 64-column B panels; the epilogue takes
# 32 KB, or 96 KB when the residual is staged through shared memory (unsplit tiles only).  So a generic 128 x 128 / 128 x 256 stage of
# three grouped 3x3 slabs (96 / 144 KB) always runs alone, as do tall 256 x 128 and generic 128 x 64 tiles with a staged residual; a
# 144 KB stage and the 96 KB residual staging do not fit at all (the host refuses), so unsplit generic 128 x 256 3x3 cases have no residual.
FORMS = [
    Form("tall256x128_h32", 1, 2, 128, 2, 32, 32, 256, 128, 3, 1, h_box=32, b_box=1, max_one_resid=True, two_fits_resid=False),
    Form("tall256x128_h16x2", 1, 2, 128, 4, 16, 16, 256, 128, 3, 1, h_box=16, b_box=2, max_one_resid=True, two_fits_resid=False),
    Form("tall256x64", 1, 2, 64, 2, 32, 32, 128, 128, 3, 1, h_box=32, b_box=1),
    Form("tall128x64", 1, 1, 64, 2, 16, 16, 128, 128, 3, 1, h_box=16, b_box=1),
    Form("tall128x32", 1, 1, 32, 2, 16, 16, 128, 64, 3, 1, h_box=16, b_box=1),
    Form("gen128x32_stride2", 0, 1, 32, 2, 32, 32, 128, 64, 3, 2),
    Form("gen128x32_8x8", 0, 1, 32, 4, 8, 8, 128, 64, 3, 1, b_box=2),
    Form("gen128x32_1x1", 0, 1, 32, 2, 16, 16, 768, 64, 1, 1),
    Form("gen128x64_stride2", 0, 1, 64, 2, 32, 32, 128, 128, 3, 2, max_one_resid=True, two_fits_resid=False),
    Form("gen128x64_8x8", 0, 1, 64, 4, 8, 8, 128, 128, 3, 1, b_box=2, max_one_resid=True, two_fits_resid=False),
    Form("gen128x64_1x1", 0, 1, 64, 2, 16, 16, 768, 128, 1, 1, max_one_resid=True, two_fits_resid=False),
    Form("gen128x128_stride2", 0, 1, 128, 2, 32, 32, 128, 128, 3, 2, max_one_resid=True, max_one_split=True, two_fits=False,
         two_fits_resid=False),
    Form("gen128x128_8x8", 0, 1, 128, 4, 8, 8, 128, 256, 3, 1, b_box=2, max_one_resid=True, max_one_split=True, two_fits=False,
         two_fits_resid=False),
    Form("gen128x128_1x1", 0, 1, 128, 2, 16, 16, 64, 256, 1, 1, split_ok=False),
    Form("gen128x256_stride2", 0, 1, 256, 2, 32, 32, 128, 256, 3, 2, max_one_resid=True, max_one_split=True, two_fits=False,
         two_fits_resid=False, resid_ok=False),
    Form("gen128x256_8x8", 0, 1, 256, 4, 8, 8, 128, 512, 3, 1, b_box=2, max_one_resid=True, max_one_split=True, two_fits=False,
         two_fits_resid=False, resid_ok=False),
    Form("gen128x256_1x1", 0, 1, 256, 2, 16, 16, 64, 256, 1, 1, split_ok=False),
]


def sweep_cases():
    """(id, form, split, stages requested (None = as many as fit), residual, max_ctas, expected one-stage)."""
    out = []
    for f in FORMS:
        for split in ((1, 2) if f.split_ok else (1,)):
            for stages in (1, 2, None):
                resid = f.resid_ok or split > 1
                if stages == 2 and split > 1 and not f.two_fits:          # a split tile reads its residual with plain loads
                    continue
                if stages == 2 and split == 1 and not f.two_fits_resid:
                    if not f.two_fits:
                        continue
                    resid = False                                           # two stages fit only without the staged residual
                one = stages == 1 or (stages is None and (f.max_one_split if split > 1 else f.max_one_resid))
                out.append((f"{f.name}-split{split}-stages{stages or 'max'}{'' if resid else '-noresid'}", f, split, stages, resid, None, one))
        # CTAs that walk several tiles across image boundaries (split 1 only: a split tile needs one CTA per (tile, split) pair)
        out.append((f"{f.name}-ctas3{'' if f.resid_ok else '-noresid'}", f, 1, None, f.resid_ok, 3, f.max_one_resid))
    return out


CASES = sweep_cases()


def run_case(monkeypatch, f, split, stages, resid, max_ctas, seed):
    from sr3_b200 import _native
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in f.env(split, stages, max_ctas).items():
        monkeypatch.setenv(k, v)
    g = torch.Generator().manual_seed(seed)
    OH, OW = f.H // f.s, f.W // f.s
    x = torch.randn(f.B, f.H, f.W, f.Cin, generator=g).bfloat16()
    w = torch.randn(f.Cout, f.Cin, f.k, f.k, generator=g) / math.sqrt(f.Cin * f.k * f.k)
    bias = torch.randn(f.Cout, generator=g)
    bias2 = torch.randn(f.B, f.Cout, generator=g)
    res = torch.randn(f.B, OH, OW, f.Cout, generator=g) if resid else None
    y, yb, stats, geo = _native.test_conv_ex(x.cuda(), w.cuda(), f.k, f.s, bias=bias.cuda(), bias2=bias2.cuda(),
                                             resid=res.cuda() if resid else None, want_bf16=True, want_stats=True)
    ref = conv_ref(x, w, f.s, bias, bias2, res)
    return y.cpu(), yb, stats, geo, ref


@pytest.mark.parametrize("cid,f,split,stages,resid,max_ctas,one", CASES, ids=[c[0] for c in CASES])
def test_tile_variant(monkeypatch, cid, f, split, stages, resid, max_ctas, one):
    y, yb, stats, geo, ref = run_case(monkeypatch, f, split, stages, resid, max_ctas, seed=zlib.crc32(cid.encode()))
    cell = (f.tall, f.mh, f.bn, one, split > 1)
    REPORTS[cid] = (cell, geo)
    got = (geo["tall"], geo["mh"], geo["block_n"], geo["stages"] == 1, geo["ksplit"] > 1)
    assert got == cell, f"{cid}: host ran {geo}, intended (tall, mh, block_n, one stage, split) = {cell}"
    if stages is not None:
        assert geo["stages"] == stages, f"{cid}: {stages} stages requested, host ran {geo['stages']}"
    if f.h_box is not None:
        assert geo["h_box"] == f.h_box, geo
    if f.b_box is not None:
        assert geo["b_box"] == f.b_box, geo
    if split > 1:
        assert geo["ksplit"] == split and geo["res_smem"] == 0, geo
    else:
        assert geo["res_smem"] == int(resid), geo
    if max_ctas is not None:
        assert geo["ctas"] == max_ctas and geo["tiles"] > max_ctas, geo
    check_close(y, ref, cid)
    check_stats(stats, ref)
    check_bf16_copy(yb, y)


def test_split_launch_with_too_few_ctas_is_refused(monkeypatch):
    """SR3_MAX_CTAS with a split tile would give one CTA two splits of the same tile, which then waits for itself at the split-K counter.
    make_gemm_op refuses the combination while it builds the op, before any tile kernel is launched."""
    from sr3_b200 import _native
    f = next(f for f in FORMS if f.name == "gen128x32_stride2")     # 8 output tiles, splits 2 ways
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in f.env(2, None, 4).items():
        monkeypatch.setenv(k, v)
    x = torch.zeros(f.B, f.H, f.W, f.Cin, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(f.Cout, f.Cin, 3, 3, device="cuda")
    with pytest.raises(RuntimeError, match="one CTA per"):
        _native.test_conv_ex(x, w, 3, 2)


# ------------------------------------------------------------------------------------------------ ResnetBlock block2 + 1x1 shortcut
@pytest.mark.parametrize("cin,cout,B,H", [(128, 64, 2, 16), (64, 128, 2, 32), (128, 64, 4, 8), (64, 128, 2, 16)])
def test_block2_with_shortcut(monkeypatch, cin, cout, B, H):
    """add_res_block's second conv when cin != cout: conv3x3 over the block's hidden state a (cout channels) with the res_conv 1x1 over the
    block input (cin channels) appended as extra K columns of the same GEMM.  Reference conv3x3(a) + conv1x1(raw) + both biases in fp64."""
    from sr3_b200 import _native
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)
    g = torch.Generator().manual_seed(cin * 3 + cout + H)
    a = torch.randn(B, H, H, cout, generator=g).bfloat16()
    raw = torch.randn(B, H, H, cin, generator=g).bfloat16()
    w = torch.randn(cout, cout, 3, 3, generator=g) / math.sqrt(cout * 9)
    wr = torch.randn(cout, cin, 1, 1, generator=g) / math.sqrt(cin)
    b2, br = torch.randn(cout, generator=g), torch.randn(cout, generator=g)
    y, yb, stats, geo = _native.test_conv_ex(a.cuda(), w.cuda(), 3, 1, bias=(b2 + br).cuda(), x2=raw.cuda(), w2=wr.cuda(), want_bf16=True,
                                             want_stats=True)
    ref = conv_ref(a, w, 1, b2) + conv_ref(raw, wr, 1, br)
    assert geo["tall"] == (1 if H >= 16 else 0), geo
    y = y.cpu()
    check_close(y, ref, f"block2 {cin}->{cout} at {H}x{H}")
    check_stats(stats, ref)
    check_bf16_copy(yb, y)


# ------------------------------------------------------------------------------------------------ folded upsample
FOLD_ROWS = {(0, 0): (0, 0), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2, 2)}     # phase parity, tap offset a -> kernel rows [r0, r1]


def fold_weights(w):
    """The four 2x2 phase kernels of nearest-2x -> conv3x3, as `pack_entry` type 5 forms them: the aliased taps summed in fp32 in
    row-then-column order, rounded once to bf16.  Returns [4][Cout][Cin][2][2] (fp32 holding bf16 values), phase = 2 py + px."""
    out = torch.zeros(4, w.shape[0], w.shape[1], 2, 2)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    r0, r1 = FOLD_ROWS[(py, a)]
                    s0, s1 = FOLD_ROWS[(px, b)]
                    acc = torch.zeros(w.shape[0], w.shape[1])
                    for rr in range(r0, r1 + 1):
                        for ss in range(s0, s1 + 1):
                            acc = acc + w[:, :, rr, ss]
                    out[2 * py + px, :, :, a, b] = acc.bfloat16().float()
    return out


@pytest.mark.parametrize("B,H,C,tall", [(2, 8, 64, 0), (2, 8, 128, 0), (2, 16, 64, 1), (2, 16, 128, 1)])
def test_folded_upsample(monkeypatch, B, H, C, tall):
    """Upsample (unet.py:58-65: nearest 2x, then conv3x3) run as the engine runs it: the four output phases of the conv folded onto the
    low-res input in one launch (gemm-batch z = phase, output map {2N, W, 2, H, B}).  Two references:
      * the fold restated on the CPU (aliased taps summed in fp32, rounded once to bf16), each phase a 2x2 conv in fp64: rel 2e-5;
      * conv2d(interpolate(x, 2, nearest), w) on the unfolded bf16 weights: the fold is the reference operation, up to one extra bf16
        rounding of each summed weight (2^-9 relative): rel 4e-3."""
    from sr3_b200 import _native
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)
    g = torch.Generator().manual_seed(B + H * 5 + C)
    x = torch.randn(B, H, H, C, generator=g).bfloat16()
    w = torch.randn(C, C, 3, 3, generator=g) / math.sqrt(C * 9)
    bias = torch.randn(C, generator=g)
    y, _, stats, geo = _native.test_conv_ex(x.cuda(), w.cuda(), 3, 1, bias=bias.cuda(), fold_up=True, want_stats=True)
    assert geo["tall"] == tall and geo["tiles"] % 4 == 0, geo
    # the bf16 store has no phase offsets: the host refuses a bf16 copy of this output instead of writing the phases on top of each other
    with pytest.raises(RuntimeError, match="phase-addressed"):
        _native.test_conv_ex(x.cuda(), w.cuda(), 3, 1, fold_up=True, want_bf16=True)
    y = y.cpu()
    wf = fold_weights(w).double()
    xp = F.pad(nchw(x.double()), (1, 1, 1, 1))
    ref = torch.empty(B, C, 2 * H, 2 * H, dtype=torch.float64)
    for py in range(2):
        for px in range(2):
            ref[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + H + 1], wf[2 * py + px])
    ref = ref.permute(0, 2, 3, 1) + bias.double()
    check_close(y, ref, f"folded upsample {H}->{2 * H}, C={C}")
    check_stats(stats, ref)
    up = F.interpolate(nchw(x.double()), scale_factor=2, mode="nearest")
    ref2 = F.conv2d(up, w.bfloat16().double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    assert rel(y.double(), ref2) < 4e-3, rel(y.double(), ref2)


# ------------------------------------------------------------------------------------------------ precise mode
def hi_lo(t):
    hi = t.bfloat16()
    return torch.cat([hi, (t - hi.float()).bfloat16()], dim=-1)


@pytest.mark.parametrize("B,H,Cin,Cout,tall", [(2, 32, 128, 128, 1), (4, 8, 128, 128, 0)])
def test_precise_mode_is_fp32_accurate(monkeypatch, B, H, Cin, Cout, tall):
    """Precise mode on fp32 operands that are NOT pre-rounded, against an fp64 conv of the same fp32 values.

    Each operand v is split into hi = bf16(v) and lo = bf16(v - hi); RNE gives |v - hi| <= 2^-9 |v| and |v - hi - lo| <= 2^-9 |v - hi|
    <= 2^-18 |v|.  The kernel forms hi_x hi_w + hi_x lo_w + lo_x hi_w: against x w it drops lo_x lo_w (<= 2^-18 |x w|) and the two
    residual terms hi_x r_w, r_x hi_w (<= 2^-18 |x w| each, to first order), so a product is off by at most 3 * 2^-18 ~ 2^-16.4 of |x w|,
    about 2^-17 in practice.  fp32 accumulation of the 3 K products adds ~ sqrt(3K) 2^-24 of sum |x w|.  Hence element-wise
    |y - ref| <= 2^-15 sum |x w| (+ 2^-22 |ref| for the bias and residual additions), and with random signs the relative L2 error is a few
    1e-6: bound 2e-5.  The same inputs through the plain bf16 path are off by ~2^-9 per operand and must exceed 1e-3."""
    from sr3_b200 import _native
    for k in TALL_ENV:
        monkeypatch.delenv(k, raising=False)
    g = torch.Generator().manual_seed(B * 13 + H + Cin)
    x = torch.randn(B, H, H, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (3.0 / math.sqrt(Cin * 9))      # conv part ~3x the bias and residual
    bias = torch.randn(Cout, generator=g)
    res = torch.randn(B, H, H, Cout, generator=g)
    y, yb, _, geo = _native.test_conv_ex(hi_lo(x).cuda(), w.cuda(), 3, 1, bias=bias.cuda(), resid=res.cuda(), want_bf16=True, precise=True)
    assert geo["tall"] == tall, geo
    y = y.cpu()
    ref = F.conv2d(nchw(x.double()), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1) + res.double()
    absdot = F.conv2d(nchw(x.double().abs()), w.double().abs(), padding=1).permute(0, 2, 3, 1)
    check_close(y, ref, "precise mode", rtol_l2=2e-5, elem=2.0 ** -15 * absdot + 2.0 ** -22 * ref.abs())
    yb = yb.cpu()
    hi = y.bfloat16()
    assert torch.equal(yb[..., :Cout], hi) and torch.equal(yb[..., Cout:], (y - hi.float()).bfloat16()), "precise bf16 [hi | lo] copy"
    y16, _, _, _ = _native.test_conv_ex(x.bfloat16().cuda(), w.cuda(), 3, 1, bias=bias.cuda(), resid=res.cuda())
    assert rel(y16.cpu().double(), ref) > 1e-3, "the bf16 path is as accurate as precise mode: the test cannot tell them apart"


# ------------------------------------------------------------------------------------------------ coverage
def test_every_intended_variant_cell_ran():
    """Runs after the sweep (file order): every (tall, MH, BLOCK_N, one stage, split) cell the sweep intends must have been reported by
    the host as launched.  Prints the geometry of every case."""
    intended = {(f.tall, f.mh, f.bn, one, split > 1) for _, f, split, _, _, _, one in CASES}
    ran = set()
    for cid, (cell, geo) in sorted(REPORTS.items()):
        print(f"{cid:48s} tall={geo['tall']} mh={geo['mh']} block_n={geo['block_n']:3d} h_box={geo['h_box']:2d} b_box={geo['b_box']} "
              f"ksplit={geo['ksplit']} stages={geo['stages']} ctas={geo['ctas']:3d} tiles={geo['tiles']:3d} res_smem={geo['res_smem']}")
        if (geo["tall"], geo["mh"], geo["block_n"], geo["stages"] == 1, geo["ksplit"] > 1) == cell:
            ran.add(cell)
    missing = sorted(intended - ran)
    assert not missing, f"variant cells that did not run as intended: {missing}"
    mode0 = {(mh, bn) for (_, mh, bn, _, _) in ran}
    assert mode0 == {(1, 32), (1, 64), (2, 64), (1, 128), (2, 128), (1, 256)}, mode0

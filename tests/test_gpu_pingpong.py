"""The ping-pong schedule of the tile kernel (gemm_tile_body<..., PP = true>): each consumer warpgroup owns whole tiles and the two take
turns at the MMAs, so one warpgroup's epilogue overlaps the other one's main loop.

Every case forces the schedule with SR3_PINGPONG=1 (and the tile shape with the SR3_* knobs where it matters), runs through
sr3_test_conv_ex and checks that the host reports the ping-pong schedule (sr3_tile_schedule) before comparing with the fp64 references and
bounds of test_gpu_tile_variants.py, whose helpers are reused.  CTA counts are chosen so that warpgroups walk several tiles across image
boundaries, CTAs hold odd tile counts (warpgroup 1 gets one tile fewer) or exactly one tile (warpgroup 1 gets none).
"""
import math
import zlib

import pytest
import torch

import test_gpu_tile_variants as tv
import test_gpu_unet as tu

pytestmark = pytest.mark.gpu

KNOBS = tv.TALL_ENV + ("SR3_PINGPONG",)


def pingpong_env(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("SR3_PINGPONG", "1")


def check_pingpong():
    from sr3_b200 import _native
    s = _native.last_test_conv_schedule()
    assert s is not None and s["schedule"] == "pingpong" and s["ksplit"] == 1, s
    return s


# the ping-pong instantiations in the forms the UNet builds: tall 256x64 (one 8x32 image patch, and two images of 8x16 per tile: the two
# halves of a tile are different images), tall 128x64, generic 128x64 / 128x128 at stride 2, 1x1 and 8x8 (two images per tile)
FORMS = [f for f in tv.FORMS if f.name in ("tall256x64", "tall128x64", "gen128x64_stride2", "gen128x64_8x8", "gen128x64_1x1",
                                           "gen128x128_stride2", "gen128x128_8x8", "gen128x128_1x1")]
FORMS.append(tv.Form("tall256x64_h16x2", 1, 2, 64, 6, 16, 16, 128, 128, 3, 1, h_box=16, b_box=2))
assert len(FORMS) == 9


def cases():
    out = []
    for f in FORMS:
        for stages in (1, 2, None):
            if stages == 2 and not f.two_fits_resid and not f.two_fits:
                continue
            resid = f.resid_ok and not (stages == 2 and not f.two_fits_resid)
            # max_ctas None: one tile per CTA (warpgroup 1 idle); 2 and 3: several tiles per CTA (every form has 4, 8 or 16 tiles), odd and
            # even counts
            for ctas in (None, 2, 3):
                out.append((f"{f.name}-stages{stages or 'max'}-ctas{ctas or 'all'}{'' if resid else '-noresid'}", f, stages, resid, ctas))
    return out


CASES = cases()


@pytest.mark.parametrize("cid,f,stages,resid,ctas", CASES, ids=[c[0] for c in CASES])
def test_pingpong_variant(monkeypatch, cid, f, stages, resid, ctas):
    pingpong_env(monkeypatch)
    y, yb, stats, geo, ref = tv.run_case(monkeypatch, f, 1, stages, resid, ctas, seed=zlib.crc32(cid.encode()))
    s = check_pingpong()
    assert (s["tall"], s["mh"], s["block_n"]) == (f.tall, f.mh, f.bn), s
    if f.h_box is not None:
        assert (s["h_box"], s["b_box"]) == (f.h_box, f.b_box or 1), s
    if stages is not None:
        assert s["stages"] == stages, s
    if ctas is not None:
        assert s["ctas"] == ctas and s["tiles"] > ctas, s
    else:
        assert s["ctas"] == s["tiles"], s                       # exactly one tile per CTA
    assert s["res_smem"] == int(resid), s
    tv.check_close(y, ref, cid)
    tv.check_stats(stats, ref)
    tv.check_bf16_copy(yb, y)


def test_split_request_runs_unsplit(monkeypatch):
    """A ping-pong launch is never split: SR3_KSPLIT=2 with SR3_PINGPONG=1 runs the ping-pong tile unsplit, and correctly."""
    pingpong_env(monkeypatch)
    f = next(f for f in FORMS if f.name == "tall256x64")
    y, yb, stats, geo, ref = tv.run_case(monkeypatch, f, 2, None, True, None, seed=7)
    check_pingpong()
    tv.check_close(y, ref, "split request")
    tv.check_stats(stats, ref)


def test_repeat_launches_are_bit_identical(monkeypatch):
    pingpong_env(monkeypatch)
    f = next(f for f in FORMS if f.name == "tall256x64_h16x2")
    runs = [tv.run_case(monkeypatch, f, 1, None, True, 5, seed=11) for _ in range(2)]
    check_pingpong()
    (y0, yb0, st0, _, _), (y1, yb1, st1, _, _) = runs
    assert torch.equal(y0, y1) and torch.equal(yb0, yb1) and torch.equal(st0, st1)


def test_cooperative_unless_asked(monkeypatch):
    """The shape knobs alone select the cooperative form (test_gpu_tile_variants.py relies on it), and SR3_PINGPONG=0 runs it everywhere."""
    from sr3_b200 import _native
    f = next(f for f in FORMS if f.name == "tall256x64")
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    tv.run_case(monkeypatch, f, 1, None, True, 3, seed=3)
    assert _native.last_test_conv_schedule()["schedule"] == "cooperative"
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("SR3_PINGPONG", "0")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(16, 128, 128, 64, generator=g).bfloat16()
    w = torch.randn(64, 64, 3, 3, generator=g) / 24.0
    _native.test_conv_ex(x.cuda(), w.cuda(), 3, 1)
    assert _native.last_test_conv_schedule()["schedule"] == "cooperative"


@pytest.mark.parametrize("H,C,want", [(128, 64, "pingpong"), (64, 128, "pingpong"), (32, 256, "cooperative")])
def test_model_choice_at_the_flagship_levels(monkeypatch, H, C, want):
    """Without knobs the byte model picks the 128x64 ping-pong tile for the 3x3 convs of the 16->128 step at 128x128 and 64x64 (B = 16)
    and keeps the cooperative tile at 32x32, as measured (DESIGN.md section 8)."""
    from sr3_b200 import _native
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    x = torch.zeros(16, H, H, C, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(C, C, 3, 3, device="cuda")
    _native.test_conv_ex(x, w, 3, 1)
    s = _native.last_test_conv_schedule()
    assert s["schedule"] == want, s
    if want == "pingpong":
        assert (s["tall"], s["mh"], s["block_n"], s["ksplit"]) == (1, 1, 64, 1), s


@pytest.mark.parametrize("B,H,C,tall", [(2, 8, 64, 0), (2, 8, 128, 0), (2, 16, 64, 1), (2, 16, 128, 1)])
def test_folded_upsample(monkeypatch, B, H, C, tall):
    pingpong_env(monkeypatch)
    tv.test_folded_upsample(monkeypatch, B, H, C, tall)
    check_pingpong()


@pytest.mark.parametrize("B,H,Cin,Cout,tall", [(2, 32, 128, 128, 1)])   # (the 8x8 form of that test stages its residual: no ping-pong tile fits)
def test_precise_mode(monkeypatch, B, H, Cin, Cout, tall):
    pingpong_env(monkeypatch)
    tv.test_precise_mode_is_fp32_accurate(monkeypatch, B, H, Cin, Cout, tall)
    check_pingpong()


@pytest.mark.parametrize("cin,cout,B,H", [(128, 64, 2, 16), (64, 128, 2, 32), (128, 64, 4, 8)])
def test_block2_with_shortcut(monkeypatch, cin, cout, B, H):
    pingpong_env(monkeypatch)
    tv.test_block2_with_shortcut(monkeypatch, cin, cout, B, H)
    check_pingpong()


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("B", [3, 9])
def test_padded_4x4_patch(monkeypatch, bn, B):
    """4x4 images in a 4x8 patch (rows 4..7 masked): four images per 128-row tile, FiLM bias / residual / statistics per image."""
    from sr3_b200 import _native
    pingpong_env(monkeypatch)
    monkeypatch.setenv("SR3_BLOCK_N", str(bn))
    monkeypatch.setenv("SR3_MAX_CTAS", "2")
    g = torch.Generator().manual_seed(bn * 31 + B)
    Cin, Cout = 128, 256
    x = torch.randn(B, 4, 4, Cin, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    bias, bias2 = torch.randn(Cout, generator=g), torch.randn(B, Cout, generator=g)
    res = torch.randn(B, 4, 4, Cout, generator=g)
    y, yb, stats, _ = _native.test_conv_ex(x.cuda(), w.cuda(), 3, 1, bias=bias.cuda(), bias2=bias2.cuda(), resid=res.cuda(),
                                           want_bf16=True, want_stats=True)
    s = check_pingpong()
    assert s["block_n"] == bn and s["tall"] == 0 and s["ctas"] == 2, s
    y = y.cpu()
    ref = tv.conv_ref(x, w, 1, bias, bias2, res)
    tv.check_close(y, ref, f"4x4 bn{bn} B{B}")
    tv.check_stats(stats, ref)
    tv.check_bf16_copy(yb, y)


# ------------------------------------------------------------------------------------------------ UNet level
@pytest.mark.timeout(900)
def test_full_config_eps_with_pingpong_forced(golden, monkeypatch):
    """16->128 config with every eligible tile op forced to ping-pong: eps and p_mean_variance still meet the golden at 1e-2, and the plan
    really runs ping-pong tiles at 128x128 and 64x64 (and the qkv projection of the 16x16 attention, whose v third is stored transposed)."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("SR3_PINGPONG", "1")
    tu.test_full_config_eps_and_pmv(golden)
    net = tu.build(tu.FULL_UNET, 128, 0)
    eng = net.denoise_fn.engine(2)
    tiles = [s for s in eng.tile_schedules() if s is not None]
    pp = {(s["out_hwc"][0], s["out_hwc"][2]) for s in tiles if s["schedule"] == "pingpong"}
    assert (128, 64) in pp and (64, 128) in pp, pp
    assert (16, 3 * 512) in pp, pp                              # qkv projection at 16x16 (C = 512)
    assert all(s["ksplit"] == 1 for s in tiles if s["schedule"] == "pingpong")


def test_default_plan_reports_every_tile_op():
    """Every tile op of an engine reports its variant; the non-tile ops report none."""
    net = tu.build(tu.TINY_UNET, 32, 0)
    eng = net.denoise_fn.engine(2)
    sch = eng.tile_schedules()
    prof = eng.profile_step(5, reps=1)
    assert len(sch) == len(prof)
    for (kind, _, _, _), s in zip(prof, sch):
        assert (kind == 0) == (s is not None), (kind, s)
        if s is not None:
            assert s["schedule"] in ("cooperative", "pingpong") and s["out_hwc"][2] > 0, s


@pytest.mark.parametrize("batch", [3, 40])
def test_per_layer_path_is_bit_reproducible(golden, batch, monkeypatch):
    """With ping-pong forced, two engines give the same bits.  Batch 40 gives the CTAs of the 32x32 convs several (odd and even) tile
    counts."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("SR3_PINGPONG", "1")
    schedules = tu.check_two_engines_agree(golden, batch)
    if batch > 3:
        assert any(s is not None and s["schedule"] == "pingpong" and s["tiles"] > 132 for s in schedules)

"""Pins the per-layer fp64 reference of tests/_layer_ref.py on the CPU, before any GPU compares against it:

- with rounded=False every layer function is the oracle's own layer (oracle/sr3_oracle.py) in fp64;
- the folded Upsample with rounding off is conv3x3 of the nearest-2x image;
- with rounding on, every layer moves by the order of bf16 rounding (bf16) or of the hi/lo pair's (precise mode), so the switch reaches
  each layer's rounding points."""
import pytest
import torch
import torch.nn.functional as F

import _layer_ref as lref
from oracle import sr3_oracle as orc

TINY = orc.UNetConfig(6, 3, 64, 32, (1, 2), (16,), 1, 0.0, 32)
TINY4 = orc.UNetConfig(6, 3, 64, 32, (1, 2, 2), (), 1, 0.0, 16)
# the geometry of sr_sr3_64_512 at three levels: 16 GroupNorm groups, no attention but the middle block's; its 192 and 384 concats have 12-
# and 24-channel groups that straddle the boundary at 128 and 256
G16 = orc.UNetConfig(6, 3, 64, 16, (1, 2, 4), (), 1, 0.0, 32)
# (config, batch, height, width): attention at 16x16 (and one- / two-source, identity / res_conv blocks), at 8x8 (the same net on 16x16
# images: its attention level is then 8x8), at 4x4 (the 4x4 middle of TINY4), over 512 tokens (16x32 attention of 32x64 images), and
# 16 groups (G16, its 8x8 middle attention with C = 256)
NETS = {"tiny_32x32": (TINY, 2, 32, 32), "tiny_16x16": (TINY, 3, 16, 16), "tiny4_16x16": (TINY4, 3, 16, 16), "tiny_32x64": (TINY, 2, 32, 64),
        "g16_32x32": (G16, 2, 32, 32)}


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def oracle_taps(name):
    """fp64 oracle forward with every layer's output, plus "<layer>.res_block" of the attention layers; its inputs and weights."""
    cfg, b, h, w = NETS[name]
    sd = {k: v.double() for k, v in lref.state_dict(cfg, 11).items()}
    g = torch.Generator().manual_seed(12)
    x = torch.randn(b, cfg.in_channel, h, w, generator=g, dtype=torch.float64)
    nl = torch.tensor([0.9, 0.2, 0.55], dtype=torch.float64)[:b]
    taps = {"input": x}
    with torch.no_grad():
        taps["eps"] = orc.unet_forward(sd, cfg, x, nl.view(-1, 1), taps)
        t = orc.noise_level_mlp(sd, nl.view(-1, 1), cfg.inner_channel)
        for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
            if tap.endswith(".res_block"):
                xin = taps[src] if skip is None else torch.cat([taps[src], taps[skip]], 1)
                taps[tap] = orc.resnet_block(sd, tap, xin, t, cfg.norm_groups)
    return cfg, sd, nl, taps


@pytest.fixture(scope="module", params=sorted(NETS))
def net(request):
    return (request.param,) + oracle_taps(request.param)


def test_unrounded_layers_are_the_oracle(net):
    name, cfg, sd, nl, taps = net
    kinds = set()
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        sk = None if skip is None else taps[skip]
        ref = lref.layer_reference(sd, cfg, kind, spec, taps[src], sk, nl, rounded=False)
        e = rel(ref, taps[tap])
        assert e < 1e-12, (name, tap, e)
        kinds.add((kind, skip is not None, kind == "res" and lref.residual(kind, spec, sd, taps[src]) is not None))
    if name == "g16_32x32":    # 16 groups; concats whose group straddles the boundary (12 channels at 128 + 64, 24 at 256 + 128)
        straddle = {(taps[src].shape[1], taps[skip].shape[1]) for tap, kind, spec, src, skip in lref.layer_inputs(cfg)
                    if skip is not None and taps[src].shape[1] % ((taps[src].shape[1] + taps[skip].shape[1]) // cfg.norm_groups)}
        assert cfg.norm_groups == 16 and straddle == {(128, 64), (256, 128)}, straddle
    if name == "tiny_32x32":   # every kind of layer; ResnetBlocks with one and two sources, identity and res_conv shortcuts
        assert kinds >= {("conv", False, False), ("res", False, True), ("res", False, False), ("res", True, False), ("attn", False, False),
                         ("down", False, False), ("up", False, False), ("final", False, False)}, kinds


def test_attention_geometry_of_the_nets():
    """The attention layers the cases above reach: C = 128 at 16x16, 8x8 and 4x4 (8, 2 images per 128-token batch on the device), over
    512 tokens, and C = 256 at 8x8 in the 16-group net's middle block."""
    sizes = {}
    for name, (cfg, _, h, w) in NETS.items():
        sizes[name] = set()
        for tap, kind, spec, _, _ in lref.layer_inputs(cfg):
            if kind == "attn":
                f = cfg.image_size // spec.res
                sizes[name].add((h // f, w // f))
    assert sizes == {"tiny_32x32": {(16, 16)}, "tiny_16x16": {(8, 8)}, "tiny4_16x16": {(4, 4)}, "tiny_32x64": {(16, 32)},
                     "g16_32x32": {(8, 8)}}, sizes


def test_folded_upsample_is_conv_of_nearest_2x():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(64, 64, 3, 3, generator=g) / 24
    sd = {"u.conv.weight": w, "u.conv.bias": torch.randn(64, generator=g)}
    for shape in ((2, 64, 8, 8), (1, 64, 4, 16)):
        x = torch.randn(*shape, generator=g, dtype=torch.float64)
        want = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w.double(), sd["u.conv.bias"].double(), padding=1)
        assert rel(lref.upsample(sd, "u", x, rounded=False), want) < 1e-12
        assert rel(lref.upsample(sd, "u", x, rounded=False, fold=False), want) < 1e-12
    # the packer's fp32 sums: exact sums of at most four fp32 weights, rounded once to fp32
    for f32, f64 in zip(lref.folded_weights(w), lref.folded_weights(w.double())):
        assert f32.dtype == torch.float32 and rel(f32.double(), f64) < 2.0 ** -23


def branch_rel(a, b, resid):
    """Relative L2 of a - b against b's branch (b less the residual the layer adds)."""
    return ((a - b).norm() / (b if resid is None else b - resid).norm()).item()


# bf16: an operand rounded to bf16 moves by up to 2^-9 relative (~1.1e-3 rms); precise mode: the pair leaves ~2^-17
BF16_MOVES = (3e-4, 1e-2)
PRECISE_MOVES = (1e-8, 1e-4)


def test_rounding_moves_every_layer(net):
    name, cfg, sd, nl, taps = net
    moves = {}
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        x, sk = taps[src], None if skip is None else taps[skip]
        resid = lref.residual(kind, spec, sd, x)
        plain = lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, rounded=False)
        m = {"bf16": branch_rel(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, "bf16"), plain, resid),
             "fp32": branch_rel(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, "fp32"), plain, resid)}
        if kind == "attn":
            m["unfused"] = branch_rel(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, unfused=True), plain, resid)
        if kind == "res":
            keep = (torch.rand(plain.shape, generator=torch.Generator().manual_seed(5)) >= 0.2).double() / 0.8
            drop = lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, rounded=False, keep_scale=keep)
            m["dropout"] = branch_rel(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, keep_scale=keep), drop, resid)
        moves[tap] = m
    print(name, {t: {k: f"{v:.1e}" for k, v in m.items()} for t, m in moves.items()})
    for tap, m in moves.items():
        for k, v in m.items():
            lo, hi = PRECISE_MOVES if k == "fp32" else BF16_MOVES
            assert lo < v < hi, (name, tap, k, v)


def test_groupnorm_of_the_next_image_moves_every_groupnorm_layer(net):
    """gn_stats (image b normalised with the statistics of another image) moves every layer with a GroupNorm by more than 5 times its
    bf16 rounding (measured 9x to 108x), and with the identity it is the default reference bit for bit."""
    name, cfg, sd, nl, taps = net
    b = nl.shape[0]
    moves = {}
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        if kind not in ("res", "attn", "final"):
            continue
        x, sk = taps[src], None if skip is None else taps[skip]
        resid = lref.residual(kind, spec, sd, x)
        ref = lref.layer_reference(sd, cfg, kind, spec, x, sk, nl)
        assert torch.equal(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, gn_stats=list(range(b))), ref), (name, tap)
        rounding = branch_rel(ref, lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, rounded=False), resid)
        moves[tap] = branch_rel(lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, gn_stats=lref.neighbour(b)), ref, resid) / rounding
    print(name, "moves in units of the layer's bf16 rounding:", {t: f"{v:.0f}" for t, v in moves.items()})
    assert all(v > 5 for v in moves.values()), (name, moves)


def test_noise_levels():
    """noise_levels(b): the levels of the batch-2 and -3 cases unchanged; b distinct levels in [0.05, 0.95] past that, neighbours more than
    0.45 apart."""
    import test_gpu_layers as tgl
    for b in (1, 2, 3):
        assert torch.equal(tgl.noise_levels(b), torch.tensor(tgl.NOISE_LEVELS[:b]))
    for b in (4, 5, 8, 16, 32):
        nl = tgl.noise_levels(b)
        assert nl.dtype == torch.float32 and nl.shape == (b,) and len(set(nl.tolist())) == b
        assert 0.05 - 1e-7 <= nl.min() and nl.max() <= 0.95 + 1e-7
        assert (nl[1:] - nl[:-1]).abs().min() > 0.45, nl

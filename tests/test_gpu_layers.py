"""Every layer of the native UNet forward against the fp64 layer reference of tests/_layer_ref.py, fed the engine's own activations.

For each case the engine runs one forward (unet_forward, or train_unet_forward for the training plan) and every layer's output is read
back (read_activation; "<layer>.res_block" for the ResnetBlock under an attention layer).  Each layer's reference is computed from the
device's taps of that layer's inputs -- the previous tap, the skip popped in the plan's order, the UNet input -- so it carries none of the
error of the layers above it, and rounds to bf16 exactly where the plan does.  What is left between the two:

- fp32 accumulation: ~sqrt(K) 2^-24 of the sum of |terms|, which the kernel tests hold to 2e-5 relative L2;
- the device's __expf / __fdividef SiLU and its fp32 GroupNorm scale / shift (a few 2^-24);
- rounding flips: an fp32 value and its fp64 counterpart on either side of a bf16 boundary.  A flipped operand moves by one bf16 ulp
  (2^-8 relative), which a conv output sees diluted over its K terms; in attention a flipped P~ of a key holding much of a row's weight
  moves that row by up to 2^-8 p |v| (the fused-attention kernel tests measure 3.8e-5 to 1.1e-4 relative L2 from them).

Errors are measured on the layer's branch: ||got - ref|| / ||ref - r||, where r is the residual the layer adds unrounded (x of an
identity-shortcut ResnetBlock, the ResnetBlock output of an attention layer), else 0.  A residual can outweigh its branch many times
over; relative to the branch, one bf16 rounding of a layer's operands is 2.1e-3 to 3.5e-3 (the rounded reference against the unrounded
one, tests/test_layer_ref.py).  The element-wise bound is elem (|b| + rms(b)) on the branch b.  Bounds by class of layer:

- direct (first conv, Downsample, Upsample): their bf16 operands are roundings of fp32 taps, which the reference reproduces bit for bit.
  Only the fp32 accumulation is left: the kernel tests' 2e-5 relative L2 and 1e-4 element-wise.
- chained (ResnetBlock, attention, final block): their bf16 operands are roundings of intermediates (silu(GN(.)), h, q / k / v, P~) that
  the device forms in fp32 with __expf and the reference in fp64.  About 2^-16 of them flip; a flipped a1 or n moves h or q / k / v by
  ~1e-4 relative, which then flips a few per cent of a2 or P~, each by one bf16 ulp.  The model puts this at the order of 2e-4 relative
  L2, with a heavy element-wise tail (a few flips of one output's K terms that share a sign).  Bounds 4e-4 and 1e-2.
- precise mode, both classes: the hi/lo pair holds an operand to ~2^-17 whichever way hi rounds, so flips do not propagate: the pair's
  2^-17 and the fp32 accumulation are left.  Bounds 1.5e-5 and 1e-4 up to a contraction length k = 2304 (contraction()), k / 2304 times
  that past it.  The tensor cores' fp32 accumulation error grows in proportion to k, not as sqrt(k): on the 64->512 net every precise layer
  measures 5.0e-9 k to 5.4e-9 k relative L2 (Downsample k = 576 .. 4608, ResnetBlocks up to 9216, Upsample 4096), the bf16 direct layers
  1.0e-9 k (one pass instead of three).  So at k = 18432 (the 2048-channel concat of ups.0) the accumulation alone is 5.9e-5, above the
  1.5e-5 that k <= 2304 reaches; the bound 1.5e-5 k / 2304 = 6.5e-9 k keeps every case with k <= 2304 at 1.5e-5.

Measured maxima over the cases below (NVIDIA H100 80GB HBM3, 700 W power limit), relative L2 / element-wise:
  bf16 direct     first conv 6.7e-8 / 3.4e-7, Downsample 4.7e-6 / 1.2e-5, Upsample 2.0e-6 / 5.2e-6
  bf16 chained    ResnetBlock 1.7e-4 / 4.0e-3, attention 2.7e-4 / 4.5e-3 (the 16x16 C = 512 layers of full_128x128), final 5.3e-5 / 1.4e-3
  precise         ResnetBlock 7.8e-6 / 1.7e-5, attention 4.3e-6 / 1.6e-5, convs <= 5.2e-6 / 6.9e-6
and on the sr_sr3_64_512 net (16 groups; two runs, identical to the printed digits; 1.1 to 2.2 s per case):
  bf16 direct     first conv 6.7e-8 / 4.0e-7, Downsample 4.8e-6 / 1.5e-5, Upsample 4.3e-6 / 1.2e-5 (the 1024-channel ups.2)
  bf16 chained    ResnetBlock 3.1e-4 (the 4x4 middle at 1024 channels) / 9.2e-3 (downs.1 at 512x512: the tail's largest element
                  grows with the 2^25 outputs), final 1.9e-5 / 1.7e-3; attention 3.8e-4 / 5.1e-3, the C = 1024 middle at 8x8 (two images
                  per 128-token batch): the flips' effect grows with the logits' scale, ~sqrt(C), from the 2.7e-4 of C = 512.  The
                  1024-token C = 1024 attention at 512x512 measures 2.2e-4.
  precise         5.9e-5 / 1.1e-4 (ups.0, k = 18432, bound 1.2e-4); at most 0.84 of the scaled bound on every layer (mid.1, k = 9216)
Precise mode runs the same plan wiring (only its attention core is the unfused one) and agrees to 8e-6 (on the 64->512 net, to its
accumulation error above): the bf16 excess of the chained layers is rounding, not wiring.

Each bound is shown to discriminate, the way check_fused does: the unrounded reference misses every bf16 layer by at least 5x its bound
(measured 2.1e-3 to 3.5e-3); in precise mode the bf16 reference misses by at least 100x the unscaled bound 1.5e-5 (2.2e-3 to 3.4e-3:
one bf16 rounding does not grow with k).  Two wrong references of the
wiring miss by at least 10x: the Upsample with per-tap rounded weights, where the plan rounds the fp32 sums of the aliased taps once
(2.1e-3 to 2.3e-3, 100x the Upsample's bound and under the 1e-2 of the UNet-level tests, which cannot see it), and the FiLM rows of
images 0 and 1 swapped in the first ResnetBlock (2.1e-2 to 3.0e-2)."""
import time

import pytest
import torch

import _layer_ref as lref
import _philox
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

# (precision, layer class) -> (relative L2 bound, element-wise bound factor); see the module docstring
BOUNDS = {("bf16", "direct"): (2e-5, 1e-4), ("bf16", "chained"): (4e-4, 1e-2),
          ("fp32", "direct"): (1.5e-5, 1e-4), ("fp32", "chained"): (1.5e-5, 1e-4)}
DIRECT = ("conv", "down", "up")   # bf16 operands are roundings of fp32 taps: reproduced bit for bit
MISS_UNROUNDED = 5.0          # the unrounded reference misses a bf16 layer by at least this many bounds
MISS_BF16 = 100.0             # the bf16 reference misses a precise-mode layer by at least this many bounds
MISS_WRONG = 10.0             # each wrong reference, likewise
PRECISE_K0 = 2304             # precise mode: the bounds hold up to this contraction length and grow in proportion past it

SCHED = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
TINY = dict(in_channel=6, channel_mults=(1, 2), attn_res=(16,), res_blocks=1)             # tests/_sizes_inputs.TINY
TINY4 = dict(in_channel=6, channel_mults=(1, 2, 2), attn_res=(), res_blocks=1)            # tests/_lowres_inputs.TINY4
FULL = dict(in_channel=6, channel_mults=(1, 2, 4, 8, 8), attn_res=(16,), res_blocks=2)    # sr_sr3_16_128, the benchmark's UNet
SR64_512 = dict(in_channel=6, channel_mults=(1, 2, 4, 8, 16), attn_res=(), res_blocks=1, norm_groups=16)    # sr_sr3_64_512
# name -> (net, image_size, batch, height, width, precision, training-plan dropout or None)
CASES = {
    # fused 256-token attention with C = 128, an odd batch, identity and res_conv shortcuts
    "tiny_b3": (TINY, 32, 3, 32, 32, "bf16", None),
    "tiny_b3_precise": (TINY, 32, 3, 32, 32, "fp32", None),
    # 512-token streaming attention (attn_long_kernel), non-square layers
    "tiny_32x64": (TINY, 32, 2, 32, 64, "bf16", None),
    # 4x4 middle: 16-token attention, eight images per attention batch, the allocation padded to 8 images
    "tiny4_b3": (TINY4, 16, 3, 16, 16, "bf16", None),
    "tiny4_b3_precise": (TINY4, 16, 3, 16, 16, "fp32", None),
    # five levels, concats up to 1024 channels, C = 512 attention at 16x16, the 8x8 middle attention with two images per batch
    "full_128x128": (FULL, 128, 2, 128, 128, "bf16", None),
    # unconditional: the first conv reads 3 of its 64 input channels
    "tiny_uncond": (dict(TINY, in_channel=3), 32, 2, 32, 32, "bf16", None),
    # the training plan's forward: unfused attention, Dropout in every block2 (prep_kernel<true>) with injected masks
    "tiny_train_dropout": (TINY, 32, 2, 32, 32, "bf16", 0.2),
    # sr_sr3_64_512 as it ships: 16 groups of 4 to 128 channels, 2048- and 1536-channel concats (the 96-channel groups straddle channel
    # 1024), the C = 1024 middle attention over 1024 tokens (attn_long_kernel), a 512x512 first level
    "sr64_512_512x512": (SR64_512, 512, 2, 512, 512, "bf16", None),
    "sr64_512_512x512_precise": (SR64_512, 512, 2, 512, 512, "fp32", None),
    # 8x8 middle: two images per 128-token attention batch at C = 1024
    "sr64_512_128x128_b3": (SR64_512, 512, 3, 128, 128, "bf16", None),
    # 4x4 lowest level at 1024 channels: eight images per 16-token attention batch, the allocation padded to 8 images
    "sr64_512_64x64_b3": (SR64_512, 512, 3, 64, 64, "bf16", None),
    # the training plan's forward at 16 groups: unfused C = 1024 attention, Dropout in every block2 with injected masks
    "sr64_512_train_128x128": (SR64_512, 512, 2, 128, 128, "bf16", 0.2),
}
NOISE_LEVELS = (0.9, 0.2, 0.55)      # a different noise level per image: a FiLM row read from the wrong image shows


def noise_levels(b):
    """The noise levels of a batch of b, fp32: NOISE_LEVELS for b <= 3; past that b distinct levels in [0.05, 0.95] that alternate between
    the two ends, 0.05 + k d and 0.95 - k d for images 2 k and 2 k + 1 (d = 0.45 / b): images i and i + 1 (which the wrong FiLM references
    swap) are 0.9 - i d apart, more than 0.45."""
    if b <= len(NOISE_LEVELS):
        return torch.tensor(NOISE_LEVELS[:b])
    d = 0.45 / b
    return torch.tensor([0.05 + i // 2 * d if i % 2 == 0 else 0.95 - i // 2 * d for i in range(b)], dtype=torch.float32)


def case_seed(cases, name):
    """The seed of a case's inputs: its place in sorted order, the sr64_512 cases after the others (so adding them kept every other
    case's inputs)."""
    return sorted(cases, key=lambda n: (n.startswith("sr64_512"), n)).index(name)


def oracle_cfg(net, image_size):
    return orc.UNetConfig(net["in_channel"], 3, 64, net.get("norm_groups", 32), net["channel_mults"], net["attn_res"], net["res_blocks"], 0.0,
                          image_size)


def engine_cfg(cfg, image_size, precision):
    """The engine config of an oracle config (inner_channel 64, 3 output channels; conditional when the input has more than 3)."""
    return dict(in_channel=cfg.in_channel, out_channel=3, inner_channel=64, norm_groups=cfg.norm_groups, channel_mults=tuple(cfg.channel_mults),
                attn_res=list(cfg.attn_res), res_blocks=cfg.res_blocks, image_size=image_size, channels=3, conditional=cfg.in_channel != 3,
                precision=precision)


def make_engine(case):
    """The engine of a case tuple (CASES' form) with the weights lref.state_dict(cfg, 5) and the schedule SCHED.  -> (cfg, sd, engine)."""
    from sr3_b200 import _native
    net, image_size, b, h, w, precision, drop = case
    cfg = oracle_cfg(net, image_size)
    sd = lref.state_dict(cfg, 5)
    eng = _native.Engine(engine_cfg(cfg, image_size, precision), b, torch.device("cuda", torch.cuda.current_device()), train_dropout=drop,
                         height=h, width=w)
    sch = orc.make_schedule(SCHED)
    eng.set_schedule(sch.buffers, sch.sqrt_alphas_cumprod_prev)
    eng.load_state_dict(sd)
    return cfg, sd, eng


def run_engine(case, seed, tap_dtype=torch.float64):
    """One forward of a case tuple, inputs drawn from `seed`.  -> (cfg, state dict on the GPU, noise levels, {tap: NCHW in tap_dtype}
    incl. "input" and "eps", {dropout block: scaled keep-mask}, the engine's tile_schedules())."""
    net, image_size, b, h, w, precision, drop = case
    cfg, sd, eng = make_engine(case)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cfg.in_channel, h, w, generator=g)
    nl = noise_levels(b)
    masks = {}
    if drop is None:
        eps = eng.unet_forward(x.cuda(), nl.cuda())
    else:
        shapes = {}
        for _, kind, spec, _, _ in lref.layer_inputs(cfg):
            if kind == "res":
                f = image_size // spec.res
                shapes[spec.name + ".res_block.block2"] = (b, spec.cout, h // f, w // f)
        assert sorted(eng.dropout_layers()) == sorted(shapes)
        for k, shape in shapes.items():
            keep = (torch.rand(shape, generator=g) >= drop).to(torch.uint8)
            eng.set_dropout_mask(k, keep.cuda().contiguous())
            masks[k] = _philox.scale_mask(keep, drop)
        eps, _ = eng.train_unet_forward(x.cuda(), nl.cuda())
    taps = {"input": x.cuda().to(tap_dtype), "eps": eps.to(tap_dtype)}
    for tap, _, _, _, _ in lref.layer_inputs(cfg):
        if tap != "eps":
            taps[tap] = eng.read_activation(tap).to(tap_dtype)
    plan = eng.tile_schedules()
    torch.cuda.synchronize()
    del eng
    return cfg, {k: v.cuda() for k, v in sd.items()}, nl.cuda(), taps, masks, plan


def contraction(kind, cin, cout, tokens):
    """A layer's contraction length k: that of its longest GEMM (9 Cin of a 3x3 conv over its (concatenated) input, 9 Cout of a
    ResnetBlock's second conv, 4 C of a folded Upsample phase); for attention, whose four GEMMs are of like length and chained, their sum
    (the q | k | v and output projections and q k^T over C, P v over the tokens)."""
    cin = max(cin, 64)       # the first conv's input is padded to 64 channels
    return {"up": 4 * cin, "res": 9 * max(cin, cout), "attn": 3 * cin + tokens}.get(kind, 9 * cin)


def bounds(precision, cls, k):
    """(relative L2, element-wise factor) of a layer with the longest contraction k: the class bounds, and in precise mode the class
    bounds scaled by k / PRECISE_K0 past PRECISE_K0 (see the module docstring)."""
    bound, elem = BOUNDS[precision, cls]
    f = max(1.0, k / PRECISE_K0) if precision == "fp32" else 1.0
    return bound * f, elem * f


def branch_rel(got, ref, resid):
    return ((got - ref).norm() / (ref if resid is None else ref - resid).norm().clamp_min(1e-300)).item()


def elementwise(got, ref, resid, elem):
    """(largest |got - ref| / (|b| + rms(b)) over the branch b, None or a message on the elements past elem (|b| + rms(b)), the first as
    (image, channel, row, column))."""
    b = ref if resid is None else ref - resid
    scale = b.abs() + b.pow(2).mean().sqrt()
    ratio = (got - ref).abs() / scale
    bad = (ratio > elem).nonzero()
    if not bad.numel():
        return ratio.max().item(), None
    i = tuple(bad[0].tolist())
    return ratio.max().item(), (f"{bad.shape[0]} elements past {elem:.0e} (|b| + rms(b)), first at (image {i[0]}, channel {i[1]}, row {i[2]}, "
                                f"column {i[3]}): got {got[i].item():.7g}, want {ref[i].item():.7g} (bound {elem * scale[i].item():.2e})")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_every_layer_matches_its_fp64_reference(name):
    t0 = time.time()
    net, image_size, b, h, w, precision, drop = CASES[name]
    cfg, sd, nl, taps, masks, _ = run_engine(CASES[name], case_seed(CASES, name))
    unfused = drop is not None
    failures, rows, worst = [], [], {}
    first_res = None
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        x, sk = taps[src], None if skip is None else taps[skip]
        keep = masks.get(spec.name + ".res_block.block2") if kind == "res" else None
        resid = lref.residual(kind, spec, sd, x)
        got = taps[tap]
        assert torch.isfinite(got).all(), tap
        cls = "direct" if kind in DIRECT else "chained"
        k = contraction(kind, x.shape[1] + (0 if sk is None else sk.shape[1]), got.shape[1], x.shape[2] * x.shape[3])
        bound, elem = bounds(precision, cls, k)

        def ref_of(**kw):
            return lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, **dict(dict(precision=precision, unfused=unfused, keep_scale=keep), **kw))
        ref = ref_of()
        e = branch_rel(got, ref, resid)
        r, bad = elementwise(got, ref, resid, elem)
        worst[cls] = max(worst.get(cls, (0.0, 0.0)), (e, r))
        row = f"{tap:>20} {kind:>5}  K {k:>5}  rel L2 {e:.2e} (bound {bound:.1e})  element-wise {r:.2e} (bound {elem:.1e})"
        if e >= bound:
            failures.append(f"{tap}: relative L2 {e:.3e} >= {bound:.1e}")
        if bad:
            failures.append(f"{tap}: {bad}")
        if precision == "bf16":
            miss = branch_rel(got, ref_of(rounded=False), resid)
            row += f"  unrounded {miss:.2e}"
            if miss < MISS_UNROUNDED * bound:
                failures.append(f"{tap}: the unrounded reference misses by only {miss:.2e} (< {MISS_UNROUNDED:g} x {bound:.1e})")
        else:
            # against the unscaled class bound: one bf16 rounding does not grow with k as the accumulation does
            base = BOUNDS[precision, cls][0]
            miss = branch_rel(got, ref_of(precision="bf16"), resid)
            row += f"  bf16 reference {miss:.2e}"
            if miss < MISS_BF16 * base:
                failures.append(f"{tap}: the bf16 reference misses by only {miss:.2e} (< {MISS_BF16:g} x {base:.1e})")
        if kind == "up" and precision == "bf16":
            # below the 1e-2 of the UNet-level tests, far above this bound
            wrong = branch_rel(got, lref.upsample(sd, spec.name, x, precision, fold=False), resid)
            row += f"  per-tap rounded weights {wrong:.2e}"
            if not MISS_WRONG * bound <= wrong < 1e-2:
                failures.append(f"{tap}: the per-tap rounded Upsample misses by {wrong:.2e}")
        if kind == "res" and first_res is None:
            first_res = tap
            film = lref.film_rows(sd, spec.name + ".res_block", nl, cfg.inner_channel)
            wrong = branch_rel(got, ref_of(film=film[[1, 0] + list(range(2, b))]), resid)
            row += f"  FiLM rows 0, 1 swapped {wrong:.2e}"
            if wrong < MISS_WRONG * bound:
                failures.append(f"{tap}: the swapped-FiLM reference misses by only {wrong:.2e}")
        rows.append(row)
    print(f"\n{name} ({precision}{', training plan' if unfused else ''}, batch {b}, {h}x{w}): worst (rel L2, element-wise) "
          + ", ".join(f"{k} {v[0]:.2e} {v[1]:.2e}" for k, v in sorted(worst.items())) + f"; {time.time() - t0:.1f} s\n" + "\n".join(rows))
    if failures:
        pytest.fail(f"{name}: " + "; ".join(failures))

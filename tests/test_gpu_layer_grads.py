"""Every layer of the native training backward against the fp64 backward reference of tests/_layer_grad_ref.py, fed the engine's own
activations and the engine's own gradient of each layer's output; and the promise of sr3_train_block_params on one GPU.

For each case the engine runs one train_unet_forward (with injected Dropout keep-masks where the case has Dropout) and one
train_unet_backward from a random fp32 upstream gradient, then every tensor's g, gb and gsum (read_gradient), every parameter gradient, dx
and film_state()["dfilm"] are read.  Reading them after the whole backward is valid: the contract in train_plan.inc makes a tensor's g
complete before its producer's backward runs, and nothing writes it afterwards.  Each layer's reference is computed from the engine's taps
of its inputs and the engine's g of its output, so it carries none of the error of the layers above it.  A tensor that is also a skip
source is checked against the sum of its two consumers' references (the accumulate contract).

Exact identities on every tap: gb == bf16(g) bit for bit (the last writer produced the bf16 copy), and gsum equals the pixel sums of g to
within 1e-5 of the sums of |g|.

Compared against the reference: each tensor's gradient (on the branch: less the y.g that identity shortcuts and the attention residual pass
through exactly), every parameter gradient the layers' backward blocks write, dfilm per ResnetBlock, and dx.  The FiLM projection, block1
bias and noise-level MLP gradients are identities of dfilm, tested in tests/test_gpu_noise_level_grad.py.

Error model, relative L2 over a gradient (on the branch) and element-wise as elem (|b| + rms(b)):
- direct: data and weight gradients whose bf16 operands the reference reproduces bit for bit (first conv, Downsample, Upsample: y.gb and
  a bf16 tap or packed weight; res_conv's weight gradient; bias sums of y.g).  Only fp32 accumulation is left, which the kernel tests hold
  to 2e-5 and 1e-4.  The tensor cores' fp32 accumulation error grows in proportion to the contraction length k, not as sqrt(k): measured
  1.1e-9 k relative L2 on the 64->512 net, for the Upsample data gradient (k = 16 C) and for weight gradients alike.  A weight gradient's
  k is the pixels one wgrad_kernel CTA contracts in sequence (wgrad_length): its slices split the pixels so that the output tiles fill one
  wave of CTAs, so a 512-channel Upsample at 128x128 contracts all 32768 pixels of a batch of 2 in one slice.  The direct bounds hold up to
  k = 8192 (every k of the 16->128 net and the two-level nets) and grow as k / 8192 past it: 2.4e-9 k, twice the measured slope.
  The final block's input and GroupNorm gradients are direct too: its data gradient reads bf16(deps) and packed weights, and its GroupNorm
  backward the fp32 tap itself.
- chained: everything through a GroupNorm backward whose dA comes from ghb, and the weight gradients whose operands (a1, a2, n, O, P) are
  recomputed from fp32 taps.  Their bf16 operands are roundings of values the device forms in fp32 and the reference in fp64; the rare
  ones that round the other way move by one bf16 ulp and change what is computed from them.  The forward's chained layers measured 1.7e-4
  to 2.7e-4 (tests/test_gpu_layers.py); ghb is one such rounding deep.
- attention input: the gradient of an attention layer's input passes through dO, dS and d(qkv), three such roundings, before its
  GroupNorm backward; it is the largest.
The backward is not bit-reproducible (fp32 atomics in the GroupNorm and bias sums), which moves each value by a few fp32 ulps only: far
under every bound.

Measured maxima over two runs of every case (NVIDIA H100 80GB HBM3, 700 W power limit), relative L2 / element-wise, against the bounds:
  direct            8.9e-6 / 2.0e-5    bounds 2e-5 / 1e-4
  chained           3.1e-4 / 1.7e-2    bounds 5e-4 / 4e-2
  attention input   6.6e-4 / 9.7e-3    bounds 1.2e-3 / 4e-2   (the C = 512 layers at 16x16 of full_128x128)
The smallest misses measured, in bounds: the unrounded reference 7x; the wrong references: GroupNorm per source 20x, per-tap Upsample
weights 106x, the joint softmax 682x, no keep-mask 926x, the skip omitted 1077x, another block's keep-mask 1176x, the skip one channel
late 1339x, dfilm of images 0 and 1 swapped 2089x.

On the sr_sr3_64_512 net (16 groups), over two runs: direct 3.7e-5 / 1.6e-4 (ups.5's weight gradient, k = 32768, bound 8e-5 / 4e-4),
chained 3.7e-4 / 1.6e-2, attention input 1.0e-3 / 1.3e-2 (the C = 1024 middle over 1024 tokens at 512x512).  Misses: the unrounded
reference 7x, GroupNorm per source 22x (the 96-channel groups of the 1536 concat, and 768, 384, 192), per-tap Upsample weights 57x (in
the scaled bound), the joint softmax 594x, no keep-mask 1081x, the skip omitted 1129x, another block's keep-mask 1310x, the skip one
channel late 1396x, dfilm swapped 1947x.  Wall time per case 1.8 to 6.5 s; the training engine's workspace_bytes() is 8.96 GiB at
512x512, batch 2 (2.51 GiB at 128x128, batch 3).

Each bound is shown to discriminate.  The unrounded reference misses every layer by at least 5x its bound.  Each wrong reference of the
wiring misses its layer by at least 10x: the Dropout keep-mask left out, or another block's mask of the same shape; the skip half of the
concat gradient omitted, or taken one channel late; GroupNorm statistics of the group that straddles the concat taken per source; the
softmax over the whole 128-token attention batch instead of per image (8x8 and 4x4 attention); the Upsample data gradient with per-tap
rounded weights; dfilm with images 0 and 1 swapped."""
import time

import pytest
import torch
import torch.nn.functional as F

import _layer_grad_ref as gref
import _layer_ref as lref
import _philox
import test_gpu_layers as tgl
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

# class -> (relative L2 bound, element-wise bound factor); see the module docstring
BOUNDS = {"direct": (2e-5, 1e-4), "chained": (5e-4, 4e-2), "attention input": (1.2e-3, 4e-2)}
MISS_UNROUNDED = 5.0
MISS_WRONG = 10.0
DIRECT_K0 = 8192      # the direct bounds hold up to this contraction length and grow in proportion past it

# name -> (net, image_size, batch, height, width, Dropout p of the injected masks or None)
CASES = {
    # odd batch; the 192-channel concat whose GroupNorm group straddles x and skip; 256-token attention with C = 128; Dropout masks
    "tiny_b3_drop": (tgl.TINY, 32, 3, 32, 32, 0.2),
    # 8x8 attention: two images per 128-token batch
    "tiny_16x16": (tgl.TINY, 32, 2, 16, 16, None),
    # 512-token attention, non-square layers
    "tiny_32x64": (tgl.TINY, 32, 2, 32, 64, None),
    # 4x4 middle: eight images per 16-token attention batch, the batch padded; the 4x4 weight-gradient patch
    "tiny4_b3": (tgl.TINY4, 16, 3, 16, 16, None),
    # unconditional: the first conv and dx over 3 of its 64 input channels
    "tiny_uncond": (dict(tgl.TINY, in_channel=3), 32, 2, 32, 32, None),
    # the benchmark's 16->128 UNet: concats up to 1024 channels, C = 512 attention at 16x16, the 8x8 middle; Dropout masks
    "full_128x128": (tgl.FULL, 128, 2, 128, 128, 0.2),
    # sr_sr3_64_512 as it trains (batch 2, no Dropout): 16 groups, the 2048 / 1536 concats, the C = 1024 attention backward over 1024
    # tokens, weight gradients over 2^19 pixels at the 512x512 level
    "sr64_512_512x512": (tgl.SR64_512, 512, 2, 512, 512, None),
    # its 8x8 middle (two images per 128-token batch at C = 1024), odd batch, Dropout masks at 16 groups
    "sr64_512_128x128_b3_drop": (tgl.SR64_512, 512, 3, 128, 128, 0.2),
    # its 4x4 lowest level at 1024 channels: eight images per 16-token batch, the batch padded
    "sr64_512_64x64_b3": (tgl.SR64_512, 512, 3, 64, 64, None),
}
DIRECT = ("conv", "down", "up")
DIRECT_PARAMS = (".block2.block.3.bias", ".res_conv.bias", ".res_conv.weight", ".out.bias", "final_conv.block.3.bias", "final_conv.block.0.weight",
                 "final_conv.block.0.bias")
RANK = {"direct": 0, "chained": 1, "attention input": 2}


def input_class(kind):
    """The class of a layer's input gradient: the final block's data gradient reads bf16(deps) and packed weights and its GroupNorm
    backward the fp32 tap itself; attention's passes through dO, dS and d(qkv) before its GroupNorm backward."""
    return "direct" if kind in DIRECT or kind == "final" else "attention input" if kind == "attn" else "chained"


def wgrad_length(cout, cin, taps, b, oh, ow):
    """Pixels one wgrad_kernel CTA accumulates in sequence: the b oh ow pixels (8x8 patches) split into as many slices as make the
    (cout / 128) (cin / 64) (taps / 3) output tiles one wave of CTAs (engine.cu, wgrad_shape)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    nxy = -(-cout // 128) * (max(cin, 64) // 64) * -(-taps // 3)
    patches = b * (max(oh, 8) // 8) * (max(ow, 8) // 8)
    slices = max(1, min((sms + nxy // 2) // nxy, patches // 2))
    return b * oh * ow // slices


def param_length(kind, name, x, sk, cout):
    """The contraction length of a direct weight gradient (0 for the bias and GroupNorm sums, which are not GEMMs)."""
    b, c, h, w = x.shape
    cin = c + (0 if sk is None else sk.shape[1])
    if name.endswith(".res_conv.weight"):
        return wgrad_length(cout, cin, 1, b, h, w)
    if not name.endswith(".weight") or kind not in DIRECT:
        return 0
    oh, ow = {"conv": (h, w), "down": (h // 2, w // 2), "up": (2 * h, 2 * w)}[kind]
    return wgrad_length(cout, cin, 9, b, oh, ow)


def bound_of(cls, k):
    """(relative L2, element-wise factor) of a quantity of class cls whose longest contraction is k: a direct bound grows as k / DIRECT_K0
    past DIRECT_K0 (see the module docstring)."""
    bound, elem = BOUNDS[cls]
    f = max(1.0, k / DIRECT_K0) if cls == "direct" else 1.0
    return bound * f, elem * f


def make_engine(case):
    """A bf16 training engine of a case tuple (CASES' form) with its weights (lref.state_dict) and, for a case with Dropout, injected
    keep-masks.  -> (cfg, sd, engine, {ResnetBlock tap: scaled keep-mask, fp64 on the GPU})."""
    from sr3_b200 import _native
    net, image_size, b, h, w, drop = case
    cfg = tgl.oracle_cfg(net, image_size)
    sd = lref.state_dict(cfg, 5)
    eng = _native.Engine(tgl.engine_cfg(cfg, image_size, "bf16"), b, torch.device("cuda", torch.cuda.current_device()),
                         train_dropout=drop or 0.0, height=h, width=w)
    sch = orc.make_schedule(tgl.SCHED)
    eng.set_schedule(sch.buffers, sch.sqrt_alphas_cumprod_prev)
    eng.load_state_dict(sd)
    keeps = {}
    if drop:
        g = torch.Generator().manual_seed(17)
        for tap, kind, spec, _, _ in lref.layer_inputs(cfg):
            if kind == "res":
                f = image_size // spec.res
                keep = (torch.rand((b, spec.cout, h // f, w // f), generator=g) >= drop).to(torch.uint8)
                eng.set_dropout_mask(spec.name + ".res_block.block2", keep.cuda().contiguous())
                keeps[tap] = _philox.scale_mask(keep, drop).cuda().double()
    return cfg, sd, eng, keeps


def run_backward(case, seed):
    """One forward and one backward of a case tuple, inputs drawn from `seed`: everything the engine leaves, in fp64 on the GPU, and its
    tile_schedules() (the forward's tile plan)."""
    net, image_size, b, h, w, drop = case
    cfg, sd, eng, keeps = make_engine(case)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cfg.in_channel, h, w, generator=g)
    nl = tgl.noise_levels(b)
    workspace = eng.workspace_bytes()
    eps, _ = eng.train_unet_forward(x.cuda(), nl.cuda())
    taps = {"input": x.cuda().double()}
    for tap, _, _, _, _ in lref.layer_inputs(cfg):
        if tap != "eps":
            taps[tap] = eng.read_activation(tap).double()
    deps = torch.randn(eps.shape, generator=g)
    table = eng.param_table()
    grads = [torch.full(shape, float("nan"), device="cuda") for _, shape in table]
    dx, _ = eng.train_unet_backward(deps.cuda(), grads, want_dx=True)
    torch.cuda.synchronize()
    gt = {tap: {f: eng.read_gradient(tap, f).double() for f in ("g", "gb", "gsum")} for tap in taps if tap != "input"}
    out = dict(cfg=cfg, sd={k: v.cuda() for k, v in sd.items()}, nl=nl.cuda(), keeps=keeps, taps=taps, eps=eps.double(), gt=gt,
               deps=deps.cuda().double(),
               dx=dx.double(), dfilm=eng.film_state()["dfilm"][:b].double(), pgrads={n: t.double() for (n, _), t in zip(table, grads)},
               workspace=workspace, plan=eng.tile_schedules())
    del eng
    return out


def rel(got, ref, resid=None):
    b = ref if resid is None else ref - resid
    return ((got - ref).norm() / b.norm().clamp_min(1e-300)).item()


def elementwise(got, ref, resid, elem):
    """(largest |got - ref| / (|b| + rms(b)) on the branch b, None or a message locating the first element past elem)."""
    b = ref if resid is None else ref - resid
    scale = b.abs() + b.pow(2).mean().sqrt()
    ratio = (got - ref).abs() / scale
    bad = (ratio > elem).nonzero()
    if not bad.numel():
        return ratio.max().item(), None
    i = tuple(bad[0].tolist())
    return ratio.max().item(), (f"{bad.shape[0]} elements past {elem:.0e} (|b| + rms(b)), first at index {i}: got {got[i].item():.7g}, "
                                f"want {ref[i].item():.7g} (bound {elem * scale[i].item():.2e})")


def identity_failures(gt):
    """The exact identities of every tap's gradient {tap: {"g", "gb", "gsum"}}: gb == bf16(g) bit for bit, and gsum the pixel sums of g to
    within 1e-5 of the sums of |g|.  -> the failures."""
    failures = []
    for tap, v in gt.items():
        gg = v["g"]
        assert torch.isfinite(gg).all(), tap
        if not torch.equal(v["gb"], gg.float().to(torch.bfloat16).double()):
            failures.append(f"{tap}: gb is not bf16(g) at {int((v['gb'] != gg.float().to(torch.bfloat16).double()).sum())} elements")
        err = (v["gsum"] - gg.sum((2, 3))).abs() - 1e-5 * gg.abs().sum((2, 3))
        if (err > 0).any():
            failures.append(f"{tap}: gsum is not the pixel sums of g (first bad (image, channel) {tuple((err > 0).nonzero()[0].tolist())})")
    return failures


def param_class(kind, name):
    return "direct" if kind in DIRECT or name.endswith(DIRECT_PARAMS) else "chained"


def layer_checks(r):
    """The reference of every layer, and for each layer a function from one of its results (the reference or a variant) to its checked
    quantities {label: (got, want, residual, class)}; the gradient of an input tensor is the sum over its consumers, this layer's
    contribution replaced by the variant's."""
    cfg, sd, nl, keeps, taps, gt = r["cfg"], r["sd"], r["nl"], r["keeps"], r["taps"], r["gt"]
    layers = lref.layer_inputs(cfg)
    refs, total, resid, cls, klen = [], {}, {}, {}, {}
    for tap, kind, spec, src, skip in layers:
        gy = r["deps"] if kind == "final" else gt[tap]["g"]
        # the data gradient's contraction: 9 x 64 (the first conv, the final conv's 3 outputs padded to 64), 9 C (Downsample), the
        # 4x4 kernel of the Upsample over C; the other layers' input gradients are chained
        c = taps[src].shape[1]
        klen[src] = max(klen.get(src, 0), {"conv": 576, "final": 576, "down": 9 * c, "up": 16 * c}.get(kind, 0))
        R = gref.layer_grads(sd, cfg, kind, spec, taps[src], None if skip is None else taps[skip], nl, gy, keep_scale=keeps.get(tap))
        refs.append(R)
        total[src] = total.get(src, 0) + R["x"]
        if gref.passthrough(kind, spec, sd):
            resid[src] = resid.get(src, 0) + gy
        cls[src] = max(input_class(kind), cls.get(src, "direct"), key=RANK.get)
        if skip is not None:
            total[skip] = total.get(skip, 0) + R["skip"]
            cls[skip] = max("chained", cls.get(skip, "direct"), key=RANK.get)
    foffs, f = [], 0
    for tap, kind, spec, src, skip in layers:
        foffs.append(f)
        f += spec.cout if kind == "res" else 0

    def got_of(t):
        return r["dx"] if t == "input" else gt[t]["g"]

    def quantities(i, R, with_skip=False):
        tap, kind, spec, src, skip = layers[i]
        q = {f"d {src}": (got_of(src), total[src] - refs[i]["x"] + R["x"], resid.get(src), cls[src], klen[src])}
        if with_skip and skip is not None:
            q[f"d {skip}"] = (got_of(skip), total[skip] - refs[i]["skip"] + R["skip"], resid.get(skip), cls[skip], 0)
        sk = None if skip is None else taps[skip]
        for n in gref.layer_params(sd, kind, spec):
            q[n] = (r["pgrads"][n], R[n], None, param_class(kind, n), param_length(kind, n, taps[src], sk, R["out"].shape[1]))
        if "dfilm" in R:
            q["dfilm"] = (r["dfilm"][:, foffs[i]:foffs[i] + spec.cout], R["dfilm"], None, "chained", 0)
        return q
    return layers, refs, quantities


def miss(q):
    """The largest error of a variant over a layer's quantities, in units of each quantity's bound."""
    return max(rel(got, want, res) / bound_of(c, k)[0] for got, want, res, c, k in q.values())


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", sorted(CASES))
def test_every_layer_gradient_matches_its_fp64_reference(name):
    t0 = time.time()
    r = run_backward(CASES[name], tgl.case_seed(CASES, name))
    cfg, sd, nl, keeps, taps = r["cfg"], r["sd"], r["nl"], r["keeps"], r["taps"]
    b = r["dx"].shape[0]
    rows, worst = [], {}
    failures = identity_failures(r["gt"])     # exact identities of every tensor's gradient
    params = set(r["pgrads"])
    layers, refs, quantities = layer_checks(r)
    checked = set()
    masks_by_shape = {}
    for tap, k in keeps.items():
        masks_by_shape.setdefault(tuple(k.shape), []).append(tap)
    first_res = None
    for i, (tap, kind, spec, src, skip) in enumerate(layers):
        x, sk = taps[src], None if skip is None else taps[skip]
        gy = r["deps"] if kind == "final" else r["gt"][tap]["g"]
        keep = keeps.get(tap)
        q = quantities(i, refs[i])
        checked.update(n for n in q if n in params)
        parts = []
        for label, (got, want, res, c, k) in q.items():
            bound, elem = bound_of(c, k)
            e = rel(got, want, res)
            m, bad = elementwise(got, want, res, elem)
            worst[c] = max(worst.get(c, (0.0, 0.0)), (e, m))
            parts.append(f"{label} {e:.1e}/{m:.1e}")
            if e >= bound:
                failures.append(f"{tap}: {label}: relative L2 {e:.3e} >= {bound:.0e}")
            if bad:
                failures.append(f"{tap}: {label}: {bad}")

        def grads_of(**kw):
            return gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, **dict(dict(keep_scale=keep), **kw))
        variants = {"unrounded": (grads_of(rounded=False), MISS_UNROUNDED)}
        if keep is not None:
            variants["no keep-mask"] = (grads_of(keep_scale=None), MISS_WRONG)
            other = [t for t in masks_by_shape[tuple(keep.shape)] if t != tap]
            if other:
                variants[f"{other[0]}'s keep-mask"] = (grads_of(keep_scale=keeps[other[0]]), MISS_WRONG)
        if skip is not None:
            R = refs[i]
            variants["skip omitted"] = (dict(R, skip=torch.zeros_like(R["skip"])), MISS_WRONG)
            variants["skip one channel late"] = (dict(R, skip=F.pad(R["skip"][:, 1:], (0, 0, 0, 0, 0, 1))), MISS_WRONG)
            if x.shape[1] % ((x.shape[1] + sk.shape[1]) // cfg.norm_groups):
                variants["GroupNorm per source"] = (grads_of(wrong="gn_per_source"), MISS_WRONG)
        if kind == "attn" and x.shape[2] * x.shape[3] < 128:
            variants["softmax over the 128-token batch"] = (grads_of(wrong="joint_softmax"), MISS_WRONG)
        if kind == "up":
            variants["per-tap rounded weights"] = (grads_of(wrong="per_tap"), MISS_WRONG)
        if kind == "res" and first_res is None:
            first_res = tap
            R = refs[i]
            variants["dfilm of images 0, 1 swapped"] = (dict(R, dfilm=R["dfilm"][[1, 0] + list(range(2, b))]), MISS_WRONG)
        for vname, (R, need) in variants.items():
            mv = miss(quantities(i, R, with_skip=True))
            parts.append(f"[{vname}: {mv:.0f}x]")
            if mv < need:
                failures.append(f"{tap}: the {vname} reference misses by only {mv:.1f} bounds (< {need:g})")
        rows.append(f"{tap:>18} {kind:>5}  " + "  ".join(parts))
    # every parameter is checked here, or is a FiLM / block1 bias / noise-MLP gradient (identities of dfilm)
    rest = params - checked
    assert all(k.startswith("noise_level_mlp.") or ".noise_func." in k or k.endswith(".block1.block.3.bias") for k in rest), rest
    net, image_size, bb, h, w, drop = CASES[name]
    print(f"\n{name} (batch {b}, {h}x{w}{', Dropout masks' if drop else ''}): worst (rel L2, element-wise) "
          + ", ".join(f"{k} {v[0]:.2e} {v[1]:.2e}" for k, v in sorted(worst.items())) + f"; {time.time() - t0:.1f} s; "
          + f"training engine {r['workspace'] / 2 ** 30:.2f} GiB\n"
          + "  (per quantity: relative L2 / element-wise; [wrong reference: its miss in bounds])\n" + "\n".join(rows))
    if failures:
        pytest.fail(f"{name}: " + "; ".join(failures[:40]))


def film_param(name):
    return name.startswith("noise_level_mlp.") or ".noise_func." in name or name.endswith(".block1.block.3.bias")


# parameter gradients of two backwards of the same forward differ by the order of the fp32 atomics only: at most 6.2e-3 relative on the
# two-level net (tools/gpu_grad_spread.py, DESIGN.md 3.6), 1.5e-2 measured here on the five-level net (a GroupNorm weight gradient, a sum
# with much cancellation)
SPREAD = 4e-2


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["full_128x128", "tiny_b3_drop", "sr64_512_128x128_b3_drop"])
def test_block_params_are_final_after_their_flush(name):
    """sr3_train_block_params(i): the listed gradients are final once block i and a flush have run (what DataParallelTrainer all-reduces
    bucket by bucket), every parameter is listed at most once, and the unlisted ones are exactly those finish() writes."""
    net, image_size, b, h, w, drop = CASES[name]
    cfg, sd, eng, keeps = make_engine(CASES[name])
    g = torch.Generator().manual_seed(3)
    hr = torch.rand(b, 3, h, w, generator=g).cuda() * 2 - 1
    sr = torch.rand(b, 3, h, w, generator=g).cuda() * 2 - 1 if cfg.in_channel != 3 else None
    gamma = tgl.noise_levels(b).cuda()
    noise = torch.randn(b, 3, h, w, generator=g).cuda()
    table = eng.param_table()
    names = [n for n, _ in table]
    scale = 1.0 / (b * 3 * h * w)

    eng.train_forward(hr, sr, gamma, noise, loss_type="l2")
    grads = [torch.full(s, float("nan"), device="cuda") for _, s in table]
    eng.backward_begin(scale, grads)
    snaps = {}
    for i in reversed(range(eng.num_backward_blocks())):
        eng.backward_block(i)
        eng.backward_flush()
        torch.cuda.synchronize()
        for pi in eng.block_params(i):
            assert pi not in snaps, f"{names[pi]} is listed by two blocks"
            snaps[pi] = grads[pi].clone()
    eng.backward_finish()
    torch.cuda.synchronize()
    early = [names[pi] for pi, s in snaps.items() if not torch.equal(s, grads[pi])]
    assert not early, f"listed before their gradient was final: {early}"
    unlisted = {n for i, n in enumerate(names) if i not in snaps}
    assert unlisted == {n for n in names if film_param(n)}, sorted(unlisted ^ {n for n in names if film_param(n)})
    assert all(torch.isfinite(t).all() for t in grads)

    eng.train_forward(hr, sr, gamma, noise, loss_type="l2")
    whole = [torch.full(s, float("nan"), device="cuda") for _, s in table]
    eng.train_backward(scale, whole)
    torch.cuda.synchronize()
    spread = {n: rel(a.double(), c.double()) for n, a, c in zip(names, grads, whole)}
    worst = max(spread, key=spread.get)
    print(f"\n{name}: {len(snaps)} of {len(names)} parameters listed by {eng.num_backward_blocks()} blocks; stepped vs whole backward: "
          f"largest relative difference {spread[worst]:.2e} ({worst})")
    assert spread[worst] < SPREAD, (worst, spread[worst])

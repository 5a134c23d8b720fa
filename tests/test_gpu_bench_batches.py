"""Every layer of the engines bench.py times, at the per-GPU batches it runs them, against the fp64 layer references of
tests/test_gpu_layers.py (forward) and tests/test_gpu_layer_grads.py (training backward).

Those two files run batches of 2 or 3.  The tile plan depends on the batch (conv_geometry picks tile shape, schedule, split-K, stages and
CTA count from the tile count), so the plan each benchmarked engine runs is tested here:

  16->128 bf16 at 16 images (the headline), 8 and 4 (one of 2 and 4 GPUs); 16->128 in precise mode at 16; 64->512 at 512x512, 4 images;
  the unconditional 128 net (in_channel 3) at 32 (one GPU) and 4 (one of 8); the 16->128 training step at 8 images with Dropout masks
  (p = 0.2), its forward and backward.

Every case clears the SR3_* tile overrides and runs the default plan, printed per cell (tall halo, tile rows, BLOCK_N, schedule, split-K,
stages, tiles / CTAs).  On a 132-SM device the 16->128 batch-16 plan must be test_gpu_plan.PLAN_16_128_B16, with at least one ping-pong
op whose persistent CTAs walk more than one tile: when that table is re-fitted, this test checks the accuracy of the new plan.

The bounds are the class bounds of the two files, unchanged, applied twice: over the whole batch, and on each image's slice of a layer's
output or input gradient (the largest per-image branch relative L2, and the element-wise test with each image's own rms).  A fault in one
image of 16 moves the batch relative L2 by only 1/sqrt(16) of its own error; per image it shows in full.  Parameter gradients are sums over
images and stay batch-level.

Each bound is shown to discriminate per image.  The unrounded reference (bf16) and the bf16 reference (precise mode) miss as in the two
files.  These wrong references miss every layer they apply to by at least 10 bounds:
- the FiLM rows of images B/2 - 1 and B/2 swapped, and of B - 2 and B - 1: images in different tiles and CTAs (every ResnetBlock; in the
  backward, the same swaps of dfilm);
- every GroupNorm of image b normalised with the statistics of image (b + 1) mod B (_layer_ref's gn_stats; every ResnetBlock, attention
  layer and the final block, forward and backward).
noise_levels(b) gives neighbouring images noise levels more than 0.45 apart, so a FiLM row of the wrong image shows.

The final conv's posterior epilogue is checked at the benchmark batch of 16->128 and 64->512 as test_gpu_sampling does at batch 3:
p_mean_variance bit for bit against torch-CPU fp32 predict_start_from_noise / clamp / q_posterior of unet_forward's eps, and p_sample
within the ulp bound of mean + z sigma, with sample indices that cross 2^32 inside the batch.

Each case prints its wall time and torch.cuda.max_memory_allocated() (the taps and fp64 references; the engine's own device memory is
allocated outside torch's allocator).  A forward case reads its taps in fp32 and widens each to fp64 only while a layer reads it.

Per-image bound of the bf16 chained layers (ResnetBlock, attention, final block).  At the class bound 4e-4, the first runs failed only
per image and only at the small levels: over the batch every layer stayed within 2.6e-4, but single images reached 4.1e-4 to 7.0e-4 on
the 8x8 layers (downs.13, mid.*, 32768 values per image) and 4.1e-4 on the 16x16 attention.  The failing image changed from layer to layer
(images 1, 2, 6, 13, 15, 17, 19, 21, 24), and the per-image maximum grew with the number of images drawn: 2.7e-4 at 4 images, 4.1e-4 at 8,
4.8e-4 at 16, 7.0e-4 at 32.  Precise mode, on the same layers at 16 images, was even to 3.05e-5 per image against 3.04e-5 over the batch.
So this is rounding, not routing: the error of these layers is a handful of bf16 flips per image on a small level (about 2^-16 of an
operand's 32768 values), and the error of one image fluctuates with its count of flips.  The per-image bound is therefore the class bound
times sqrt(2^18 / n) for an image slice of n < 2^18 values: x2.83 at 8x8x512, x1.41 at 16x16x512, x1 from 32x32x256 up.  The other
classes, precise mode and the backward keep the class bounds per image.

Measured over the cases (NVIDIA H100 80GB HBM3, 700 W power limit), batch / worst image, relative L2:
  forward bf16 chained  <= 2.7e-4 / at most 0.81 of the per-image bound (4.6e-4 of 5.7e-4, downs.10 attention at 16 images); largest
                        per image 6.3e-4 of 1.13e-3 (8x8, 32 images); element-wise <= 5.9e-3 (bound 1e-2)
  forward bf16 direct   <= 4.8e-6 / 4.8e-6
  precise mode          chained 3.0e-5 / 3.1e-5, direct 2.2e-5 / 2.2e-5 (k-scaled bounds; at most 0.85 of the bound)
  backward (8 images)   direct 8.8e-6 / 8.9e-6, chained 2.7e-4 / 2.8e-4, attention input 7.5e-4 / 9.9e-4 (bound 1.2e-3); weight
                        gradients contract 248 to 8192 pixels per wgrad_kernel slice
Smallest misses in bounds: unrounded 5x (64->512) to 7x; bf16 reference in precise mode 148x; FiLM swaps 16x (forward, uncond 128 at 32
images, 8x8 against the scaled bound) and 2545x (dfilm); GroupNorm of image b + 1 18x forward, 303x backward.
Wall time 1.5 to 8.8 s per case; torch peak 1.2 GiB (16->128 at 4 images) to 12.1 GiB (64->512 at 512x512), 11.3 GiB for the training
case (plus the training engine's own 3.84 GiB).  With film_kernel made to write image b's row to image b ^ 1 for b >= 8, the 16->128
batch-16 cases (bf16 and precise) failed, naming images 8 to 15 from the first ResnetBlock on (1.8e-2 per image, 45x the bound), while
every case of tests/test_gpu_layers.py (batches <= 3) still passed."""
import math
import time

import numpy as np
import pytest
import torch

import _layer_grad_ref as gref
import _layer_ref as lref
import _philox
import test_gpu_layer_grads as tglg
import test_gpu_layers as tgl
import test_gpu_plan as tgp
import test_gpu_sampling as tgs
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

UNCOND = dict(tgl.FULL, in_channel=3)            # sample_sr3_128: the 16->128 UNet without a condition
# name -> test_gpu_layers case (net, image_size, batch, height, width, precision, None)
FORWARD = {
    "sr16_128_b16": (tgl.FULL, 128, 16, 128, 128, "bf16", None),
    "sr16_128_b8": (tgl.FULL, 128, 8, 128, 128, "bf16", None),
    "sr16_128_b4": (tgl.FULL, 128, 4, 128, 128, "bf16", None),
    "sr16_128_b16_precise": (tgl.FULL, 128, 16, 128, 128, "fp32", None),
    "sr64_512_512x512_b4": (tgl.SR64_512, 512, 4, 512, 512, "bf16", None),
    "uncond_128_b32": (UNCOND, 128, 32, 128, 128, "bf16", None),
    "uncond_128_b4": (UNCOND, 128, 4, 128, 128, "bf16", None),
}
# name -> test_gpu_layer_grads case (net, image_size, batch, height, width, Dropout p)
TRAIN = {"sr16_128_train_b8": (tgl.FULL, 128, 8, 128, 128, 0.2)}
POSTERIOR = ("sr16_128_b16", "sr64_512_512x512_b4")
MISS_WRONG = 10.0
IMAGE_N0 = 2 ** 18     # bf16 chained layers: the per-image relative L2 bound grows as sqrt(IMAGE_N0 / n) for an image slice of n < IMAGE_N0 values
NOISE_SEED = tgs.SEED


def seed_of(name):
    """The seed of a case's inputs: 1000 + its place among all cases here in sorted order."""
    return 1000 + sorted(list(FORWARD) + list(TRAIN)).index(name)


@pytest.fixture(autouse=True)
def default_plan(monkeypatch):
    for k in tgp.KNOBS:
        monkeypatch.delenv(k, raising=False)


def plan_rows(plan):
    """The tile ops of tile_schedules(): (op, (H, W, C), tall, rows, BLOCK_N, schedule, split-K, stages, tiles, CTAs)."""
    return [(i, tuple(s["out_hwc"]), s["tall"], 128 * s["mh"], s["block_n"], s["schedule"], s["ksplit"], s["stages"], s["tiles"], s["ctas"])
            for i, s in enumerate(plan) if s is not None]


def plan_summary(rows):
    """One line per plan cell: the ops with the same output shape and variant."""
    cells = {}
    for r in rows:
        cells.setdefault(r[1:], []).append(r[0])
    return "\n".join(f"  {'x'.join(map(str, k[0])):>12}  tall {k[1]}  rows {k[2]:>3}  BLOCK_N {k[3]:>3}  {k[4]:>11}  split-K {k[5]}  stages {k[6]}  "
                     f"tiles / CTAs {k[7]:>5} / {k[8]:>3}  ops {','.join(map(str, ops))}" for k, ops in cells.items())


def plan_failures(name, rows):
    """The 16->128 batch-16 plan on a 132-SM device is test_gpu_plan's table, and persistent CTAs of a ping-pong op walk several tiles."""
    if name != "sr16_128_b16":
        return []
    if torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count != 132:
        print("the plan table is for a 132-SM H100: not compared")
        return []
    failures = []
    bad = [(g, w) for g, w in zip([r[:7] for r in rows], tgp.PLAN_16_128_B16) if g != w]
    if len(rows) != len(tgp.PLAN_16_128_B16) or bad:
        failures.append(f"the plan is not test_gpu_plan.PLAN_16_128_B16: {len(rows)} tile ops, first differences {bad[:3]}")
    if not any(r[5] == "pingpong" and r[8] > r[9] for r in rows):
        failures.append("no ping-pong op walks more tiles than it has CTAs")
    return failures


def image_rel(got, ref, resid):
    """[B]: each image's relative L2 of got - ref on the branch (ref less the residual)."""
    n = got.shape[0]
    b = (ref if resid is None else ref - resid).reshape(n, -1)
    return (got - ref).reshape(n, -1).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)


def per_image(label, got, ref, resid, bound, elem):
    """(per-image relative L2 [B], per-image largest |got - ref| / (|b| + rms(b)) with the image's own rms [B], failures naming the image)."""
    n = got.shape[0]
    rel = image_rel(got, ref, resid)
    b = (ref if resid is None else ref - resid).reshape(n, -1)
    d = (got - ref).reshape(n, -1)
    ratio = d.abs() / (b.abs() + b.pow(2).mean(1, keepdim=True).sqrt())
    worst = ratio.amax(1)
    failures = [f"{label}: image {i}: relative L2 {rel[i].item():.3e} >= {bound:.1e}" for i in (rel >= bound).nonzero().flatten().tolist()]
    for i in (worst > elem).nonzero().flatten().tolist():
        j = int((ratio[i] > elem).nonzero()[0])
        at = tuple(int(v) for v in np.unravel_index(j, tuple(got.shape[1:])))
        failures.append(f"{label}: image {i}: {int((ratio[i] > elem).sum())} elements past {elem:.0e} (|b| + rms(b) of the image), first at "
                        f"{at}: got {got.reshape(n, -1)[i, j].item():.7g}, want {ref.reshape(n, -1)[i, j].item():.7g}")
    return rel, worst, failures


def image_bound(precision, cls, bound, n):
    """The per-image relative L2 bound of a layer whose image slice holds n values: the class bound, and for bf16 chained layers (whose
    error is a few rounding flips per image on the small levels) the class bound sqrt(IMAGE_N0 / n) times below IMAGE_N0 values."""
    return bound * max(1.0, math.sqrt(IMAGE_N0 / n)) if (precision, cls) == ("bf16", "chained") else bound


def film_swaps(b):
    """The two wrong FiLM permutations: images B/2 - 1 and B/2 swapped, and B - 2 and B - 1."""
    out = {}
    for p, q in ((b // 2 - 1, b // 2), (b - 2, b - 1)):
        perm = list(range(b))
        perm[p], perm[q] = q, p
        out[f"FiLM {p},{q} swapped"] = perm
    return out


def note_miss(misses, vname, m, need, label, failures):
    misses[vname] = min(misses.get(vname, math.inf), m)
    if m < need:
        failures.append(f"{label}: the {vname} reference misses by only {m:.1f} bounds (< {need:g})")
    return f"[{vname}: {m:.0f}x]"


def check_forward(cfg, sd, nl, taps, precision, unfused, keeps, failures):
    """Every layer of one forward against lref over the batch and per image, and the wrong references' misses.  taps {tap: NCHW} is
    consumed: each tap is widened to fp64 while a layer reads it and dropped after its last reader.  keeps: {ResnetBlock tap: scaled
    keep-mask}.  -> (rows, {class: [batch rel L2, batch element-wise, worst image rel L2, worst image element-wise]}, {wrong: least miss})."""
    layers = lref.layer_inputs(cfg)
    last = {}
    for i, (tap, kind, spec, src, skip) in enumerate(layers):
        for t in (tap, src, skip):
            last[t] = i
    b = nl.shape[0]
    rows, worst, misses = [], {}, {}
    for i, (tap, kind, spec, src, skip) in enumerate(layers):
        x, sk, got = taps[src].double(), None if skip is None else taps[skip].double(), taps[tap].double()
        keep = keeps.get(tap)
        resid = lref.residual(kind, spec, sd, x)
        assert torch.isfinite(got).all(), tap
        cls = "direct" if kind in tgl.DIRECT else "chained"
        k = tgl.contraction(kind, x.shape[1] + (0 if sk is None else sk.shape[1]), got.shape[1], x.shape[2] * x.shape[3])
        bound, elem = tgl.bounds(precision, cls, k)
        ibound = image_bound(precision, cls, bound, got[0].numel())

        def ref_of(**kw):
            return lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, **dict(dict(precision=precision, unfused=unfused, keep_scale=keep), **kw))
        ref = ref_of()
        e = tgl.branch_rel(got, ref, resid)
        m, bad = tgl.elementwise(got, ref, resid, elem)
        ei, mi, bad_i = per_image(tap, got, ref, resid, ibound, elem)
        wi = int(ei.argmax())
        w = worst.setdefault(cls, [0.0] * 4)
        for j, v in enumerate((e, m, ei.max().item(), mi.max().item())):
            w[j] = max(w[j], v)
        row = (f"{tap:>20} {kind:>5}  K {k:>5}  rel L2 {e:.2e} (bound {bound:.1e}), worst image {wi:>2} {ei[wi].item():.2e} (bound {ibound:.1e})  "
               f"element-wise {m:.2e}, worst image {mi.max().item():.2e} (bound {elem:.1e})")
        if e >= bound:
            failures.append(f"{tap}: relative L2 {e:.3e} >= {bound:.1e}")
        if bad:
            failures.append(f"{tap}: {bad}")
        failures.extend(bad_i)
        if precision == "bf16":
            row += "  " + note_miss(misses, "unrounded", tgl.branch_rel(got, ref_of(rounded=False), resid) / bound, tgl.MISS_UNROUNDED, tap,
                                    failures)
        else:
            base = tgl.BOUNDS[precision, cls][0]
            row += "  " + note_miss(misses, "bf16 reference", tgl.branch_rel(got, ref_of(precision="bf16"), resid) / base, tgl.MISS_BF16, tap,
                                    failures)
        if kind == "res":
            film = lref.film_rows(sd, spec.name + ".res_block", nl, cfg.inner_channel)
            for vname, perm in film_swaps(b).items():
                mv = image_rel(got, ref_of(film=film[perm]), resid).max().item() / ibound
                row += " " + note_miss(misses, vname, mv, MISS_WRONG, tap, failures)
        if kind in ("res", "attn", "final"):
            mv = image_rel(got, ref_of(gn_stats=lref.neighbour(b)), resid).max().item() / ibound
            row += " " + note_miss(misses, "GroupNorm of image b + 1", mv, MISS_WRONG, tap, failures)
        rows.append(row)
        del x, sk, got, ref
        for t in {tap, src, skip} - {None}:
            if last[t] == i:
                del taps[t]
    return rows, worst, misses


def summary(worst, misses):
    return ("worst (rel L2 batch / image, element-wise batch / image): "
            + ", ".join(f"{c} {v[0]:.2e} / {v[2]:.2e}, {v[1]:.2e} / {v[3]:.2e}" for c, v in sorted(worst.items()))
            + "\nleast misses in bounds: " + ", ".join(f"{k} {v:.0f}x" for k, v in misses.items()))


def resources(t0):
    return f"{time.time() - t0:.1f} s, torch peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB"


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", sorted(FORWARD))
def test_bench_batch_forward_layers(name):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    case = FORWARD[name]
    net, image_size, b, h, w, precision, _ = case
    cfg, sd, nl, taps, _, plan = tgl.run_engine(case, seed_of(name), tap_dtype=torch.float32)
    prow = plan_rows(plan)
    failures = plan_failures(name, prow)
    rows, worst, misses = check_forward(cfg, sd, nl, taps, precision, False, {}, failures)
    print(f"\n{name} ({precision}, batch {b}, {h}x{w}): {resources(t0)}\nplan:\n{plan_summary(prow)}\n{summary(worst, misses)}\n"
          + "\n".join(rows))
    if failures:
        pytest.fail(f"{name}: " + "; ".join(failures[:40]))


def image_miss(q, params):
    """The largest error of a variant over a layer's quantities in bounds: per image for data gradients and dfilm, over the batch for
    parameter gradients."""
    return max((tglg.rel(got, want, res) if label in params else image_rel(got, want, res).max().item()) / tglg.bound_of(c, k)[0]
               for label, (got, want, res, c, k) in q.items())


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", sorted(TRAIN))
def test_bench_batch_training_layers(name):
    """The training step at its per-GPU batch: every layer's forward (train_unet_forward) and backward (train_unet_backward)."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    case = TRAIN[name]
    net, image_size, b, h, w, drop = case
    r = tglg.run_backward(case, seed_of(name))
    cfg, sd, nl, keeps, taps = r["cfg"], r["sd"], r["nl"], r["keeps"], r["taps"]
    prow = plan_rows(r["plan"])
    failures = tglg.identity_failures(r["gt"])
    frows, fworst, fmisses = check_forward(cfg, sd, nl, dict(taps, eps=r.pop("eps")), "bf16", True, keeps, failures)

    params = set(r["pgrads"])
    layers, refs, quantities = tglg.layer_checks(r)
    checked, rows, worst, misses = set(), [], {}, {}
    for i, (tap, kind, spec, src, skip) in enumerate(layers):
        x, sk = taps[src], None if skip is None else taps[skip]
        gy = r["deps"] if kind == "final" else r["gt"][tap]["g"]
        q = quantities(i, refs[i])
        checked.update(n for n in q if n in params)
        parts = []
        for label, (got, want, res, c, k) in q.items():
            bound, elem = tglg.bound_of(c, k)
            e = tglg.rel(got, want, res)
            m, bad = tglg.elementwise(got, want, res, elem)
            wv = worst.setdefault(c, [0.0] * 4)
            if label in params:
                parts.append(f"{label} {e:.1e}/{m:.1e}")
                wv[:2] = max(wv[0], e), max(wv[1], m)
            else:
                ei, mi, bad_i = per_image(f"{tap}: {label}", got, want, res, bound, elem)
                wi = int(ei.argmax())
                parts.append(f"{label} {e:.1e}/{m:.1e} (image {wi} {ei[wi].item():.1e}/{mi.max().item():.1e})")
                failures.extend(bad_i)
                wv[:] = max(wv[0], e), max(wv[1], m), max(wv[2], ei.max().item()), max(wv[3], mi.max().item())
            if e >= bound:
                failures.append(f"{tap}: {label}: relative L2 {e:.3e} >= {bound:.0e}")
            if bad:
                failures.append(f"{tap}: {label}: {bad}")

        def grads_of(**kw):
            return gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, **dict(dict(keep_scale=keeps.get(tap)), **kw))
        mv = tglg.miss(quantities(i, grads_of(rounded=False), with_skip=True))
        parts.append(note_miss(misses, "unrounded", mv, tglg.MISS_UNROUNDED, tap, failures))
        if kind == "res":
            for vname, perm in film_swaps(b).items():
                R = dict(refs[i], dfilm=refs[i]["dfilm"][perm])
                parts.append(note_miss(misses, "d" + vname, image_miss(quantities(i, R, with_skip=True), params), MISS_WRONG, tap, failures))
        if kind in ("res", "attn", "final"):
            mv = image_miss(quantities(i, grads_of(wrong="gn_neighbour"), with_skip=True), params)
            parts.append(note_miss(misses, "GroupNorm of image b + 1", mv, MISS_WRONG, tap, failures))
        rows.append(f"{tap:>18} {kind:>5}  " + "  ".join(parts))
    rest = params - checked
    assert all(tglg.film_param(k) for k in rest), rest
    wg = sorted({tglg.param_length(kind, n, taps[src], None if skip is None else taps[skip], refs[i]["out"].shape[1])
                 for i, (tap, kind, spec, src, skip) in enumerate(layers) for n in gref.layer_params(sd, kind, spec)} - {0})
    print(f"\n{name} (batch {b}, {h}x{w}, Dropout masks p = {drop}): {resources(t0)}; training engine {r['workspace'] / 2 ** 30:.2f} GiB\n"
          f"forward plan:\n{plan_summary(prow)}\nweight-gradient contraction lengths (pixels per wgrad_kernel slice): {wg}\n"
          f"forward: {summary(fworst, fmisses)}\n" + "\n".join(frows)
          + f"\nbackward: {summary(worst, misses)}\n"
          + "  (per quantity: relative L2 / element-wise over the batch (worst image); [wrong reference: its miss in bounds])\n" + "\n".join(rows))
    if failures:
        pytest.fail(f"{name}: " + "; ".join(failures[:40]))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", POSTERIOR)
def test_bench_batch_posterior_epilogue(name):
    """p_mean_variance equals torch-CPU fp32 predict_start_from_noise / clamp / q_posterior on unet_forward's eps bit for bit, and p_sample
    is mean + z sigma within tests/test_gpu_sampling's ulp bound with z the documented Philox stream, at t = T - 1, T / 2, 1 (t = 0: the
    mean), for sample indices 2^32 - B / 2 .. 2^32 + B / 2 - 1 (2^32 - 8 onwards at 16 images): the high word changes inside the batch."""
    case = FORWARD[name]
    net, image_size, b, h, w, precision, _ = case
    cfg, sd, eng = tgl.make_engine(case)
    sch = orc.make_schedule(tgl.SCHED)
    T = sch.num_timesteps
    g = torch.Generator().manual_seed(seed_of(name) + 100)
    cond, x_t = torch.rand(b, 3, h, w, generator=g) * 2 - 1, torch.randn(b, 3, h, w, generator=g)
    first = 2 ** 32 - b // 2
    idx = first + np.arange(b, dtype=np.uint64)
    for t in (T - 1, T // 2, 1, 0):
        eps = eng.unet_forward(torch.cat([cond, x_t], 1), orc.noise_level_for_t(sch, t, b)).cpu()
        x0 = orc.predict_start_from_noise(sch, x_t, t, eps)
        for clip in (True, False):
            mean, lv = eng.p_mean_variance(x_t, t, clip, cond)
            ref, ref_lv = orc.q_posterior(sch, x0.clamp(-1.0, 1.0) if clip else x0, x_t, t)
            diff = (mean.cpu() != ref).flatten(1).sum(1)
            assert not diff.any(), f"t={t} clip={clip}: means differ at {diff.tolist()} elements per image"
            assert lv == float(ref_lv)
        x = eng.p_sample(x_t, t, cond, None, NOISE_SEED, first)
        mean = eng.p_mean_variance(x_t, t, True, cond)[0]
        if t == 0:
            assert torch.equal(x, mean)
            continue
        x, mean = x.cpu().double().numpy(), mean.cpu().double().numpy()
        sigma = math.exp(0.5 * float(sch.buffers["posterior_log_variance_clipped"][t]))
        z = _philox.sampling_noise(NOISE_SEED, idx, t, h, w)
        ratio = (np.abs(x - (mean + z * sigma)) / tgs._noise_bound(mean, z, sigma)).reshape(b, -1).max(1)
        print(f"{name} t={t}: max |x - (mean + z sigma)| / bound per image {np.array2string(ratio, precision=3)}")
        assert ratio.max() <= 1.0, (t, [i for i in range(b) if ratio[i] > 1.0])
    del eng

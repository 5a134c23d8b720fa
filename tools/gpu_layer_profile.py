"""Per-launch profile of one eager reverse step, with the tile-kernel variant of every launch; and, with --sweep, the same profile once per
tile-kernel candidate, so that the plan of conv_geometry can be checked (and fitted) launch by launch.

For each launch of the step (sr3_engine_profile_step: CUDA events around every launch, averaged over --reps after a warm-up) it lists the
kind, the output resolution and channels, the tile shape, schedule (cooperative / ping-pong), split-K factor and tiles per CTA (from
sr3_tile_schedule), the time and the algorithmic TFLOP/s.  It then sums the time by resolution level and by variant, and records the card
name, power limit and SM clocks read in the same process.  Writes JSON (--out) and prints a summary.

    python tools/gpu_layer_profile.py --out prof.json [--label change] [--root <other checkout>] [--config sr_64_512_b4]
    python tools/gpu_layer_profile.py --sweep --out sweep.json [--config all]

--config names a workload of bench.py (sr_16_128_b16, the flagship, by default; the batch follows it unless --batch is given).
SR3_PINGPONG=0|1 in the environment forces the schedule (DESIGN.md section 3.7).  --root profiles another checkout of the project (e.g. the
parent commit, built in place); a checkout without sr3_tile_schedule reports launches without their variant.

--sweep builds one engine per candidate of SWEEP, each forced with the planner's knobs (SR3_TALL_MH / SR3_TALL_BN / SR3_BLOCK_N /
SR3_PINGPONG / SR3_KSPLIT / SR3_STAGES; a knob applies to every layer it can, so one engine times one candidate of many layers), and keys
each tile op's time by the variant it actually ran.  For every tile op it reports the variant the unforced plan chose, the fastest one
measured and their ratio; then the sum of the chosen and of the per-op best times.  A launch the model ranks wrongly shows there.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

KINDS = {0: "tile", 1: "groupnorm_apply", 2: "cast", 3: "softmax", 4: "other"}
KNOBS = ("SR3_TALL_MH", "SR3_TALL_BN", "SR3_BLOCK_N", "SR3_PINGPONG", "SR3_KSPLIT", "SR3_STAGES")


def sweep_candidates():
    """Knob settings of the sweep: the unforced plan first, then every tall (MH, BLOCK_N) and generic BLOCK_N tile cooperative with the
    split the launch allows and unsplit, ping-pong wherever gemm_pingpong_ok has that form, and the split factors and pipeline depths on
    the model's shapes."""
    c = [{}, {"SR3_PINGPONG": "0"}, {"SR3_PINGPONG": "1"}]
    for mh, bn in ((2, 128), (2, 64), (1, 64), (1, 32)):
        shape = {"SR3_TALL_MH": str(mh), "SR3_TALL_BN": str(bn)}
        c += [shape, dict(shape, SR3_KSPLIT="1")]
        if (mh, bn) in ((2, 64), (1, 64)):
            c.append(dict(shape, SR3_PINGPONG="1"))
    for bn in (128, 64, 32):
        c += [{"SR3_BLOCK_N": str(bn)}, {"SR3_BLOCK_N": str(bn), "SR3_KSPLIT": "1"}]
        if bn in (128, 64):
            c.append({"SR3_BLOCK_N": str(bn), "SR3_PINGPONG": "1"})
    c += [{"SR3_KSPLIT": str(k)} for k in (2, 4, 8)]
    c += [{"SR3_STAGES": str(s)} for s in (2, 3)]
    return c


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        info["nvidia_smi"] = dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def variant_of(g):
    return (f"{'tall' if g['tall'] else 'gen'} {128 * g['mh']}x{g['block_n']} {g['schedule']}"
            f"{' split' + str(g['ksplit']) if g['ksplit'] > 1 else ''} st{g['stages']}")


def make_net(config):
    import torch
    import bench
    import sr3_b200
    unet, image, cond = bench.WORKLOADS[config][:3]
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = sr3_b200.define_G(bench.make_opt(bench.SCHED, unet, image, cond)).to(dev)
    net.set_new_noise_schedule(bench.SCHED, dev)
    return net


def profile_engine(net, config, B, t, reps):
    """[(kind, ms, flops, bytes)] and the tile schedules of one eager step of a fresh engine of `net`, planned under the current
    environment."""
    import torch
    import bench
    image, cond = bench.WORKLOADS[config][1:3]
    dev = torch.device("cuda", 0)
    net.denoise_fn._engines.clear()                    # plan anew: the knobs are read when an engine is built
    net.denoise_fn._engine_versions.clear()
    eng = net.denoise_fn.engine(B, conditional=cond, channels=3)
    torch.manual_seed(1)
    c = (torch.rand(B, 3, image, image) * 2 - 1).to(dev) if cond else None
    eng.loop_begin(c, torch.randn(B, 3, image, image).to(dev), seed=1)
    eng.steps(1999, 3)
    torch.cuda.synchronize()
    prof = eng.profile_step(t, reps=reps)
    scheds = eng.tile_schedules() if hasattr(eng, "tile_schedules") else [None] * len(prof)
    net.denoise_fn._engines.clear()
    net.denoise_fn._engine_versions.clear()
    del eng
    torch.cuda.empty_cache()
    return prof, scheds


def sweep(config, B, args):
    saved = {k: os.environ.pop(k, None) for k in KNOBS}
    ops = None
    net = make_net(config)
    try:
        for env in sweep_candidates():
            for k in KNOBS:
                os.environ.pop(k, None)
            os.environ.update(env)
            prof, scheds = profile_engine(net, config, B, args.t, args.reps)
            if ops is None:
                ops = [{"op": i, "res": g["out_hwc"][0], "cout": g["out_hwc"][2], "gflop": fl / 1e9, "times": {}, "geometry": {}}
                       if g is not None else None for i, ((kind, ms, fl, by), g) in enumerate(zip(prof, scheds))]
            assert len(prof) == len(ops), "the candidates built different op lists"
            for r, (kind, ms, fl, by), g in zip(ops, prof, scheds):
                if r is None:
                    continue
                v = variant_of(g)
                r["times"][v] = min(ms, r["times"].get(v, 1e30))
                r["geometry"][v] = {k: g[k] for k in ("h_box", "b_box", "tiles", "ctas", "res_smem")}
                if not env:
                    r["chosen"] = v
            print(f"  {config} {env or 'model'}: tile {sum(ms for (k, ms, _, _) in prof if k == 0):.3f} ms", flush=True)
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    tile = [r for r in ops if r is not None]
    for r in tile:
        r["best"] = min(r["times"], key=r["times"].get)
        r["chosen_over_best"] = r["times"][r["chosen"]] / r["times"][r["best"]]
    chosen_ms = sum(r["times"][r["chosen"]] for r in tile)
    best_ms = sum(r["times"][r["best"]] for r in tile)
    print(f"[{config} B={B}] tile ops {len(tile)}: chosen {chosen_ms:.3f} ms, per-op best {best_ms:.3f} ms ({chosen_ms / best_ms - 1:+.1%})")
    for r in tile:
        flag = "  <-- " if r["chosen_over_best"] > 1.05 else ""
        print(f"  op {r['op']:3d} {r['res']:4d}^2 cout {r['cout']:5d}  chosen {r['chosen']:34s} {r['times'][r['chosen']] * 1e3:8.1f} us  "
              f"best {r['best']:34s} {r['times'][r['best']] * 1e3:8.1f} us  x{r['chosen_over_best']:.3f}{flag}")
    return {"config": config, "batch": B, "chosen_ms": chosen_ms, "best_ms": best_ms, "candidates": sweep_candidates(), "ops": tile}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--label", default="")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--config", default="sr_16_128_b16", help="a workload of bench.WORKLOADS, or 'all' (with --sweep)")
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--t", type=int, default=1000)
    ap.add_argument("--sweep", action="store_true", help="profile once per candidate of sweep_candidates() and compare with the plan")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import bench

    if args.sweep:
        configs = list(bench.WORKLOADS) if args.config == "all" else [args.config]
        info_before = gpu_info()
        out = [sweep(c, args.batch or bench.WORKLOADS[c][3], args) for c in configs]
        result = {"label": args.label, "reps": args.reps, "t": args.t, "gpu_before": info_before, "gpu_after": gpu_info(), "sweeps": out}
        print(f"{info_before['name']} before: {info_before.get('nvidia_smi')}\n  after: {result['gpu_after'].get('nvidia_smi')}")
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
        return

    B = args.batch or bench.WORKLOADS[args.config][3]
    info_before = gpu_info()
    prof, scheds = profile_engine(make_net(args.config), args.config, B, args.t, args.reps)
    info_after = gpu_info()

    rows = []
    by_level = defaultdict(lambda: {"ms": 0.0, "tile_ms": 0.0, "launches": 0})
    by_variant = defaultdict(lambda: {"ms": 0.0, "launches": 0, "flops": 0.0})
    for i, ((kind, ms, fl, by), g) in enumerate(zip(prof, scheds)):
        r = {"op": i, "kind": KINDS.get(kind, str(kind)), "ms": ms, "tflops": (fl / (ms * 1e-3) / 1e12) if ms > 0 and fl > 0 else 0.0,
             "gflop": fl / 1e9}
        if g is not None:
            oh, ow, c = g["out_hwc"]
            ksplit = g["ksplit"]
            r.update(res=oh, cout=c, tile=f"{128 * g['mh']}x{g['block_n']}", tall=g["tall"], schedule=g["schedule"], split=ksplit,
                     stages=g["stages"], tiles=g["tiles"], ctas=g["ctas"], tiles_per_cta=round(g["tiles"] * ksplit / max(g["ctas"], 1), 2))
            lv = by_level[str(oh)]
            lv["tile_ms"] += ms
            var = f"{r['tile']} {'tall' if g['tall'] else 'generic'} {g['schedule']}{' split' if ksplit > 1 else ''}"
            v = by_variant[var]
            v["ms"] += ms; v["launches"] += 1; v["flops"] += fl
        else:
            lv = by_level["(no variant)" if kind == 0 else "other kinds"]
        lv["ms"] += ms
        lv["launches"] += 1
        rows.append(r)
    for v in by_variant.values():
        v["tflops"] = v.pop("flops") / (v["ms"] * 1e-3) / 1e12 if v["ms"] > 0 else 0.0
    tile_ms = sum(r["ms"] for r in rows if r["kind"] == "tile")
    result = {
        "label": args.label, "root": os.path.abspath(args.root), "SR3_PINGPONG": os.environ.get("SR3_PINGPONG"),
        "config": args.config, "batch": B, "reps": args.reps, "t": args.t,
        "gpu_before": info_before, "gpu_after": info_after,
        "step_ms_eager": sum(r["ms"] for r in rows), "tile_ms": tile_ms,
        "by_level": dict(by_level), "by_variant": dict(by_variant), "launches": rows,
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(f"[{args.label}] SR3_PINGPONG={result['SR3_PINGPONG']} {info_before['name']} {info_before.get('nvidia_smi')}")
    print(f"  eager step {result['step_ms_eager']:.3f} ms, tile kernel {tile_ms:.3f} ms")
    for k in sorted(by_level, key=lambda s: (not s.isdigit(), -int(s) if s.isdigit() else 0)):
        print(f"  level {k:>12s}: {by_level[k]['ms']:.3f} ms ({by_level[k]['launches']} launches, tile {by_level[k]['tile_ms']:.3f} ms)")
    for k in sorted(by_variant, key=lambda s: -by_variant[s]["ms"]):
        v = by_variant[k]
        print(f"  {k:40s} {v['ms']:.3f} ms  {v['launches']:3d} launches  {v['tflops']:.1f} TFLOP/s")


if __name__ == "__main__":
    main()

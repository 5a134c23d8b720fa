"""Per-launch profile of one eager reverse step of the flagship workload (16->128 SR3, B = 16), with the tile-kernel variant of every launch.

For each launch of the step (sr3_engine_profile_step: CUDA events around every launch, averaged over --reps after a warm-up) it lists the
kind, the output resolution and channels, the tile shape, schedule (cooperative / ping-pong), split-K factor and tiles per CTA (from
sr3_tile_schedule), the time and the algorithmic TFLOP/s.  It then sums the time by resolution level and by variant, and records the card
name, power limit and SM clocks read in the same process.  Writes JSON (--out) and prints a summary.

    python tools/gpu_layer_profile.py --out prof.json [--label change] [--root <other checkout>]

SR3_PINGPONG=0|1 in the environment forces the schedule (DESIGN.md section 3.7).  --root profiles another checkout of the project (e.g. the
parent commit, built in place); a checkout without sr3_tile_schedule reports launches without their variant.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

KINDS = {0: "tile", 1: "groupnorm_apply", 2: "cast", 3: "softmax", 4: "other"}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--label", default="")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--t", type=int, default=1000)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    import bench
    import sr3_b200
    from sr3_b200 import _native

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = sr3_b200.define_G(bench.make_opt(bench.SCHED)).to(dev)
    net.set_new_noise_schedule(bench.SCHED, dev)
    B = args.batch
    eng = net.denoise_fn.engine(B, conditional=True, channels=3)
    eng.loop_begin((torch.rand(B, 3, 128, 128) * 2 - 1).to(dev), torch.randn(B, 3, 128, 128).to(dev), seed=1)
    eng.steps(1999, 3)
    torch.cuda.synchronize()
    info_before = gpu_info()
    prof = eng.profile_step(args.t, reps=args.reps)
    info_after = gpu_info()
    scheds = eng.tile_schedules() if hasattr(eng, "tile_schedules") else [None] * len(prof)

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
        "config": "sr_sr3_16_128", "batch": B, "reps": args.reps, "t": args.t,
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

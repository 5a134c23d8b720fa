"""Continuous batching of canvases of any size (GaussianDiffusion.super_resolution_windowed_stream, sr3_wstream_*) on the 16->128 config
in bf16, window 128x128, overlap 32, a short schedule.  A traffic mix of canvas sizes is drawn from a seed; two arms run the same requests
in the same process, alternated round by round:
  (a) the windowed stream at a few slot counts, driven through WindowedStreamSampler exactly as windowed_stream_plan says (one step per
      plan step, idle slots included); a CUDA event after every step gives each request's latency from the start of its arrival step to
      the end of its last step;
  (b) super_resolution_windowed once per request, in arrival order (the engine by WINDOW_PASS_SIZES, the canvas sampler made per size);
      CUDA events around each request give its service time.  With all requests arriving at once its latencies are the cumulative end
      times; with staggered arrivals they are a first-come-first-served queue over those service times, the arrivals placed at the
      times the stream arm of the same round reached their arrival steps.
Prints one JSON line: images/s, window-steps/s, latency (ms, and steps for the stream arms: mean and p95) per arm and arrival pattern, the schedule, and the
GPU's name and power limit read in the same run.

    python tools/gpu_windowed_stream_bench.py [--requests 16] [--rounds 2] [--slots 16,32] [--timesteps 100] [--seed 0]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE, OVERLAP = 128, 32
SIZES = [(128, 128), (200, 312), (256, 384), (160, 240)]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def stats(v):
    import numpy as np
    a = np.asarray(v, dtype=np.float64)
    return {"mean": float(a.mean()), "p95": float(np.percentile(a, 95))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--slots", default="16,32")
    ap.add_argument("--timesteps", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sr3_b200
    from sr3_b200 import _native
    assert torch.cuda.is_available(), "this measurement needs an H100"
    T = args.timesteps
    sched = {"schedule": "linear", "n_timestep": T, "linear_start": 1e-6, "linear_end": 1e-2}
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET), "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                     "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    name, limit = smi("name,power.limit")

    rng = np.random.default_rng(args.seed)
    sizes = [SIZES[i] for i in rng.integers(0, len(SIZES), size=args.requests)]
    g = torch.Generator().manual_seed(args.seed)
    reqs = [((torch.rand(3, H, W, generator=g) * 2 - 1).cuda(), torch.randn(3, H, W, generator=g).cuda()) for H, W in sizes]
    windows = [len(_native.window_grid(H, IMAGE, OVERLAP)) * len(_native.window_grid(W, IMAGE, OVERLAP)) for H, W in sizes]
    slot_counts = [int(v) for v in args.slots.split(",")]
    # staggered: Poisson arrivals (in steps) at about 3/4 of the smallest stream's window capacity
    rate = 0.75 * min(slot_counts) / (T * float(np.mean(windows)))
    stagger = np.ceil(np.cumsum(rng.exponential(1.0 / rate, size=args.requests))).astype(int).tolist()
    stagger = [a - stagger[0] for a in stagger]
    patterns = {"all_at_once": [0] * args.requests, "staggered": stagger}

    def stream_arm(slots, arrivals):
        plan = list(_native.windowed_stream_plan(zip(arrivals, windows), slots, T))
        s = _native.WindowedStreamSampler(net._engine(slots, IMAGE, IMAGE), 7, OVERLAP, OVERLAP)
        steps = max(f for _, _, f in plan)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        ids = {}
        torch.cuda.synchronize()
        ev[0].record()
        for k in range(steps):
            for n, (sl, a, _) in enumerate(plan):
                if a == k:
                    ids[n] = s.admit(sl, reqs[n][0], reqs[n][1], n)
            s.step()
            ev[k + 1].record()
            for n, (_, _, f) in enumerate(plan):
                if f == k + 1:
                    s.retire(ids[n])
        torch.cuda.synchronize()
        at = [0.0] + [ev[0].elapsed_time(e) for e in ev[1:]]
        lat_ms = [at[f] - at[arr] for (_, _, f), arr in zip(plan, arrivals)]
        lat_steps = [f - arr for (_, _, f), arr in zip(plan, arrivals)]
        return at[-1], lat_ms, lat_steps, [at[a] for a in arrivals]

    def baseline_arm(arrivals_ms):
        e0 = torch.cuda.Event(enable_timing=True)
        ends = [torch.cuda.Event(enable_timing=True) for _ in reqs]
        torch.cuda.synchronize()
        e0.record()
        for n, (c, x) in enumerate(reqs):
            img = net.super_resolution_windowed(c[None], window=(IMAGE, IMAGE), overlap=OVERLAP, x_T=x[None], seed=7, first_index=n)
            ends[n].record()
        torch.cuda.synchronize()
        assert torch.isfinite(img).all()
        end = [e0.elapsed_time(e) for e in ends]
        service = [end[0]] + [b - a for a, b in zip(end, end[1:])]
        lat, free = [], 0.0
        for a, sv in zip(arrivals_ms, service):
            free = max(free, a) + sv
            lat.append(free - a)
        return end[-1], lat, service

    # warm-up: every engine, every canvas size's sampler graph, every stream
    for slots in slot_counts:
        stream_arm(slots, [0] * min(4, args.requests))
    baseline_arm([0.0] * args.requests)

    total_ws = sum(windows) * T
    res = {p: {"stream_%d" % s: [] for s in slot_counts} for p in patterns}
    for p in patterns:
        res[p]["per_request"] = []
    for _ in range(args.rounds):
        for p, arrivals in patterns.items():
            arr_ms = None
            for slots in slot_counts:
                total, lat_ms, lat_steps, a_ms = stream_arm(slots, arrivals)
                res[p]["stream_%d" % slots].append((total, lat_ms, lat_steps))
                if arr_ms is None:
                    arr_ms = a_ms
            total, lat_ms, service = baseline_arm(arr_ms)
            res[p]["per_request"].append((total, lat_ms, None))
    sm_clock, power = smi("clocks.sm,power.draw")

    out = {"config": "16->128 (sr_sr3_16_128) bf16, window %dx%d, overlap %d, linear schedule n_timestep = %d" % (IMAGE, IMAGE, OVERLAP, T),
           "gpu": {"name": name, "power_limit": limit, "sm_clock_after": sm_clock, "power_draw_after": power},
           "requests": args.requests, "sizes": ["%dx%d" % s for s in sizes], "windows": windows, "window_steps": total_ws,
           "staggered_arrival_steps": stagger, "rounds": args.rounds, "arms": {}}
    for p in patterns:
        out["arms"][p] = {}
        for arm, runs in res[p].items():
            # the median round by total time
            runs = sorted(runs, key=lambda r: r[0])
            total, lat_ms, lat_steps = runs[len(runs) // 2]
            d = {"total_ms": total, "total_ms_rounds": [r[0] for r in res[p][arm]], "images_per_s": args.requests / total * 1e3,
                 "window_steps_per_s": total_ws / total * 1e3, "latency_ms": stats(lat_ms)}
            if lat_steps is not None:
                d["latency_steps"] = stats(lat_steps)
            out["arms"][p][arm] = d
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Continuous batching (GaussianDiffusion.super_resolution_stream: one-window requests on sr3_wstream_*) on the 16->128 config at
128x128 with 16 slots.  Prints one JSON line:
  * steady-state ms per step with every slot busy, the stream (gather + engine step graph + means + merge) against sr3_p_sample_steps
    (the lockstep sampler) on the same engine, the two arms alternated round by round (CUDA events around K steps; median and min..max);
  * request latency under Poisson arrivals at several loads for two policies, in steps from the deterministic plans (the lockstep policy
    starts a batch when the previous one ends, with the requests waiting at that moment; the continuous one is _native.stream_plan) and
    in seconds at the measured ms per step of each arm;
  * the GPU's name, power limit and maximum SM clock, and the SM clock and power draw observed right after the timed rounds.

    python tools/gpu_stream_bench.py [--steps 50] [--warmup 5] [--rounds 5] [--loads 0.25,0.5,0.75,0.9] [--requests 2000]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE, SLOTS = 128, 16


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def spread(v):
    return {"median_ms_per_step": statistics.median(v), "min": min(v), "max": max(v), "rounds": len(v)}


def poisson_arrivals(rate, n, seed):
    """Integer arrival steps (a request arriving during step k - 1 waits for step k) of n requests at `rate` requests per step."""
    import numpy as np
    t = np.cumsum(np.random.default_rng(seed).exponential(1.0 / rate, size=n))
    return [int(math.ceil(v)) for v in t]


def lockstep_latencies(arrivals, slots, T):
    """A batch of up to `slots` waiting requests starts when the previous batch ends (or at the next arrival when none waits)."""
    out, i, free = [], 0, 0
    while i < len(arrivals):
        start = max(free, arrivals[i])
        j = i
        while j < len(arrivals) and j - i < slots and arrivals[j] <= start:
            j += 1
        out += [start + T - a for a in arrivals[i:j]]
        i, free = j, start + T
    return out


def summary(lat, ms):
    import numpy as np
    a = np.asarray(lat, dtype=np.float64)
    p = {"mean": float(a.mean()), "p50": float(np.percentile(a, 50)), "p95": float(np.percentile(a, 95)), "max": float(a.max())}
    return {"steps": p, "seconds": {k: v * ms / 1000.0 for k, v in p.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loads", default="0.25,0.5,0.75,0.9")
    ap.add_argument("--requests", type=int, default=2000)
    args = ap.parse_args()
    import torch
    import sr3_b200
    from sr3_b200 import _native
    assert torch.cuda.is_available(), "this measurement needs an H100"
    T = SCHED["n_timestep"]
    assert args.warmup + args.steps <= T
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET), "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    name, limit, max_clock = smi("name,power.limit,clocks.max.sm")
    g = torch.Generator().manual_seed(3)
    cond = (torch.rand(SLOTS, 3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda()
    x_T = torch.randn(SLOTS, 3, IMAGE, IMAGE, generator=g).cuda()
    eng = net._engine(SLOTS, IMAGE, IMAGE)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def lockstep():
        eng.loop_begin(cond, x_T, 7, 0)
        eng.steps(T - 1, args.warmup)
        torch.cuda.synchronize()
        e0.record()
        eng.steps(T - 1 - args.warmup, args.steps)
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(eng.read_state()).all()
        return e0.elapsed_time(e1) / args.steps

    def stream():
        s = _native.WindowedStreamSampler(eng, 7, 0, 0)
        for k in range(SLOTS):
            s.admit([k], cond[k], x_T[k], k)
        s.step(args.warmup)
        torch.cuda.synchronize()
        e0.record()
        s.step(args.steps)
        e1.record()
        torch.cuda.synchronize()
        assert s.slot_state()[2] == [1] * SLOTS
        assert torch.isfinite(eng.read_state()).all()
        return e0.elapsed_time(e1) / args.steps

    lock_ms, stream_ms = [], []
    for _ in range(args.rounds):
        lock_ms.append(lockstep())
        stream_ms.append(stream())
    sm_clock, power = smi("clocks.sm,power.draw")
    lm, sm = statistics.median(lock_ms), statistics.median(stream_ms)
    out = {"config": "16->128 (sr_sr3_16_128) at 128x128, %d slots, T = %d" % (SLOTS, T),
           "gpu": {"name": name, "power_limit": limit, "max_sm_clock": max_clock, "sm_clock_after": sm_clock, "power_draw_after": power},
           "steps": args.steps, "warmup": args.warmup,
           "lockstep": spread(lock_ms), "stream": spread(stream_ms), "stream_over_lockstep": sm / lm, "latency": []}
    for load in [float(v) for v in args.loads.split(",")]:
        arrivals = poisson_arrivals(load * SLOTS / T, args.requests, 11)
        cont = [f - a for (_, _, f), a in zip(_native.stream_plan(arrivals, SLOTS, T), arrivals)]
        out["latency"].append({"load": load, "requests": args.requests, "lockstep": summary(lockstep_latencies(arrivals, SLOTS, T), lm),
                               "continuous": summary(cont, sm)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()

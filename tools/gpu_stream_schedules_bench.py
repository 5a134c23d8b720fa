"""Continuous batching with per-request noise schedules (sr3_wstream_add_schedule / sr3_wstream_admit_scheduled) on the 16->128 config of
bench.py in bf16: 128x128 requests, 16 slots, a two-tier mix drawn from a seed -- a quality tier on the module's 2000-step linear schedule
and a preview tier on a 100-step linear schedule -- sharing the batch.  Requests arrive as a Poisson process at a given load (the share
of slot-steps the traffic asks for) and are driven through WindowedStreamSampler exactly as windowed_stream_plan says, one step per plan
step; a CUDA event after every step gives each request's latency from the start of its arrival step to the end of its last step.
Prints one JSON line: ms per stream step (median, min and max over all steps), per-tier latency in steps and ms (mean, p50, p95, max),
images/s over the whole run, and the GPU's name and power limit, the SM clock and power draw read in the same run.

    python tools/gpu_stream_schedules_bench.py [--requests 48] [--quality-share 0.25] [--load 0.75] [--preview-steps 100] [--seed 0]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

QUALITY = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE, SLOTS = 128, 16


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def stats(v):
    import numpy as np
    a = np.asarray(v, dtype=np.float64)
    return {"mean": float(a.mean()), "p50": float(np.percentile(a, 50)), "p95": float(np.percentile(a, 95)), "max": float(a.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--quality-share", type=float, default=0.25)
    ap.add_argument("--load", type=float, default=0.75)
    ap.add_argument("--preview-steps", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sr3_b200
    from sr3_b200 import _native
    from sr3_b200.model.sr3_modules.diffusion import noise_schedule_buffers
    assert torch.cuda.is_available(), "this measurement needs an H100"
    preview = dict(QUALITY, n_timestep=args.preview_steps)
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                     "beta_schedule": {"train": dict(QUALITY), "val": dict(QUALITY)},
                     "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(QUALITY, "cuda")
    net.eval()
    name, limit = smi("name,power.limit")

    rng = np.random.default_rng(args.seed)
    tier = (rng.random(args.requests) < args.quality_share).astype(int)       # 1: quality (module schedule), 0: preview
    steps = [QUALITY["n_timestep"] if q else preview["n_timestep"] for q in tier]
    rate = args.load * SLOTS / float(np.mean(steps))                             # requests per step
    arrivals = np.ceil(np.cumsum(rng.exponential(1.0 / rate, size=args.requests))).astype(int)
    arrivals = (arrivals - arrivals[0]).tolist()
    g = torch.Generator().manual_seed(args.seed)
    reqs = [((torch.rand(3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda(), torch.randn(3, IMAGE, IMAGE, generator=g).cuda())
            for _ in range(args.requests)]
    plan = list(_native.windowed_stream_plan(zip(arrivals, [1] * args.requests, steps), SLOTS, QUALITY["n_timestep"]))
    n_steps = max(f for _, _, f in plan)

    eng = net._engine(SLOTS, IMAGE, IMAGE)

    def run(plan, n_steps, quality):
        """Drive the stream through `plan`; request n samples on the module's schedule when quality[n], else on the preview schedule."""
        s = _native.WindowedStreamSampler(eng, 7, 0, 0)
        sid = s.add_schedule(*noise_schedule_buffers(preview))
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(n_steps + 1)]
        ids = {}
        torch.cuda.synchronize()
        ev[0].record()
        for k in range(n_steps):
            for n, (sl, a, _) in enumerate(plan):
                if a == k:
                    ids[n] = s.admit(sl, reqs[n][0], reqs[n][1], n, schedule=None if quality[n] else sid)
            s.step()
            ev[k + 1].record()
            for n, (_, _, f) in enumerate(plan):
                if f == k + 1:
                    s.retire(ids[n])
        torch.cuda.synchronize()
        return [0.0] + [ev[0].elapsed_time(e) for e in ev[1:]]

    # warm-up: the engine's step graph and the stream's kernels (which launch the same way whatever the schedules), two preview requests
    warm = list(_native.windowed_stream_plan([(0, 1, preview["n_timestep"])] * 2, SLOTS, QUALITY["n_timestep"]))
    run(warm, preview["n_timestep"], [0, 0])
    at = run(plan, n_steps, tier)
    sm_clock, power = smi("clocks.sm,power.draw")
    per_step = np.diff(np.asarray(at))
    ms_step = float(np.median(per_step))
    out = {"config": "16->128 (sr_sr3_16_128) bf16, %dx%d requests, %d slots; quality tier: the module's linear schedule n_timestep = %d, "
                     "preview tier: linear n_timestep = %d" % (IMAGE, IMAGE, SLOTS, QUALITY["n_timestep"], preview["n_timestep"]),
           "gpu": {"name": name, "power_limit": limit, "sm_clock_after": sm_clock, "power_draw_after": power},
           "requests": args.requests, "quality_requests": int(tier.sum()), "preview_requests": int(len(tier) - tier.sum()),
           "load": args.load, "stream_steps": n_steps, "total_ms": at[-1], "images_per_s": args.requests / at[-1] * 1e3,
           "ms_per_stream_step": {"median": ms_step, "min": float(per_step.min()), "max": float(per_step.max())}, "tiers": {}}
    for label, q in (("quality", 1), ("preview", 0)):
        idx = [n for n in range(args.requests) if tier[n] == q]
        if idx:
            out["tiers"][label] = {"steps_per_request": steps[idx[0]],
                                   "latency_steps": stats([plan[n][2] - arrivals[n] for n in idx]),
                                   "latency_ms": stats([at[plan[n][2]] - at[arrivals[n]] for n in idx])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

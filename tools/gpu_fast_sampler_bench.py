"""Wall time to a finished batch with the few-step samplers (DESIGN.md 3.11) on the 16->128 config of bench.py in bf16, batch 16:
DDPM over the trained 2000 steps, DDIM at 50 and 100 steps (eta = 0) and DPM-Solver++(2M) at 20 and 25 steps, each through
super_resolution.  Every sampler is warmed up once (engine, canvas, graphs), then timed `--reps` times with a host clock around the call
and a device synchronise; ms per step = wall time / steps, so the solver merge's cost per step shows against DDIM's.  The DPM-Solver++
canvas step is also split into gather / engine / merge with CUDA events (WindowedSampler.profile_step), next to the posterior-sample
merge of the same canvas.  Prints one JSON line with the GPU's name and power limit and the SM clock read in the same run.

    python tools/gpu_fast_sampler_bench.py [--reps 3] [--ddpm-reps 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.2)
IMAGE, BATCH = 128, 16
SAMPLERS = [("ddpm_2000", None, 2000), ("ddim_100", {"sampler": "ddim", "steps": 100, "eta": 0.0}, 100),
            ("ddim_50", {"sampler": "ddim", "steps": 50, "eta": 0.0}, 50), ("dpmpp_2m_25", {"sampler": "dpmpp_2m", "steps": 25}, 25),
            ("dpmpp_2m_20", {"sampler": "dpmpp_2m", "steps": 20}, 20)]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ddpm-reps", type=int, default=1)
    args = ap.parse_args()
    import torch
    import sr3_b200
    from sr3_b200 import _native
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                     "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    name, limit = smi("name,power.limit")
    g = torch.Generator().manual_seed(1)
    cond = (torch.rand(BATCH, 3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda()
    x_T = torch.randn(BATCH, 3, IMAGE, IMAGE, generator=g).cuda()
    res = {}
    for label, spec, steps in SAMPLERS:
        reps = args.ddpm_reps if spec is None else args.reps
        # warm-up: engine / canvas creation and graph capture (a short DDIM stands in for the 2000-step loop)
        net.super_resolution(cond, x_T=x_T, seed=1, sampler=spec or {"sampler": "ddim", "steps": 2, "eta": 0.0})
        torch.cuda.synchronize()
        times = []
        for r in range(reps):
            t0 = time.perf_counter()
            out = net.super_resolution(cond, x_T=x_T, seed=1 + r, sampler=spec)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        assert torch.isfinite(out).all()
        best = min(times)
        res[label] = {"steps": steps, "s_per_batch": [round(t, 4) for t in times], "best_s": round(best, 4),
                      "ms_per_step": round(1e3 * best / steps, 4), "images_per_s": round(BATCH / best, 2)}
    # one canvas step split into its launches: the solver merge against the posterior-sample merge of the same canvas
    canvas = net._windowed_sampler(BATCH, IMAGE, IMAGE, (IMAGE, IMAGE), 0)
    canvas.begin(cond, x_T, 1, 0)
    prof = {"posterior_merge": canvas.profile_step(1, reps=20)}
    tables = net._sampler_tables(("dpmpp_2m", 25, None))
    with canvas.engine.sampling_on(tables):
        canvas.set_solver(tables[2])
        try:
            prof["solver_merge"] = canvas.profile_step(10, reps=20)
        finally:
            canvas.set_solver(None)
    clock = smi("clocks.sm")[0]
    print(json.dumps({"gpu": name, "power_limit": limit, "sm_clock_after": clock, "config": "sr_sr3_16_128 bf16 B=16 128x128",
                      "samplers": res, "canvas_step_ms": prof}))


if __name__ == "__main__":
    main()

"""Speed of windowed sampling (GaussianDiffusion.super_resolution_windowed) on the 16->128 config with 128x128 windows, one image per canvas.
Prints one JSON line:
  * per canvas: windows per step, windows per engine pass, ms per canvas step (state resident on the device, CUDA events around K graph
    launches, `rounds` repetitions: median and min..max), and the device time of the gathers, the engine passes and the merge in an eager step
    (sr3_windowed_profile_step);
  * 128x128 (one window) against the plain sampler at 128x128, and 512x512 windowed against 512x512 in one piece, the two arms of each
    pair alternated round by round;
  * the GPU's name, power limit and maximum SM clock, and the SM clock and power draw observed right after the timed rounds.

    python tools/gpu_windowed_bench.py [--steps 20] [--warmup 3] [--rounds 5] [--canvases 128x128,200x312,512x512,720x1280]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE = 128
PLAIN = {(128, 128), (512, 512)}          # canvases also sampled in one piece


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def inputs(H, W):
    import torch
    g = torch.Generator().manual_seed(3)
    return (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda(), torch.randn(1, 3, H, W, generator=g).cuda()


def timed(obj, begin, K, warm):
    """ms per step of K steps after `warm` warm-up steps, from a fresh state."""
    import torch
    T = SCHED["n_timestep"]
    begin()
    obj.steps(T - 1, warm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    obj.steps(T - 1 - warm, K)
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(obj.read_state()).all(), "sampler state is not finite"
    return e0.elapsed_time(e1) / K


def spread(v):
    return {"median_ms_per_step": statistics.median(v), "min": min(v), "max": max(v), "rounds": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--canvases", default="128x128,200x312,512x512,720x1280")
    args = ap.parse_args()
    import torch
    import sr3_b200
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET), "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    name, limit, max_clock = smi("name,power.limit,clocks.max.sm")
    out = {"config": "16->128 (sr_sr3_16_128), window 128x128, overlap 32, one image per canvas",
           "gpu": {"name": name, "power_limit": limit, "max_sm_clock": max_clock}, "canvases": []}
    for H, W in [tuple(int(v) for v in s.split("x")) for s in args.canvases.split(",")]:
        cond, x_T = inputs(H, W)
        sampler = net._windowed_sampler(1, H, W)
        oy, ox, _, _ = sampler.grid()
        plain = net._engine(1, H, W) if (H, W) in PLAIN else None
        win_ms, plain_ms = [], []
        for _ in range(args.rounds):                     # the two arms alternate
            win_ms.append(timed(sampler, lambda: sampler.begin(cond, x_T, 1234, 0), args.steps, args.warmup))
            if plain is not None:
                plain_ms.append(timed(plain, lambda: plain.loop_begin(cond, x_T, seed=1234, first_index=0), args.steps, args.warmup))
        clock, power = smi("clocks.sm,power.draw")
        sampler.begin(cond, x_T, 1234, 0)
        prof = sampler.profile_step(SCHED["n_timestep"] // 2, reps=3)
        total = sum(prof.values())
        row = {"canvas": f"{H}x{W}", "windows_per_step": len(oy) * len(ox), "windows_per_pass": sampler.engine.batch, "windowed": spread(win_ms),
               "eager_step_ms": prof, "gather_share": prof["gather"] / total, "merge_share": prof["merge"] / total,
               "observed_sm_clock": clock, "observed_power_draw": power}
        if plain is not None:
            row["in_one_piece"] = spread(plain_ms)
        out["canvases"].append(row)
        net._windowed = None
        net.denoise_fn._engines.clear()                  # one canvas's workspace at a time
        net.denoise_fn._engine_versions.clear()
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

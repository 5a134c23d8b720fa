"""Training speed and memory of the 16->128 config (sr_sr3_16_128: image_size 128, attention on the 16x16 level of a 128x128 image) at
other image sizes.  The attention layers stay on the level image_size placed them on: 256 tokens per image at 128x128, 512 at 128x256 and
1024 at 256x256 (the training plan always runs S = q k^T, the row softmax and P v as separate launches, and keeps S, P, dS and bf16 dS for
the backward: nz * tokens^2 each).  Prints one JSON line:
  * per size, at a fixed batch: training steps/s of DDPM.optimize_parameters' arithmetic (p_losses -> sum / (b c h w) -> backward ->
    FusedAdam), CUDA events around K steps after W warm-up steps;
  * the plan's device bytes (sr3_engine_workspace_bytes), torch's peak allocation (parameters, gradients, Adam state, inputs) and the
    device memory in use after the timed steps (total - free);
  * the GPU's name, power limit and clocks, read in the same run.

    python tools/gpu_train_sizes_bench.py [--batch 8] [--steps 10] [--warmup 3] [--sizes 128x128,128x256,256x256]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE = 128


def make_opt():
    return {"phase": "train", "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                      "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                      "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    vals = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return dict(zip(("name", "power_limit", "max_sm_clock", "sm_clock", "mem_clock"), vals))


def training(net, opt, B, H, W, K, warm):
    import torch
    g = torch.Generator().manual_seed(3)
    hr = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).cuda()
    sr = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).cuda()
    torch.cuda.reset_peak_memory_stats()

    def step():
        opt.zero_grad()
        l = net.p_losses({"HR": hr, "SR": sr})
        (l.sum() / (B * 3 * H * W)).backward()
        opt.step()
        return l

    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        l = step()
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(l).all(), "training loss is not finite"
    ms = e0.elapsed_time(e1) / K
    free, total = torch.cuda.mem_get_info()
    eng = next(iter(net.denoise_fn._engines.values()))
    return {"size": f"{H}x{W}", "batch": B, "attention_tokens": (H // 8) * (W // 8), "ms_per_step": ms, "steps_per_s": 1e3 / ms,
            "images_per_s": B * 1e3 / ms, "plan_bytes": eng.workspace_bytes(), "torch_peak_bytes": torch.cuda.max_memory_allocated(),
            "device_used_bytes": total - free}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="128x128,128x256,256x256")
    args = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    import numpy as np
    import torch
    import sr3_b200
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    np.random.seed(0)
    net = sr3_b200.define_G(make_opt()).cuda()
    net.set_loss("cuda")
    net.set_new_noise_schedule(SCHED, "cuda")
    net.train()
    opt = sr3_b200.FusedAdam(list(net.parameters()), lr=1e-4)
    out = {"config": "16->128 (sr_sr3_16_128), attention on the 16x16 level of image_size 128", "gpu": gpu_info(), "training": []}
    for H, W in sizes:
        out["training"].append(training(net, opt, args.batch, H, W, args.steps, args.warmup))
        net.denoise_fn._engines.clear()                  # one size's plan at a time
        net.denoise_fn._engine_versions.clear()
        torch.cuda.empty_cache()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

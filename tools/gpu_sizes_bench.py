"""Speed of the 16->128 config (sr_sr3_16_128: image_size 128, attention on the 16x16 level of a 128x128 image) at other image sizes.
The attention layers stay on the level image_size placed them on, so their token count grows with the image: 256 tokens at 128x128
(attn_kernel), 512 at 128x256, 1024 at 256x256 and 4096 at 512x512 (attn_long_kernel, the streaming-softmax form: one launch as well).
Prints one JSON line:
  * sampling steps/s per size at a fixed batch (sampler state resident on the device, CUDA events around K steps);
  * the per-launch time split of one eager step (sr3_engine_profile_step), summed by launch kind, with the attention core (the fused launches;
    in a plan that does not fuse, the S and P v tile launches and the softmax) also summed on its own, and the plan's device bytes;
  * the GPU's name, power limit and maximum SM clock, read in the same run.

    python tools/gpu_sizes_bench.py [--batch 4] [--steps 20] [--warmup 3] [--sizes 128x128,128x256,256x256,512x512]
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
KINDS = {0: "tile_kernel", 1: "groupnorm_apply", 2: "cast", 3: "softmax", 4: "other", 5: "attention"}


def make_opt():
    return {"phase": "val", "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                      "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                      "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def sampling(net, B, H, W, K, warm):
    import torch
    eng = net.denoise_fn.engine(B, conditional=True, channels=3, height=H, width=W)
    g = torch.Generator().manual_seed(3)
    cond = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).cuda()
    xT = torch.randn(B, 3, H, W, generator=g).cuda()
    T = SCHED["n_timestep"]
    eng.loop_begin(cond, xT, seed=1234, first_index=0)
    eng.steps(T - 1, warm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.steps(T - 1 - warm, K)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    assert torch.isfinite(eng.read_state()).all(), "sampler state is not finite"
    prof = eng.profile_step(T // 2, reps=3)
    sched = eng.tile_schedules()
    by_kind, attn = {}, 0.0
    for i, (k, t, _, _) in enumerate(prof):
        by_kind[KINDS.get(k, str(k))] = by_kind.get(KINDS.get(k, str(k)), 0.0) + t
        # the attention core: the fused kernel, the softmax, and the tile launches over token rows (S = q k^T and P v: one output row)
        if k in (3, 5) or (k == 0 and sched[i] is not None and sched[i]["out_hwc"][0] == 1):
            attn += t
    return {"size": f"{H}x{W}", "batch": B, "attention_tokens": (H // 8) * (W // 8), "ms_per_step": ms, "steps_per_s": 1e3 / ms,
            "images_per_s": B * 1e3 / ms, "launches_per_step": eng.launches_per_step(), "workspace_bytes": eng.workspace_bytes(), "eager_step_ms_by_kind": by_kind,
            "eager_step_attention_core_ms": attn, "eager_step_ms_total": sum(t for _, t, _, _ in prof)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="128x128,128x256,256x256,512x512")
    args = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    import torch
    import sr3_b200
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt()).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    out = {"config": "16->128 (sr_sr3_16_128), attention on the 16x16 level of image_size 128", "gpu": gpu_info(), "sampling": []}
    for H, W in sizes:
        out["sampling"].append(sampling(net, args.batch, H, W, args.steps, args.warmup))
        net.denoise_fn._engines.clear()                  # one size's workspace at a time
        net.denoise_fn._engine_versions.clear()
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

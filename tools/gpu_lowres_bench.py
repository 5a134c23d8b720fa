"""Speed of a UNet whose lowest level is 4x4: the 16->64 config (channel_multiplier (1, 2, 4, 8, 8): 64 -> 32 -> 16 -> 8 -> 4, attention at
16x16 and in the 4x4 middle block, two ResnetBlocks per level).  Prints one JSON line:
  * sampling steps/s at batch 16 and batch 1 (sampler state resident on the device, CUDA events around K steps);
  * the per-launch time split of one eager step at both batches (sr3_engine_profile_step), summed by launch kind, and every tile-kernel
    launch in plan order;
  * the training step (forward + backward + Adam) at 8 images;
  * the GPU's name and power limit, read in the same run.

    python tools/gpu_lowres_bench.py [--steps 50] [--warmup 5] [--train-steps 10]
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
IMAGE = 64
KINDS = {0: "tile_kernel", 1: "groupnorm_apply", 2: "cast", 3: "softmax", 4: "other", 5: "attention"}


def make_opt(phase):
    return {"phase": phase, "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                      "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                      "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def sampling(net, B, K, W):
    import torch
    eng = net.denoise_fn.engine(B, conditional=True, channels=3)
    g = torch.Generator().manual_seed(3)
    cond = (torch.rand(B, 3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda()
    xT = torch.randn(B, 3, IMAGE, IMAGE, generator=g).cuda()
    T = SCHED["n_timestep"]
    eng.loop_begin(cond, xT, seed=1234, first_index=0)
    eng.steps(T - 1, W)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.steps(T - 1 - W, K)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    assert torch.isfinite(eng.read_state()).all(), "sampler state is not finite"
    # one eager step, every launch timed with CUDA events (plan order)
    prof = eng.profile_step(T // 2, reps=5)
    by_kind = {}
    for k, t, _, _ in prof:
        by_kind[KINDS.get(k, str(k))] = by_kind.get(KINDS.get(k, str(k)), 0.0) + t
    return {"batch": B, "ms_per_step": ms, "steps_per_s": 1e3 / ms, "launches_per_step": eng.launches_per_step(),
            "eager_step_ms_by_kind": by_kind, "eager_step_ms_total": sum(t for _, t, _, _ in prof),
            "tile_kernel_launches_ms": [round(t, 4) for k, t, _, _ in prof if k == 0]}


def training(B, K, W):
    import torch
    import sr3_b200
    from sr3_b200 import parallel
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt("train")).cuda()
    net.set_loss("cuda")
    net.set_new_noise_schedule(SCHED, "cuda")
    net.train()
    g = torch.Generator().manual_seed(5)
    hr = (torch.rand(B, 3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda()
    sr = (torch.rand(B, 3, IMAGE, IMAGE, generator=g) * 2 - 1).cuda()
    tr = parallel.DataParallelTrainer(net, lr=1e-4)
    losses = [tr.step(hr, sr, global_batch=B) for _ in range(W)]
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        losses.append(tr.step(hr, sr, global_batch=B))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    assert all(l == l for l in losses), "training loss is not finite"
    return {"batch": B, "ms_per_step": ms, "steps_per_s": 1e3 / ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import sr3_b200
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt("val")).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    out = {"config": "16->64, channel_multiplier (1, 2, 4, 8, 8), attn_res [16], res_blocks 2 (lowest level 4x4)", "gpu": gpu_info(),
           "sampling": [sampling(net, B, args.steps, args.warmup) for B in (16, 1)]}
    del net
    torch.cuda.empty_cache()
    out["training"] = training(8, args.train_steps, 3)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

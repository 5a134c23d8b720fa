"""Cost of the differentiable denoiser on the 16->128 config (sr_sr3_16_128) at 128x128, batch 8.  Prints one JSON line with ms per
iteration (CUDA events around K iterations after W warm-up iterations) of:
  * a p_losses training step: p_losses -> backward (the native loss gradient);
  * the autograd forward plus backward of denoise_fn(cat(SR, x_noisy), gamma) with a summed L1 loss on eps, parameters only
    (set_differentiable(True), no dx);
  * the same with x requiring grad (dx computed as well);
and the GPU's name, power limit and clocks, read in the same run.  The first two run the same plan and the same backward apart from how
the upstream gradient is loaded.

    python tools/gpu_unet_grad_bench.py [--batch 8] [--size 128] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_train_sizes_bench import SCHED, gpu_info, make_opt  # noqa: E402


def timed(fn, K, warm):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import sr3_b200
    assert torch.cuda.is_available(), "this measurement needs an H100"
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt()).cuda()
    net.set_loss("cuda")
    net.set_new_noise_schedule(SCHED, "cuda")
    net.train()
    dn = net.denoise_fn
    B, R = args.batch, args.size
    g = torch.Generator().manual_seed(3)
    hr = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).cuda()
    sr = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).cuda()
    noise = torch.randn(B, 3, R, R, generator=g).cuda()
    gamma = torch.rand(B, generator=g).cuda() * 0.5 + 0.5
    x_in = torch.cat([sr, net.q_sample(hr, gamma.view(-1, 1, 1, 1), noise)], dim=1)

    def zero():
        for p in dn.parameters():
            p.grad = None

    def p_losses_step():
        zero()
        net.p_losses({"HR": hr, "SR": sr}, noise=noise, gamma=gamma).backward()

    def autograd_step(want_dx):
        zero()
        x = x_in.detach().requires_grad_(want_dx)
        (dn(x, gamma.view(B, 1)) - noise).abs().sum().backward()

    dn.set_differentiable(True)
    out = {"config": "16->128 (sr_sr3_16_128)", "batch": B, "size": f"{R}x{R}", "gpu": gpu_info(), "ms_per_iteration": {}}
    res = out["ms_per_iteration"]
    for rep in range(2):                              # alternating, twice: the spread between repetitions is the noise
        res.setdefault("p_losses_step", []).append(timed(p_losses_step, args.steps, args.warmup))
        res.setdefault("unet_autograd_no_dx", []).append(timed(lambda: autograd_step(False), args.steps, args.warmup))
        res.setdefault("unet_autograd_with_dx", []).append(timed(lambda: autograd_step(True), args.steps, args.warmup))
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

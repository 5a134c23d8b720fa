"""The attention core alone, fused against unfused, at the attention shapes the supported configs produce above 256 tokens per image:
(tokens, C) = (512, 512) 16->128 at 128x256, (1024, 512) at 256x256, (4096, 512) at 512x512, (1024, 1024) the 32x32 mid block of 64->512,
(16384, 512) 16->128 at 1024x1024 (one image).  Both paths run on the same random bf16 operands through the library's test hooks:
  fused    sr3_test_attention: attn_long_kernel, one launch
  unfused  sr3_test_attention_unfused: S = q k^T on the tile kernel, softmax_kernel, P v on the tile kernel
alternated in one process, CUDA events around each call (a call ends in a stream synchronise, inside the timed window for both).
Prints one JSON line: ms and algorithmic TFLOP/s (4 nz Lt^2 C FLOP) per shape and path, their relative L2 difference, and the GPU's name,
power limit and maximum SM clock read in the same run.

    python tools/gpu_attention_bench.py [--nz 4] [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (tokens per image, C, attention batches; None = --nz)
SHAPES = [(512, 512, None), (1024, 512, None), (4096, 512, None), (1024, 1024, None), (16384, 512, 1)]


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nz", type=int, default=4)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from sr3_b200 import _native
    assert torch.cuda.is_available(), "this measurement needs an H100"
    out = {"gpu": gpu_info(), "reps": args.reps, "shapes": []}
    for Lt, C, nz in SHAPES:
        nz = nz or args.nz
        g = torch.Generator().manual_seed(Lt + C)
        qk = torch.cat([2.0 * torch.randn(nz * Lt, C, generator=g), torch.randn(nz * Lt, C, generator=g)], 1).bfloat16().cuda()
        vT = torch.randn(nz * C, Lt, generator=g).bfloat16().cuda()
        paths = {"fused": lambda: _native.test_attention(qk, vT, nz, Lt, Lt, C),
                 "unfused": lambda: _native.test_attention_unfused(qk, vT, nz, Lt, Lt, C)[2]}
        ms, last = {k: [] for k in paths}, {}
        for r in range(args.warmup + args.reps):
            for k, fn in paths.items():
                t, last[k] = timed(fn)
                if r >= args.warmup:
                    ms[k].append(t)
        a, b = last["fused"].double(), last["unfused"].double()
        flop = 4.0 * nz * Lt * Lt * C
        row = {"tokens": Lt, "C": C, "nz": nz, "rel_l2_fused_vs_unfused": ((a - b).norm() / b.norm()).item()}
        for k, v in ms.items():
            v.sort()
            med = v[len(v) // 2]
            row[k] = {"ms_median": med, "ms_min": v[0], "ms_max": v[-1], "algorithmic_tflops": flop / (med * 1e-3) / 1e12}
        out["shapes"].append(row)
        del qk, vT, last
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

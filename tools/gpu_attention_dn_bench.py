"""attn_kernel per channel slice: the time of one launch at dn = 64, 128 and 256 output channels per CTA, at the attention shapes the
benchmarked engines run up to 256 tokens (C = 512): 16x16 images (256 tokens per attention batch) and 8x8 images two to a 128-token
batch, at batch 16 (16->128), 4 and 32 (unconditional 128x128).  Each (shape, dn) is timed through sr3_bench_attention: one captured
graph of --reps launches, CUDA events around it, the average per launch; --rounds rounds alternate the slices.  The outputs of the
slices must be bit-identical.  Prints one JSON line with the GPU's name, power limit and maximum SM clock read in the same run, the
CTA count and the median / min / max microseconds per slice, and the slice the library picks.

    python tools/gpu_attention_dn_bench.py [--reps 200] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C = 512
SHAPES = [(B, Lt, HW) for B in (16, 4, 32) for Lt, HW in ((256, 256), (128, 64))]
SLICES = (64, 128, 256)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    name, power, clock, cur = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "sm_clock_at_start": cur}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    from sr3_b200 import _native
    assert torch.cuda.is_available(), "this measurement needs an H100"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"gpu": gpu_info(), "sms": sms, "reps": args.reps, "rounds": args.rounds, "shapes": []}
    for B, Lt, HW in SHAPES:
        nz = B * HW // Lt
        g = torch.Generator().manual_seed(B + Lt)
        qk = torch.cat([2.0 * torch.randn(nz * Lt, C, generator=g), torch.randn(nz * Lt, C, generator=g)], 1).bfloat16().cuda()
        vT = torch.randn(nz * C, Lt, generator=g).bfloat16().cuda()
        us, outs = {dn: [] for dn in SLICES}, {}
        for _ in range(args.rounds):
            for dn in SLICES:
                ms, outs[dn] = _native.bench_attention(qk, vT, nz, Lt, HW, C, dn, args.reps)
                us[dn].append(ms * 1e3)
        row = {"batch": B, "tokens": Lt, "hw": HW, "nz": nz, "picked_dn": _native.attention_dn(nz, Lt, C),
               "bit_identical": all(torch.equal(outs[dn], outs[SLICES[0]]) for dn in SLICES)}
        for dn in SLICES:
            v = sorted(us[dn])
            row[f"dn{dn}"] = {"ctas": (Lt // 128) * (C // dn) * nz, "us_median": round(v[len(v) // 2], 2), "us_min": round(v[0], 2),
                              "us_max": round(v[-1], 2)}
        out["shapes"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

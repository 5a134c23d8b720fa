"""Cost of scoring a sampled batch (sr.py:216-217 for every image): sr3_b200.core.metrics.psnr_ssim on the device against the reference's
calculate_ssim (core/metrics.py:75-93: cv2.filter2D in float64, three identical calls per RGB image) on the host cores.  Prints one JSON line:
  * psnr_ssim per batch at 16x3x128x128 (16 -> 128) and 4x3x512x512 (64 -> 512): CUDA events around each call (every call ends in its
    device-to-host copy of the results), mean and median over --reps calls after --warmup;
  * the reference's calculate_ssim per image and per batch on the uint8 images of the same batch, imported from oracle/_ref when its
    core/metrics.py imports there (it needs cv2), else "not available";
  * the GPU's name, power limit and clock state, read in the same run.

    python tools/gpu_metrics_bench.py [--reps 50] [--warmup 5] [--ref-reps 3]
"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(16, 3, 128, 128), (4, 3, 512, 512)]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "not available"


def reference_metrics():
    path = os.path.join(ROOT, "oracle", "_ref", "core", "metrics.py")
    if not os.path.exists(path):
        return None, "oracle/_ref is absent"
    try:
        spec = importlib.util.spec_from_file_location("ref_core_metrics", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    except ImportError as e:
        return None, str(e)
    return mod, None


def batch(shape, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    hr = torch.rand(*shape, generator=g) * 2 - 1
    sr = (hr + torch.randn(*shape, generator=g) * 0.08).clamp(-1, 1)
    return sr.cuda(), hr.cuda()


def time_device(sr, hr, reps, warmup):
    import torch
    from sr3_b200.core import metrics
    for _ in range(warmup):
        metrics.psnr_ssim(sr, hr)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        metrics.psnr_ssim(sr, hr)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {"ms_per_batch_mean": statistics.fmean(ms), "ms_per_batch_median": statistics.median(ms), "reps": reps}


def time_reference(ref, sr, hr, reps):
    from sr3_b200.core import metrics
    imgs = [(metrics.tensor2img(sr[i]), metrics.tensor2img(hr[i])) for i in range(sr.shape[0])]
    ref.calculate_ssim(*imgs[0])                                      # warm: cv2's first call allocates
    per_image = []
    for _ in range(reps):
        for a, b in imgs:
            t0 = time.perf_counter()
            ref.calculate_ssim(a, b)
            per_image.append((time.perf_counter() - t0) * 1e3)
    med = statistics.median(per_image)
    return {"ms_per_image_median": med, "ms_per_batch": med * sr.shape[0], "host_cores": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import numpy as np
    from sr3_b200.core import metrics
    assert torch.cuda.is_available(), "this measurement needs an H100"
    ref, why = reference_metrics()
    out = {"gpu": smi("name,power.limit,clocks.max.sm"), "results": []}
    for k, shape in enumerate(SHAPES):
        sr, hr = batch(shape, k)
        r = {"shape": list(shape), "psnr_ssim": time_device(sr, hr, args.reps, args.warmup)}
        r["clock_after_timed_window"] = smi("clocks.sm,clocks_throttle_reasons.active")
        psnr, ssim = metrics.psnr_ssim(sr, hr)
        assert np.isfinite(psnr).all() and np.isfinite(ssim).all()
        r["mean_psnr_db"], r["mean_ssim"] = float(psnr.mean()), float(ssim.mean())
        if ref is None:
            r["reference_calculate_ssim"] = "not available (%s)" % why
        else:
            r["reference_calculate_ssim"] = time_reference(ref, sr, hr, args.ref_reps)
            r["speedup_vs_reference"] = r["reference_calculate_ssim"]["ms_per_batch"] / r["psnr_ssim"]["ms_per_batch_median"]
        out["results"].append(r)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

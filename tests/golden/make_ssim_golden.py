"""Generate tests/golden/sr3_ssim_golden.pt: what the UNMODIFIED reference's core/metrics.py (cv2.filter2D in float64) computes for
`ssim` / `calculate_ssim` (core/metrics.py:52-93) on a set of uint8 image pairs.  Run once where the reference and cv2 are installed:

    python tests/golden/make_ssim_golden.py [reference checkout]

Every pair is drawn from numpy.random.RandomState(seed) by `pair()` below (tests/test_ssim.py draws them the same way); the fixture keeps
the seeds, shapes, a sha256 of every pair (so a test knows it drew the same images), the raw arrays of the small pairs, and per case
either the reference's value (a float, nan, or None) or the message of the ValueError it raised.
"""
import hashlib
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SR3_REFERENCE", "/root/reference")

# name: (seed, shape1, shape2, kind, amplitude); kind "noisy": b = clip(a + uniform integer noise in [-amplitude, amplitude]),
# "same": b = a, "const": a and b constant (amplitude = b's value, a's is 200), "indep": b drawn independently of a.
CASES = {
    "noisy_128x128x3": (0, (128, 128, 3), (128, 128, 3), "noisy", 20),
    "noisy_512x512x3": (1, (512, 512, 3), (512, 512, 3), "noisy", 12),
    "gray_37x23": (2, (37, 23), (37, 23), "noisy", 30),
    "single_pixel_11x11x1": (3, (11, 11, 1), (11, 11, 1), "noisy", 25),
    "noisy_64x48x3": (4, (64, 48, 3), (64, 48, 3), "noisy", 40),
    "identical_96x80x3": (5, (96, 80, 3), (96, 80, 3), "same", 0),
    "constant_40x40x3": (6, (40, 40, 3), (40, 40, 3), "const", 37),
    "uncorrelated_64x64x3": (7, (64, 64, 3), (64, 64, 3), "indep", 0),
    "too_small_8x8x3": (8, (8, 8, 3), (8, 8, 3), "noisy", 20),
    "four_channels_32x32x4": (9, (32, 32, 4), (32, 32, 4), "noisy", 20),
    "shape_mismatch": (10, (16, 16, 3), (16, 17, 3), "indep", 0),
    "four_dims": (11, (2, 16, 16, 3), (2, 16, 16, 3), "noisy", 20),
}
SMALL = 64 * 64 * 4          # pairs up to this many elements per image are stored raw


def pair(seed, shape1, shape2, kind, amp):
    rs = np.random.RandomState(seed)
    if kind == "const":
        return np.full(shape1, 200, np.uint8), np.full(shape2, amp, np.uint8)
    a = rs.randint(0, 256, shape1).astype(np.uint8)
    if kind == "same":
        return a, a.copy()
    if kind == "indep":
        return a, rs.randint(0, 256, shape2).astype(np.uint8)
    return a, np.clip(a.astype(np.int32) + rs.randint(-amp, amp + 1, shape2), 0, 255).astype(np.uint8)


def digest(a, b):
    return hashlib.sha256(a.tobytes() + b.tobytes()).hexdigest()


def run(fn, a, b):
    """('value', float | nan | None) or ('error', message)."""
    try:
        v = fn(a, b)
    except ValueError as e:
        return "error", str(e)
    return "value", None if v is None else float(v)


def main(ref_root):
    sys.dont_write_bytecode = True
    import torch
    spec = importlib.util.spec_from_file_location("ref_core_metrics", os.path.join(ref_root, "core", "metrics.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)                       # imports cv2 and torchvision, as the reference does
    out = {}
    for name, case in CASES.items():
        a, b = pair(*case)
        seed, shape1, shape2, kind, amp = case
        rec = {"seed": seed, "shape1": shape1, "shape2": shape2, "kind": kind, "amplitude": amp, "sha256": digest(a, b),
               "calculate_ssim": run(ref.calculate_ssim, a, b)}
        if a.shape == b.shape and a.ndim in (2, 3):
            rec["ssim"] = run(ref.ssim, a, b)          # the raw metric as well (for the 4-channel case: the value calculate_ssim drops)
        if a.size <= SMALL:
            rec["a"], rec["b"] = torch.from_numpy(a.copy()), torch.from_numpy(b.copy())
        out[name] = rec
        print(name, rec["calculate_ssim"], rec.get("ssim"))
    torch.save(out, os.path.join(HERE, "sr3_ssim_golden.pt"))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else REF)

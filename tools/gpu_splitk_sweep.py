"""Single-conv timings of the low-resolution, long-K layers with and without global split-K (SR3_KSPLIT)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sr3_b200 import _native
torch.zeros(1).cuda()
SHAPES = {"8x8 512 B16": (16, 8, 8, 512, 512), "8x8 1024 B16": (16, 8, 8, 1024, 512), "8x8 512 B2": (2, 8, 8, 512, 512), "8x8 1024 B2": (2, 8, 8, 1024, 512),
          "16x16 512 B16": (16, 16, 16, 512, 512), "16x16 1024 B16": (16, 16, 16, 1024, 512), "32x32 256 B4": (4, 32, 32, 256, 256), "64x64 128 B2": (2, 64, 64, 128, 128),
          "16x16 512 B2": (2, 16, 16, 512, 512), "16x16 1024 B2": (2, 16, 16, 1024, 512), "16x16 512 B4": (4, 16, 16, 512, 512)}
KEYS = ("SR3_KSPLIT", "SR3_BLOCK_N", "SR3_TALL_BN", "SR3_TALL_MH")
def run(tag, shape, env=None, **kw):
    for k in KEYS:
        os.environ.pop(k, None)
    for k, v in (env or {}).items():
        os.environ[k] = str(v)
    B, H, W, ci, co = SHAPES[shape]
    try:
        ms = _native.bench_conv(B, H, W, ci, co, **kw)
    except Exception as e:
        print(shape, tag, "FAILED", e, flush=True)
        return
    gf = 2.0 * B * H * W * ci * co * 9 / 1e9
    print(f"{shape:14s} {tag:34s} {ms*1000:8.1f} us  {gf/ms:8.1f} TF/s", flush=True)
for shape in SHAPES:
    run("model (default)", shape)
    run("model, resid", shape, resid=True)
    run("no split-K", shape, {"SR3_KSPLIT": 1})
    run("no split-K, resid", shape, {"SR3_KSPLIT": 1}, resid=True)
    if shape.startswith("8x8"):
        for bn in (128, 64, 32):
            run(f"BN{bn} split<=16", shape, {"SR3_BLOCK_N": bn, "SR3_KSPLIT": 16})
    else:
        for mh, bn in ((2, 128), (2, 64), (1, 64), (1, 32)):
            run(f"tall {mh*128}x{bn} split<=16", shape, {"SR3_TALL_MH": mh, "SR3_TALL_BN": bn})
            run(f"tall {mh*128}x{bn} no split", shape, {"SR3_TALL_MH": mh, "SR3_TALL_BN": bn, "SR3_KSPLIT": 1})

"""The tile plan of the flagship step: for every tile op of the 16->128 engine at B = 16, conv_geometry's fitted byte model (DESIGN.md
section 3.1) picks the variant recorded here, the one the per-layer sweep (`tools/gpu_layer_profile.py --sweep`, DESIGN.md section 8)
timed as its choice.

The plan is a deterministic function of shape, batch, precision and SM count, so the table below holds on any 132-SM H100.  An edit to
the model that changes a row changes the flagship's speed: re-run the sweep and update the table together with DESIGN.md section 8.
"""
import pytest
import torch

import test_gpu_unet as tu

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")

# (op index of the eager step, output (H, W, C), tall halo, tile rows, BLOCK_N, schedule, split-K factor)
PLAN_16_128_B16 = [
    (  3, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (  5, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (  7, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (  9, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    ( 11, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    ( 12, (64, 64, 64), 0, 128,  64, "pingpong", 1),
    ( 14, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    ( 16, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    ( 18, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    ( 20, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    ( 21, (32, 32, 128), 0, 128,  64, "pingpong", 1),
    ( 23, (32, 32, 256), 1, 128,  64, "pingpong", 1),
    ( 25, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    ( 27, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    ( 29, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    ( 30, (16, 16, 256), 0, 128,  64, "pingpong", 1),
    ( 32, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 34, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 36, (16, 16, 1536), 0, 128, 128, "cooperative", 1),
    ( 38, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    ( 40, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 42, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 44, (16, 16, 1536), 0, 128, 128, "cooperative", 1),
    ( 46, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    ( 47, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 49, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 51, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 53, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 55, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 57, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 59, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 61, (8, 8, 1536), 0, 128, 128, "cooperative", 1),
    ( 63, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 65, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 67, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 69, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 71, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 73, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 75, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 77, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 79, (8, 8, 512), 0, 128,  32, "cooperative", 1),
    ( 80, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    ( 82, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 84, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 86, (16, 16, 1536), 0, 128, 128, "cooperative", 1),
    ( 88, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    ( 90, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 92, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    ( 94, (16, 16, 1536), 0, 128, 128, "cooperative", 1),
    ( 96, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    ( 98, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    (100, (16, 16, 512), 1, 256,  64, "cooperative", 1),
    (102, (16, 16, 1536), 0, 128, 128, "cooperative", 1),
    (104, (16, 16, 512), 0, 128, 128, "cooperative", 1),
    (105, (32, 32, 512), 1, 256,  64, "cooperative", 1),
    (107, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (109, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (111, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (113, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (115, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (117, (32, 32, 256), 1, 256,  64, "cooperative", 1),
    (118, (64, 64, 256), 1, 128,  64, "pingpong", 1),
    (120, (64, 64, 128), 1, 256,  64, "cooperative", 1),
    (122, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    (124, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    (126, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    (128, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    (130, (64, 64, 128), 1, 128,  64, "pingpong", 1),
    (131, (128, 128, 128), 1, 128,  64, "pingpong", 1),
    (133, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (135, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (137, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (139, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (141, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (143, (128, 128, 64), 1, 128,  64, "pingpong", 1),
    (145, (128, 128, 3), 1, 256,  16, "cooperative", 1)
]


def test_flagship_plan(monkeypatch):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the plan table is for a 132-SM H100")
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    net = tu.build(tu.FULL_UNET, 128, 0)
    eng = net.denoise_fn.engine(16)
    got = [(i, tuple(s["out_hwc"]), s["tall"], 128 * s["mh"], s["block_n"], s["schedule"], s["ksplit"])
           for i, s in enumerate(eng.tile_schedules()) if s is not None]
    assert len(got) == len(PLAN_16_128_B16)
    bad = [(g, w) for g, w in zip(got, PLAN_16_128_B16) if g != w]
    assert not bad, bad

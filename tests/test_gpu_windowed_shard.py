"""A windowed canvas sharded by window across ranks (parallel.window_shard_plan, WindowedSampler with a window range, the two-phase step):
the result is GaussianDiffusion.super_resolution_windowed bit for bit when every rank runs engines of the shape the one-canvas run uses.

Ranks are emulated on one device with the in-process exchange, which runs the plan the NCCL exchange runs.  Each emulated rank's x_T and
condition are NaN outside its band and its means arena is NaN before the first step, so a rank that read a row or a mean it does not own
or receive would put NaN into the result."""
import math
import os
import socket

import pytest
import torch

import _sizes_inputs as si
from test_gpu_windowed import build, draws, rel

pytestmark = pytest.mark.gpu

SEED, FIRST = 2 ** 33 + 7, 5


def emulate(net, cond, x_T, window, overlap, world, seed=SEED, first=FIRST):
    """The finished canvas of `world` ranks emulated on this device, each with its inputs poisoned outside its band."""
    from sr3_b200 import parallel
    B, _, H, W = cond.shape
    geo = net._window_geometry(H, W, window, overlap)
    plan = parallel.window_shard_plan(B, H, W, *geo, world)
    samplers, arenas, states = [], [], []
    for sh in plan:
        if sh.n1 == sh.n0:
            arenas.append(None)
            continue
        keep = torch.zeros(B, 1, H, 1, dtype=torch.bool, device=cond.device)
        for b, (y0, y1) in enumerate(sh.bands):
            keep[b, :, y0:y1] = True
        s = net._windowed_range_sampler(B, H, W, *geo, sh)
        assert s.means.isnan().all()
        s.begin(torch.where(keep, cond, math.nan), torch.where(keep, x_T, math.nan), seed, first)
        samplers.append(s)
        arenas.append(s.means)
    out = iter(parallel.sharded_windowed_loop(samplers, parallel.local_exchange(plan, arenas)))
    states = [None if a is None else next(out) for a in arenas]
    return parallel.assemble_rows(plan, states)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("B,H,W,overlap", [(1, 40, 72, 8), (1, 40, 72, 24), (2, 100, 70, 8), (2, 100, 70, 24)])
def test_emulated_ranks_equal_one_canvas(monkeypatch, precision, B, H, W, overlap):
    net = build(monkeypatch, si.TINY, 32, precision=precision)
    monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (2,))
    cond, x_T, _ = draws(B, H, W, 60 + overlap)
    ref = net.super_resolution_windowed(cond, window=(32, 32), overlap=overlap, continous=True, x_T=x_T, seed=SEED, first_index=FIRST)[-B:]
    assert torch.isfinite(ref).all()
    from sr3_b200 import _native
    n = B * len(_native.window_grid(H, 32, overlap)) * len(_native.window_grid(W, 32, overlap))
    worlds = (1, 2, 3, 5) + ((n + 2,) if n <= 24 else ())
    for world in worlds:
        got = emulate(net, cond, x_T, (32, 32), overlap, world)
        assert torch.isfinite(got).all(), world
        assert torch.equal(got, ref), (world, rel(got, ref))


@pytest.mark.timeout(1800)
def test_full_config_two_and_four_ranks(monkeypatch):
    """The 16->128 config at 200x312 (6 windows of 128x128): bit for bit under one fixed pass size; with the default pass sizes each rank
    may run a smaller engine than the one-canvas run (other split-K choices), and the difference is reported and bounded."""
    net = build(monkeypatch, si.FULL, 128)
    cond, x_T, _ = draws(1, 200, 312, 77)
    kw = dict(window=(128, 128), overlap=32, continous=True, x_T=x_T, seed=SEED, first_index=FIRST)
    one_default = net.super_resolution_windowed(cond, **kw)[-1:]
    for world in (2, 4):
        got = emulate(net, cond, x_T, (128, 128), 32, world)
        r = rel(got, one_default)
        print("16->128, 200x312, %d ranks, default pass sizes: relative L2 difference to one GPU %.3e" % (world, r))
        assert torch.isfinite(got).all() and r < 1e-2, r
    monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (1,))
    ref = net.super_resolution_windowed(cond, **kw)[-1:]
    for world in (2, 4):
        got = emulate(net, cond, x_T, (128, 128), 32, world)
        assert torch.equal(got, ref), (world, rel(got, ref))


def test_ranged_sampler_refuses_misuse(monkeypatch):
    from sr3_b200 import parallel
    net = build(monkeypatch, si.TINY, 32)
    plan = parallel.window_shard_plan(1, 40, 72, (32, 32), (8, 8), 2)
    s = net._windowed_range_sampler(1, 40, 72, (32, 32), 8, plan[0])
    cond, x_T, _ = draws(1, 40, 72, 3)
    s.begin(cond, x_T, 1, 0)
    with pytest.raises(RuntimeError, match="phase"):
        s.steps(9, 1)
    with pytest.raises(RuntimeError, match="phase_merge without"):
        s.phase_merge()
    s.phase_begin(0)
    s.phase_means()
    with pytest.raises(RuntimeError, match="out of order"):
        s.phase_means()
    s.phase_merge()
    with pytest.raises(RuntimeError, match="out of order"):
        s.phase_means()
    with pytest.raises(ValueError, match="window range"):
        net._windowed_range_sampler(1, 40, 72, (32, 32), 8, plan[0]._replace(n1=99))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, path):
    import torch.distributed as dist
    from sr3_b200 import parallel
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        mp = pytest.MonkeyPatch()
        net = build(mp, si.TINY, 32)
        mp.setattr(type(net), "WINDOW_PASS_SIZES", (2,))
        cond, x_T, _ = draws(1, 100, 70, 90)
        out = parallel.sharded_super_resolution(net, cond.cpu(), x_T=x_T.cpu(), seed=SEED, window=(32, 32), overlap=8)
        torch.save(out.cpu(), f"{path}.rank{rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(900)
def test_two_nccl_ranks_shard_one_image(monkeypatch, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    path = str(tmp_path / "out")
    mp.spawn(_nccl_worker, args=(2, _free_port(), path), nprocs=2, join=True)
    outs = [torch.load(f"{path}.rank{r}") for r in range(2)]
    assert torch.equal(outs[0], outs[1]) and outs[0].shape == (1, 3, 100, 70)
    net = build(monkeypatch, si.TINY, 32)
    monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", (2,))
    cond, x_T, _ = draws(1, 100, 70, 90)
    emu = emulate(net, cond, x_T, (32, 32), 8, 2, first=0)
    ref = net.super_resolution_windowed(cond, window=(32, 32), overlap=8, continous=True, x_T=x_T, seed=SEED)[-1:]
    assert torch.equal(outs[0], emu.cpu()) and torch.equal(outs[0], ref.cpu())

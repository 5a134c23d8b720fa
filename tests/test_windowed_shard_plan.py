"""A canvas sharded by window without a GPU: the ownership and exchange plan (parallel.window_shard_plan) over many geometries, the sharded
loop restated on the CPU oracle against the one-canvas loop, and the point-to-point exchange over two gloo ranks."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _windowed_shard_ref as sref
from oracle import sr3_oracle as orc
from oracle import windowed_oracle as worc
from sr3_b200 import _native, parallel


def geometries():
    """(B, H, W, side, overlap): one window up to several images, overlap 0, a quarter of the side and side - 1."""
    for side in (32, 64):
        for overlap in (0, side // 4, side - 1):
            for B, H, W in ((1, side, side), (1, side, 3 * side + 5), (1, 2 * side + 7, side), (2, 100, 70), (3, 2 * side + 1, 2 * side + 9)):
                if H >= side and W >= side:
                    yield B, H, W, side, overlap


def check_plan(B, H, W, side, overlap, world):
    oy, ox = _native.window_grid(H, side, overlap), _native.window_grid(W, side, overlap)
    ny, nx = len(oy), len(ox)
    n = B * ny * nx
    plan = parallel.window_shard_plan(B, H, W, side, overlap, world)
    assert len(plan) == world
    owner = {}
    for r, sh in enumerate(plan):                  # owned ranges partition the window list, balanced
        assert (sh.n0, sh.n1) == parallel.shard_bounds(n, world, r)
        for m in range(sh.n0, sh.n1):
            owner[m] = r
    assert sorted(owner) == list(range(n))

    def rows(m):
        y0 = oy[(m % (ny * nx)) // nx]
        return m // (ny * nx), y0, y0 + side

    for r, sh in enumerate(plan):
        assert len(sh.bands) == B
        for b, (y0, y1) in enumerate(sh.bands):    # bands contain every row their windows read, and no more
            mine = [rows(m) for m in range(sh.n0, sh.n1) if rows(m)[0] == b]
            if not mine:
                assert y1 <= y0
                continue
            assert (y0, y1) == (min(a for _, a, _ in mine), max(c for _, _, c in mine))
        got = []
        for src, m0, m1 in sh.recv:                # every receive comes from the owner; none is owned
            assert src != r and m0 < m1
            for m in range(m0, m1):
                assert owner[m] == src and not sh.n0 <= m < sh.n1
                got.append(m)
        assert len(got) == len(set(got))           # received exactly once
        need = set()
        for m in range(n):                         # every window meeting a band is owned or received
            b, a, c = rows(m)
            y0, y1 = sh.bands[b]
            if a < y1 and c > y0:
                need.add(m)
        assert set(got) | set(range(sh.n0, sh.n1)) >= need and set(got) <= need
        assert set(range(sh.n0, sh.n1)) <= need
    sends = sorted((src, r, m0, m1) for r, sh in enumerate(plan) for src, m0, m1 in sh.recv)
    assert sorted((s, d, m0, m1) for s, sh in enumerate(plan) for d, m0, m1 in sh.send) == sends      # send lists = transposed receives
    for s, sh in enumerate(plan):                  # one pair's messages are posted in the same (ascending) order on both sides
        for d in range(world):
            out = [(m0, m1) for dd, m0, m1 in sh.send if dd == d]
            assert out == sorted(out) == [(m0, m1) for src, m0, m1 in plan[d].recv if src == s]
    for b in range(B):                             # output rows partition every image, each inside its rank's band
        cover = torch.zeros(H, dtype=torch.int32)
        for sh in plan:
            for bb, y0, y1 in sh.rows:
                if bb == b:
                    assert sh.bands[b][0] <= y0 < y1 <= sh.bands[b][1]
                    cover[y0:y1] += 1
        assert (cover == 1).all()
    return n


@pytest.mark.parametrize("B,H,W,side,overlap", list(geometries()))
def test_plan_properties(B, H, W, side, overlap):
    n = None
    for world in (1, 2, 3, 4, 5, 8):
        n = check_plan(B, H, W, side, overlap, world)
    check_plan(B, H, W, side, overlap, min(n, 40) + 3)      # more ranks than windows (where there are few): the last ranks own nothing


def test_plan_of_a_frame():
    """720x1280 with 128x128 windows at overlap 32 on 8 ranks: 104 windows, 13 per rank, each rank receives the rows of windows above and
    below its own (at most 2 x 13)."""
    plan = parallel.window_shard_plan(1, 720, 1280, 128, 32, 8)
    assert [sh.n1 - sh.n0 for sh in plan] == [13] * 8
    assert max(sum(m1 - m0 for _, m0, m1 in sh.recv) for sh in plan) <= 26
    check_plan(1, 720, 1280, 128, 32, 8)


def test_plan_refuses_bad_requests():
    with pytest.raises(ValueError):
        parallel.window_shard_plan(1, 20, 64, 32, 8, 2)
    with pytest.raises(ValueError):
        parallel.window_shard_plan(1, 64, 64, 32, 32, 2)
    with pytest.raises(ValueError):
        parallel.window_shard_plan(1, 64, 64, 32, 8, 0)


TINY = orc.UNetConfig(6, 3, 64, 32, (1, 2), (16,), 1, 0.0, 32)
SCHED3 = {"schedule": "linear", "n_timestep": 3, "linear_start": 1e-4, "linear_end": 2e-2}


@pytest.mark.parametrize("B,H,W,overlap,worlds", [(1, 40, 72, (8, 8), (1, 2, 3, 7)), (2, 48, 40, (24, 8), (2, 3, 13))])
def test_sharded_oracle_equals_the_one_canvas_loop(B, H, W, overlap, worlds):
    sd = orc.init_state_dict(TINY, 0)
    sch = orc.make_schedule(SCHED3)
    g = torch.Generator().manual_seed(3)
    cond, x_T = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.randn(B, 3, H, W, generator=g)
    noises = torch.randn(3, B, 3, H, W, generator=g)

    def mean_fn(x, c, t):        # window by window, so that a window's mean cannot depend on the batch it runs in
        return torch.cat([orc.p_mean_variance(sd, TINY, sch, x[i:i + 1], t, True, c[i:i + 1])[0] for i in range(x.shape[0])])

    with torch.no_grad():
        ref = worc.p_sample_loop_windowed(sd, TINY, sch, cond, x_T, noises, True, (32, 32), overlap, mean_fn=mean_fn)
        n = len(sref.crops(B, H, W, (32, 32), overlap))
        for world in worlds:
            got = sref.p_sample_loop_windowed_sharded(mean_fn, sch, cond, x_T, noises, (32, 32), overlap, world)
            assert torch.isfinite(got).all() and torch.equal(got[-1], ref), world
        assert max(worlds) > n


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _exchange_worker(rank, world, port, geom, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        B, H, W, side, overlap = geom
        plan = parallel.window_shard_plan(B, H, W, side, overlap, world)
        n = plan[-1].n1
        sh = plan[rank]
        arena = torch.full((n, 3, side, side), float("nan"))
        mark = lambda m: torch.full((3, side, side), float(1000 * (m + 1)))        # noqa: E731  owner-independent content of slot m
        for m in range(sh.n0, sh.n1):
            arena[m] = mark(m)
        exchange = parallel.p2p_exchange(plan, rank, arena)
        for _ in range(2):                                                          # the same exchange, once per step
            exchange()
        want = set(range(sh.n0, sh.n1)) | {m for _, m0, m1 in sh.recv for m in range(m0, m1)}
        ok = bool(sh.recv)
        for m in range(n):
            ok = ok and (torch.equal(arena[m], mark(m)) if m in want else bool(arena[m].isnan().all()))
        ret[rank] = ok
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("geom", [(1, 40, 72, 32, 8), (1, 100, 70, 32, 31), (3, 40, 72, 32, 8)])
def test_p2p_exchange_two_ranks_gloo(geom):
    """Each rank holds exactly its own and its owners' received slabs after the exchange, and nothing else."""
    world = 2
    with mp.Manager() as m:
        ret = m.dict()
        mp.spawn(_exchange_worker, args=(world, _free_port(), geom, ret), nprocs=world, join=True)
        assert dict(ret) == {0: True, 1: True}


def test_merge_kernel_keeps_registers():
    """The band-restricted merge kernel compiles without a stack frame or spills (ptxas -v of the library build)."""
    import test_ptxas_pipeline as tp
    log = tp._build_log()
    i = log.index("Function properties for _ZN3sr319window_merge_kernelENS_11WindowMergeE")
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in log[i:].splitlines()[1]

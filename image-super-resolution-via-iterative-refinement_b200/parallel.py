"""Multi-GPU sampling: the reverse trajectories of different images are independent (GroupNorm and attention are per
sample), so the batch is sharded across ranks with NO per-step communication and the finished images are collected with one
all-gather (SURVEY.md 8e).  The reference only offers nn.DataParallel for training and samples on GPU 0
(model/model.py:60-78); this is the H100-native replacement for that path: one process per GPU, NCCL over NVLink.

Noise comes from Philox streams keyed by the GLOBAL sample index, so the result does not depend on the number of ranks.

A batch of fewer images than ranks (one large photograph) is sharded by WINDOW instead (window_shard_plan, DESIGN.md 5): every rank
runs a contiguous range of the canvas's window list and exchanges the means of the windows along its band's edges with its neighbours once
per reverse step; the result is the one-GPU windowed canvas bit for bit when every rank runs engines of the same shape.

Training (SURVEY.md 8e, config 4) is plain data parallelism with ONE exchange step: every rank runs forward / backward on its slice of the
batch, the parameter gradients are summed with NCCL all-reduces in buckets that are issued while the backward of the earlier layers is still
running (the native backward is replayed layer by layer: sr3_train_backward_block), and Adam is applied redundantly on every rank.  The
reference's own multi-GPU training is nn.DataParallel (model/networks.py:113-115: replicate + scatter + gather every forward).
"""
import bisect
from typing import Callable, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_bounds(global_batch: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced [lo, hi) slice of the batch owned by `rank` (first `global_batch % world_size` ranks get one more)."""
    if global_batch < 0 or world_size < 1 or not (0 <= rank < world_size):
        raise ValueError("bad shard request")
    base, rem = divmod(global_batch, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_shards(local: torch.Tensor, global_batch: int, group=None) -> torch.Tensor:
    """All-gather row shards of possibly unequal length into the [global_batch, ...] tensor (same on every rank)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(global_batch, world, r)[1] - shard_bounds(global_batch, world, r)[0] for r in range(world)]
    assert local.shape[0] == sizes[rank], (local.shape, sizes, rank)
    mx = max(sizes)
    if all(s == mx for s in sizes):
        out = torch.empty((global_batch,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[:s] for p, s in zip(parts, sizes)], dim=0)


def sharded_sample(sample_fn: Callable[[Optional[torch.Tensor], torch.Tensor, int], torch.Tensor], cond: Optional[torch.Tensor],
                   x_T: torch.Tensor, group=None) -> torch.Tensor:
    """Run `sample_fn(cond_shard, x_T_shard, first_global_index)` on this rank's slice and all-gather the finished images.

    `cond` / `x_T` are the GLOBAL tensors (every rank holds or can build them, e.g. from a shared seed)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = x_T.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    local = sample_fn(None if cond is None else cond[lo:hi], x_T[lo:hi], lo)
    if world == 1:
        return local
    return gather_shards(local, n, group)


def sharded_super_resolution(netG, x_in: torch.Tensor, x_T: Optional[torch.Tensor] = None, seed: int = 0, group=None, window=None,
                             overlap=None) -> torch.Tensor:
    """Batch-sharded `GaussianDiffusion.super_resolution` (reference: model/sr3_modules/diffusion.py:176-210 run on GPU 0 only,
    model/model.py:60-78): returns the [B,3,H,W] finished images x_0 on every rank, at the size of `x_in` (any size the engine accepts).

    `x_in` / `x_T` are the GLOBAL (host or device) tensors; each rank copies and samples only its slice; the Philox noise streams are keyed
    by the global sample index (`first_index`), so the images do not depend on the number of ranks.

    `window` / `overlap` (either one given): every rank runs `GaussianDiffusion.super_resolution_windowed`'s loop on its slice instead, for
    `x_in` of any size; its noise is keyed by the global sample index and the pixel's index in the canvas, so this too is rank independent.
    With fewer images than ranks the windows of the whole batch are sharded across the ranks instead (sharded_windowed_super_resolution),
    so one large image runs on every GPU."""
    dev = netG.betas.device
    if x_T is None:
        g = torch.Generator().manual_seed(seed)
        x_T = torch.randn(tuple(x_in.shape), generator=g)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if (window is not None or overlap is not None) and x_in.shape[0] < world:
        return sharded_windowed_super_resolution(netG, x_in, x_T, seed, 0, window, overlap, group)

    def fn(c, xt, first):
        if c.shape[0] == 0:
            return torch.empty((0,) + tuple(xt.shape[1:]), device=dev)
        if window is not None or overlap is not None:
            sampler = netG._windowed_sampler(c.shape[0], c.shape[2], c.shape[3], window, overlap)
            return sampler.sample_loop(c.to(dev, non_blocking=True), xt.to(dev, non_blocking=True), None, seed, first, want_snapshots=False)[0]
        # images of the net's image_size keep the plain `_engine(batch)` call (all a stand-in net without an image_size offers); other
        # sizes name theirs
        size, image_size = tuple(c.shape[2:]), getattr(netG, "image_size", None)
        eng = netG._engine(c.shape[0]) if image_size is None or size == (image_size, image_size) else netG._engine(c.shape[0], *size)
        final, _ = eng.p_sample_loop(c.to(dev, non_blocking=True), xt.to(dev, non_blocking=True), None, seed, first, want_snapshots=False)
        return final

    return sharded_sample(fn, x_in, x_T, group)


# ---------------------------------------------------------------------------------------------------- windowed canvas, sharded by window
class WindowShard(NamedTuple):
    """One rank's part of a canvas sharded by window.  Window n of the list is (image n // (ny nx), row (n // nx) % ny, column n % nx)."""
    n0: int                                 # owned windows [n0, n1) (n0 == n1: none)
    n1: int
    bands: List[Tuple[int, int]]            # per image: rows [y0, y1) the owned windows read, full width ((0, 0): none)
    recv: List[Tuple[int, int, int]]        # (src rank, m0, m1): not-owned windows [m0, m1) whose rows meet a band, owned by src
    send: List[Tuple[int, int, int]]        # (dst rank, m0, m1): the transpose of the other ranks' receive lists
    rows: List[Tuple[int, int, int]]        # (image, y0, y1): the rows this rank contributes to the finished canvas


def _pair(v):
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def window_shard_plan(batch: int, height: int, width: int, window, overlap, world: int) -> List[WindowShard]:
    """Ownership and exchange plan of a canvas [batch, C, height, width] covered by `window` = (wh, ww) windows that overlap by `overlap`
    (ints or pairs), on the grid of _native.window_grid, split over `world` ranks.  Rank r owns the balanced range shard_bounds(N, world, r)
    of the N windows; its band in an image runs from its first owned window's origin row to its last one's origin row + wh.  Every
    window covering a pixel of the band meets the band's rows, so the owned and received means are all a merge of the band reads.  The
    output rows give every row of every image to exactly one rank whose band contains it."""
    from ._native import window_grid
    (wh, ww), (ovh, ovw) = _pair(window), _pair(overlap)
    oy, ox = window_grid(height, wh, ovh), window_grid(width, ww, ovw)
    ny, nx = len(oy), len(ox)
    per = ny * nx
    n = batch * per
    if batch < 1 or world < 1:
        raise ValueError("bad plan request: batch %d, world %d" % (batch, world))
    starts = [shard_bounds(n, world, r)[0] for r in range(world)]

    shards = []
    for r in range(world):
        n0, n1 = shard_bounds(n, world, r)
        bands, recv = [(0, 0)] * batch, []
        for b in range(batch):
            lo, hi = max(n0, b * per), min(n1, (b + 1) * per)
            if lo >= hi:
                continue
            y0, y1 = oy[(lo - b * per) // nx], oy[(hi - 1 - b * per) // nx] + wh
            bands[b] = (y0, y1)
            hit = [iy for iy in range(ny) if oy[iy] < y1 and oy[iy] + wh > y0]
            for m in range(b * per + hit[0] * nx, b * per + (hit[-1] + 1) * nx):
                if n0 <= m < n1:
                    continue
                src = bisect.bisect_right(starts, m) - 1        # ranks that own nothing start at n, past every window
                if recv and recv[-1][0] == src and recv[-1][2] == m:
                    recv[-1] = (src, recv[-1][1], m + 1)
                else:
                    recv.append((src, m, m + 1))
        shards.append((n0, n1, bands, recv))
    send = [[] for _ in range(world)]
    for r, (_, _, _, recv) in enumerate(shards):
        for src, m0, m1 in recv:
            send[src].append((r, m0, m1))
    rows = [[] for _ in range(world)]
    for b in range(batch):
        cur = 0
        for r in range(world):
            y0, y1 = shards[r][2][b]
            if y1 > cur:
                assert y0 <= cur, (b, r, y0, cur)          # bands start in rank order and leave no gap: the windows cover the canvas
                rows[r].append((b, cur, y1))
                cur = y1
        assert cur == height, (b, cur, height)
    return [WindowShard(n0, n1, bands, recv, send[r], rows[r]) for r, (n0, n1, bands, recv) in enumerate(shards)]


def local_exchange(plan: Sequence[WindowShard], arenas: Sequence[Optional[torch.Tensor]]) -> Callable[[], None]:
    """The exchange between the means arenas of len(plan) ranks emulated in one process (None: a rank that owns nothing): every receive
    of the plan as a tensor copy from its owner's arena, on the current stream."""
    copies = [(arenas[r][m0:m1], arenas[src][m0:m1]) for r, sh in enumerate(plan) for src, m0, m1 in sh.recv]

    def run():
        for dst, src in copies:
            dst.copy_(src)
    return run


def p2p_exchange(plan: Sequence[WindowShard], rank: int, arena: Optional[torch.Tensor], group=None) -> Callable[[], None]:
    """The exchange of this rank's slabs with torch.distributed point-to-point operations (NCCL on GPUs: queued behind and waited for on
    the current stream, no host synchronisation).  Sends and receives of one pair are posted in ascending window order on both sides."""
    peer = (lambda r: r) if group is None else (lambda r: dist.get_global_rank(group, r))
    sh = plan[rank]
    ops = [dist.P2POp(dist.isend, arena[m0:m1], peer(dst), group) for dst, m0, m1 in sh.send] + \
          [dist.P2POp(dist.irecv, arena[m0:m1], peer(src), group) for src, m0, m1 in sh.recv]

    def run():
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
    return run


def sharded_windowed_loop(samplers: Sequence, exchange: Callable[[], None]) -> List[torch.Tensor]:
    """The whole reverse loop of range samplers (_native.WindowedSampler with a window_range, begin() already called), every step:
    phase (a) on every sampler, exchange(), phase (b) on every sampler.  Returns each sampler's final canvas state (its band rows hold
    the result; other rows are whatever begin() put there)."""
    if samplers:
        T = samplers[0].engine.T
        for s in samplers:
            s.phase_begin(T - 1)
        for _ in range(T):
            for s in samplers:
                s.phase_means()
            exchange()
            for s in samplers:
                s.phase_merge()
    return [s.read_state() for s in samplers]


def assemble_rows(plan: Sequence[WindowShard], states: Sequence[Optional[torch.Tensor]]) -> torch.Tensor:
    """The finished canvas from the states of emulated ranks: every row from the rank the plan gives it to."""
    ref = next(s for s in states if s is not None)
    out = torch.empty_like(ref)
    for sh, st in zip(plan, states):
        for b, y0, y1 in sh.rows:
            out[b, :, y0:y1] = st[b, :, y0:y1]
    return out


def gather_rows(plan: Sequence[WindowShard], rank: int, state: Optional[torch.Tensor], shape, device, group=None) -> torch.Tensor:
    """The finished canvas on every rank: each rank's output rows, all-gathered (padded to the longest) and placed; exact."""
    B, C, H, W = shape
    sizes = [sum(y1 - y0 for _, y0, y1 in sh.rows) * C * W for sh in plan]
    buf = torch.zeros(max(sizes), dtype=torch.float32, device=device)
    if sizes[rank]:
        buf[:sizes[rank]] = torch.cat([state[b, :, y0:y1].reshape(-1) for b, y0, y1 in plan[rank].rows])
    parts = [torch.empty_like(buf) for _ in plan]
    dist.all_gather(parts, buf, group=group)
    out = torch.empty(shape, dtype=torch.float32, device=device)
    for sh, part in zip(plan, parts):
        off = 0
        for b, y0, y1 in sh.rows:
            k = (y1 - y0) * C * W
            out[b, :, y0:y1] = part[off:off + k].view(C, y1 - y0, W)
            off += k
    return out


def sharded_windowed_super_resolution(netG, x_in: torch.Tensor, x_T: torch.Tensor, seed: int, first_index: int, window, overlap,
                                      group=None) -> torch.Tensor:
    """`GaussianDiffusion.super_resolution_windowed` of the whole batch with its windows sharded across the ranks of `group`: each rank
    builds the same plan, runs its window range on an engine chosen from its own window count, exchanges the means its band needs every
    step over point-to-point operations and ends with the whole finished [B, C, H, W] canvas."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = netG.betas.device
    B, _, H, W = x_in.shape
    (wh, ww), ov = netG._window_geometry(H, W, window, overlap)
    plan = window_shard_plan(B, H, W, (wh, ww), ov, world)
    sh = plan[rank]
    sampler = None
    if sh.n1 > sh.n0:
        sampler = netG._windowed_range_sampler(B, H, W, (wh, ww), ov, sh)
        sampler.begin(x_in.to(dev, non_blocking=True), x_T.to(dev, non_blocking=True), seed, first_index)
    dist.all_reduce(torch.zeros(1, device=dev), group=group)     # every rank joins the group's first operation before the point-to-point
    states = sharded_windowed_loop([sampler] if sampler else [], p2p_exchange(plan, rank, sampler.means if sampler else None, group))
    return gather_rows(plan, rank, states[0] if states else None, (B, netG.channels, H, W), dev, group)


# ---------------------------------------------------------------------------------------------------------------- training
def plan_buckets(block_param_indices, param_numels, bucket_elems):
    """Group the backward's layers (last layer first) into gradient buckets of about `bucket_elems` elements.

    block_param_indices[i] = parameter indices whose gradient is final once backward block i has run (blocks run n-1 .. 0); parameters that
    appear in no block (FiLM projections, noise-level MLP: final only after the whole backward) form the last bucket.  Returns
    [(first_block_done, [param indices])]: the bucket may be reduced as soon as block `first_block_done` has run (-1: after finish)."""
    n_blocks = len(block_param_indices)
    seen = set()
    buckets, cur, cur_n = [], [], 0
    for i in range(n_blocks - 1, -1, -1):
        for pi in block_param_indices[i]:
            if pi in seen:
                continue
            seen.add(pi)
            cur.append(pi)
            cur_n += param_numels[pi]
        if cur_n >= bucket_elems:
            buckets.append((i, cur))
            cur, cur_n = [], 0
    rest = [pi for pi in range(len(param_numels)) if pi not in seen]
    if cur:
        buckets.append((0, cur))
    if rest:
        buckets.append((-1, rest))
    return buckets


class GradientBuckets:
    """Flat fp32 gradient arena cut into buckets in the order the backward finishes them; parameter i's gradient is the view `views[i]`.
    ready(block) all-reduces (sum) every bucket that became final with backward block `block` -- on CUDA on a side stream, ordered behind the
    work queued on the current stream so far, so the transfer overlaps the layers still to run; finish() joins the streams."""

    def __init__(self, params, block_param_indices, bucket_elems, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        numels = [p.numel() for p in params]
        self.buckets = plan_buckets(block_param_indices, numels, bucket_elems)
        dev = params[0].device
        self.flat = torch.zeros(sum(numels), dtype=torch.float32, device=dev)
        self.views = [None] * len(params)
        self.slices = []
        off = 0
        for first_block, idxs in self.buckets:
            lo = off
            for pi in idxs:
                self.views[pi] = self.flat[off:off + numels[pi]].view(params[pi].shape)
                off += numels[pi]
            self.slices.append((first_block, lo, off))
        assert off == self.flat.numel()
        self.cuda = dev.type == "cuda"
        self.comm_stream = torch.cuda.Stream(device=dev) if (self.cuda and self.world > 1) else None
        self.pending = []
        self.n_reduced = 0
        self._t0 = self._t1 = None

    def begin(self):
        self.pending = list(self.slices)
        self.n_reduced = 0
        if self.comm_stream is not None:
            self._t0, self._t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def ready(self, block):
        while self.pending and self.pending[0][0] == block:
            _, lo, hi = self.pending.pop(0)
            self.n_reduced += 1
            if self.world == 1:
                continue
            if self.comm_stream is None:
                dist.all_reduce(self.flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group)
                continue
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream())
            self.comm_stream.wait_event(done)
            with torch.cuda.stream(self.comm_stream):
                if self.n_reduced == 1:
                    self._t0.record(self.comm_stream)
                dist.all_reduce(self.flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group)

    def finish(self):
        self.ready(-1)
        assert not self.pending, "backward blocks were skipped"
        if self.comm_stream is not None:
            self._t1.record(self.comm_stream)
            torch.cuda.current_stream().wait_stream(self.comm_stream)

    def comm_window_ms(self):
        """Device time from the start of the first to the end of the last all-reduce of the most recent step (overlapping the backward)."""
        if self.comm_stream is None or self._t0 is None:
            return 0.0
        torch.cuda.synchronize()
        return self._t0.elapsed_time(self._t1)


class DataParallelTrainer:
    """One process per GPU.  step(hr, sr) = DDPM.optimize_parameters (model/model.py:48-58) on this rank's slice of the global batch:
    native forward -> native backward replayed layer by layer, each finished bucket of gradients all-reduced (sum) on a side stream while the
    remaining layers run -> one fused Adam launch (gradients are scaled by 1 / (global b c h w) when they are produced, so the all-reduced
    sum IS the gradient of the global mean the reference optimises).  Without a process group (world size 1) the collectives are skipped."""

    def __init__(self, netG, lr=1e-4, bucket_mb=64.0, group=None):
        from .optim import FusedAdam
        self.net = netG
        self.group = group
        self.opt = FusedAdam(list(netG.denoise_fn.parameters()), lr=lr)
        self.bucket_elems = int(bucket_mb * (1 << 20) / 4)
        self._eng = None
        self.buckets = None

    def _prepare(self, eng):
        if self._eng is eng:
            return
        by_name = dict(self.net.denoise_fn.named_parameters())
        params = [by_name[n] for n, _ in eng.param_table()]
        blocks = [eng.block_params(i) for i in range(eng.num_backward_blocks())]
        self.buckets = GradientBuckets(params, blocks, self.bucket_elems, self.group)
        for p, v in zip(params, self.buckets.views):
            p.grad = v                           # the optimizer reads the all-reduced arena directly
        self._eng = eng

    def step(self, hr, sr, gamma=None, noise=None, dropout_seed=None, global_batch=None):
        """hr / sr: THIS rank's slice [b,3,H,W] (device or host), H x W any size _native.check_image_size accepts.  Returns the summed loss
        of the slice (python float)."""
        import numpy as np
        net = self.net
        b, c, h, w = hr.shape
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        gb = global_batch if global_batch is not None else b * world
        drop = float(getattr(net.denoise_fn, "dropout", 0) or 0) if net.training else 0.0
        eng = net.denoise_fn.engine(b, conditional=net.conditional, channels=net.channels, train_dropout=drop, height=h, width=w)
        self._prepare(eng)
        if gamma is None:
            t = np.random.randint(1, net.num_timesteps + 1)
            gamma = torch.FloatTensor(np.random.uniform(net.sqrt_alphas_cumprod_prev[t - 1], net.sqrt_alphas_cumprod_prev[t], size=b))
        if noise is None:
            noise = torch.randn(hr.shape, device=net.betas.device)
        if dropout_seed is None:
            dropout_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        loss = eng.train_forward(hr, sr if net.conditional else None, gamma, noise, net.loss_type, dropout_seed)
        bk = self.buckets
        eng.backward_begin(1.0 / float(gb * c * h * w), bk.views)
        bk.begin()
        boundaries = {fb for fb, _, _ in bk.slices}
        for i in range(eng.num_backward_blocks() - 1, -1, -1):
            eng.backward_block(i)
            if i in boundaries:
                eng.backward_flush()             # the bucket's conv weight gradients: partial tiles -> OIHW, one launch
                bk.ready(i)
        eng.backward_finish()
        bk.finish()
        self.opt.step()
        return loss

    def comm_window_ms(self):
        return self.buckets.comm_window_ms() if self.buckets is not None else 0.0

"""Multi-GPU sampling: the reverse trajectories of different images are independent (GroupNorm and attention are per
sample), so the batch is sharded across ranks with NO per-step communication and the finished images are collected with one
all-gather (SURVEY.md 8e).  The reference only offers nn.DataParallel for training and samples on GPU 0
(model/model.py:60-78); this is the H100-native replacement for that path: one process per GPU, NCCL over NVLink.

Noise comes from Philox streams keyed by the GLOBAL sample index, so the result does not depend on the number of ranks.

Training (SURVEY.md 8e, config 4) is plain data parallelism with ONE exchange step: every rank runs forward / backward on its slice of the
batch, the parameter gradients are summed with NCCL all-reduces in buckets that are issued while the backward of the earlier layers is still
running (the native backward is replayed layer by layer: sr3_train_backward_block), and Adam is applied redundantly on every rank.  The
reference's own multi-GPU training is nn.DataParallel (model/networks.py:113-115: replicate + scatter + gather every forward).
"""
from typing import Callable, Optional, Tuple

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
    `x_in` of any size; its noise is keyed by the global sample index and the pixel's index in the canvas, so this too is rank independent."""
    dev = netG.betas.device
    if x_T is None:
        g = torch.Generator().manual_seed(seed)
        x_T = torch.randn(tuple(x_in.shape), generator=g)

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

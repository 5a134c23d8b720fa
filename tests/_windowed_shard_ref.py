"""The window-sharded reverse loop restated on the CPU on top of oracle/windowed_oracle.windowed_step, for R simulated ranks.

Every rank holds a canvas that is NaN outside its band and a means arena that is NaN outside its owned and received slots.  A step is:
every rank computes the means of its own windows from its canvas; the plan's receives copy slots between the arenas; every rank runs
windowed_step with its arena standing in for the UNet and keeps the rows of its band.  The result is assembled from the output rows.  A
rank that read a row or a mean it should not have would carry NaN into its band."""
import math

import torch

from oracle import sr3_oracle as orc
from oracle import windowed_oracle as worc
from sr3_b200 import parallel


def crops(B, H, W, window, overlap):
    wh, ww = window
    return [(slice(b, b + 1), slice(None), slice(y0, y0 + wh), slice(x0, x0 + ww))
            for b in range(B) for y0 in worc.window_grid(H, wh, overlap[0]) for x0 in worc.window_grid(W, ww, overlap[1])]


def band_mask(sh, B, H):
    keep = torch.zeros(B, 1, H, 1, dtype=torch.bool)
    for b, (y0, y1) in enumerate(sh.bands):
        keep[b, :, y0:y1] = True
    return keep


def p_sample_loop_windowed_sharded(mean_fn, sch: orc.Schedule, x_in, x_T, noises, window, overlap, world):
    """The final canvas [B, C, H, W] of p_sample_loop_windowed (conditional) with the windows sharded over `world` simulated ranks."""
    B, C, H, W = x_T.shape
    plan = parallel.window_shard_plan(B, H, W, window, overlap, world)
    cs = crops(B, H, W, window, overlap)
    n = len(cs)
    keeps = [band_mask(sh, B, H) for sh in plan]
    nan = torch.tensor(math.nan)
    xs = [torch.where(k, x_T, nan) for k in keeps]
    conds = [torch.where(k, x_in, nan) for k in keeps]
    for t in reversed(range(sch.num_timesteps)):
        arenas = [torch.full((n, C) + tuple(window), math.nan) for _ in plan]
        for sh, x, c, a in zip(plan, xs, conds, arenas):
            if sh.n1 > sh.n0:
                a[sh.n0:sh.n1] = mean_fn(torch.cat([x[cs[m]] for m in range(sh.n0, sh.n1)]),
                                         torch.cat([c[cs[m]] for m in range(sh.n0, sh.n1)]), t)
        for sh, a in zip(plan, arenas):
            for src, m0, m1 in sh.recv:
                a[m0:m1] = arenas[src][m0:m1]
        xs = [torch.where(k, worc.windowed_step(lambda xc, cc, tt, a=a: a, sch, x, c, t, noises[t], window, overlap), nan)
              for k, x, c, a in zip(keeps, xs, conds, arenas)]
    out = torch.full_like(x_T, math.nan)
    for sh, x in zip(plan, xs):
        for b, y0, y1 in sh.rows:
            out[b, :, y0:y1] = x[b, :, y0:y1]
    return out

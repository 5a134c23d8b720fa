"""Windowed sampling restated on the CPU (torch fp32) on top of sr3_oracle.p_mean_variance: the window grid, the blend weights, one merged
reverse step and the loop over them, as DESIGN.md 3.9 defines them.

A canvas [B, C, H, W] of any size H >= wh, W >= ww is covered per axis by windows of the window's side: one when the side equals the
canvas's, else n = ceil((L - overlap) / (side - overlap)) at origins round-half-up(i (L - side) / (n - 1)).  Every reverse step t runs
p_mean_variance (clip_denoised) on each window's crop of the canvas x_t and of the condition and blends the posterior means
    mean(p) = sum_n w_n(p) mean_n(p) / sum_n w_n(p)      (windows covering p in ascending index, fp32, products and sums rounded separately)
with w_n(p) = wy(y) wx(x), w(i) = min(i + 1, side - i, ramp) / ramp, ramp = max(overlap, 1), the ramp towards a border of the canvas replaced
by 1; then x_{t-1} = mean + exp(0.5 logvar_t) z for t > 0 with ONE z per canvas pixel."""
from typing import Callable, List, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import sr3_oracle as orc


def window_grid(length: int, side: int, overlap: int) -> List[int]:
    if length < side:
        raise ValueError("canvas side %d is smaller than the window side %d" % (length, side))
    if not 0 <= overlap < side:
        raise ValueError("overlap %d must be at least 0 and below the window side %d" % (overlap, side))
    if length == side:
        return [0]
    n = -(-(length - overlap) // (side - overlap))
    return [(2 * i * (length - side) + (n - 1)) // (2 * (n - 1)) for i in range(n)]


def window_weights(n: int, side: int, overlap: int) -> Tensor:
    """[n, side] fp32."""
    ramp = max(overlap, 1)
    out = torch.empty(n, side, dtype=torch.float32)
    for k in range(n):
        for i in range(side):
            m = ramp
            if k > 0:
                m = min(m, i + 1)
            if k < n - 1:
                m = min(m, side - i)
            out[k, i] = m
    return out / torch.tensor(float(ramp), dtype=torch.float32)


def merge_means(means: Sequence[Tensor], shape: Tuple[int, int, int, int], window: Tuple[int, int], overlap: Tuple[int, int]) -> Tensor:
    """means[n]: [C, wh, ww] of window n = (image b, row iy, column ix) in that nesting order -> the blended canvas mean [B, C, H, W]."""
    B, C, H, W = shape
    wh, ww = window
    oy, ox = window_grid(H, wh, overlap[0]), window_grid(W, ww, overlap[1])
    wy, wx = window_weights(len(oy), wh, overlap[0]), window_weights(len(ox), ww, overlap[1])
    num = torch.zeros(shape, dtype=torch.float32)
    den = torch.zeros(B, 1, H, W, dtype=torch.float32)
    n = 0
    for b in range(B):
        for iy, y0 in enumerate(oy):
            for ix, x0 in enumerate(ox):
                w = wy[iy][:, None] * wx[ix][None, :]
                num[b, :, y0:y0 + wh, x0:x0 + ww] = num[b, :, y0:y0 + wh, x0:x0 + ww] + w * means[n]
                den[b, :, y0:y0 + wh, x0:x0 + ww] = den[b, :, y0:y0 + wh, x0:x0 + ww] + w
                n += 1
    return num / den


def windowed_step(mean_fn: Callable[[Tensor, Optional[Tensor], int], Tensor], sch: orc.Schedule, x_t: Tensor, cond: Optional[Tensor], t: int,
                  noise: Optional[Tensor], window: Tuple[int, int], overlap: Tuple[int, int]) -> Tensor:
    """One merged reverse step.  mean_fn(x_crops [N, C, wh, ww], cond_crops or None, t) -> posterior means [N, C, wh, ww]; the windows of
    all images run as one batch, in list order (image, row, column)."""
    B, C, H, W = x_t.shape
    wh, ww = window
    crops = [(slice(b, b + 1), slice(None), slice(y0, y0 + wh), slice(x0, x0 + ww))
             for b in range(B) for y0 in window_grid(H, wh, overlap[0]) for x0 in window_grid(W, ww, overlap[1])]
    means = mean_fn(torch.cat([x_t[c] for c in crops]), None if cond is None else torch.cat([cond[c] for c in crops]), t)
    mean = merge_means(means, tuple(x_t.shape), window, overlap)
    if t == 0:
        return mean
    return mean + noise * (0.5 * sch.buffers["posterior_log_variance_clipped"][t]).exp()


def p_sample_loop_windowed(sd, cfg, sch: orc.Schedule, x_in: Optional[Tensor], x_T: Tensor, noises: Sequence[Tensor], conditional: bool,
                           window: Tuple[int, int], overlap: Tuple[int, int], continous: bool = False, mean_fn=None) -> Tensor:
    """sr3_oracle.p_sample_loop with every step replaced by windowed_step; noises[i] (canvas shape) is used at step i."""
    if mean_fn is None:
        mean_fn = lambda x, c, t: orc.p_mean_variance(sd, cfg, sch, x, t, True, c)[0]
    T = sch.num_timesteps
    inter = 1 | (T // 10)
    img = x_T
    ret = x_in if conditional else x_T
    for i in reversed(range(T)):
        img = windowed_step(mean_fn, sch, img, x_in if conditional else None, i, noises[i], window, overlap)
        if i % inter == 0:
            ret = torch.cat([ret, img], dim=0)
    return ret if continous else ret[-1]

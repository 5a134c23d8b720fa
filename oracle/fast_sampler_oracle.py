"""Few-step samplers restated on the CPU in fp64 (DESIGN.md 3.11): respaced DDIM and DPM-Solver++(2M) on the trained schedule, written
straight from their definitions, independently of the package's tables.

Timesteps tau_k = round(k (T - 1) / (K - 1)) (tau = [T - 1] for K = 1), abar_k = alphas_cumprod[tau_k], abar_{-1} = 1; step k runs from
K - 1 down to 0 and conditions the model on fp32(sqrt(abar_k)).  x0_k = clamp(sqrt(1 / abar_k) x_k - sqrt(1 / abar_k - 1) eps, -1, 1).
* DDIM:  x_{k-1} = sqrt(abar') x0 + sqrt(1 - abar' - sigma^2) eps(x0) + sigma z,  eps(x0) = (x_k - sqrt(abar_k) x0) / sqrt(1 - abar_k),
         sigma = eta sqrt((1 - abar') / (1 - abar_k)) sqrt(1 - abar_k / abar'),  abar' = abar_{k-1}.
* DPM-Solver++(2M):  alpha = sqrt(abar), sigma = sqrt(1 - abar), lambda = log(alpha / sigma), h = lambda_{k-1} - lambda_k,
         D = x0_k (first step) or (1 + 1 / 2r) x0_k - x0_{k+1} / 2r with r = h_{k+1} / h_k,
         x_{k-1} = (sigma_{k-1} / sigma_k) x_k + alpha_{k-1} (1 - e^-h) D;  the last step (abar_{-1} = 1) returns x0_0.

`eps_fn(x, k, noise_level)` is the model: unet_eps() wraps sr3_oracle's UNet (fp64), canvas_x0() blends the windows' x0 on a canvas as
windowed_oracle does, and the tests also pass closed-form models."""
import math
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import sr3_oracle as orc
from . import windowed_oracle as worc


def timesteps(T: int, K: int) -> List[int]:
    if K == 1:
        return [T - 1]
    return [int(math.floor(k * (T - 1) / (K - 1) + 0.5)) for k in range(K)]


def alphas_cumprod(schedule_opt) -> np.ndarray:
    betas = orc.make_beta_schedule(schedule_opt["schedule"], schedule_opt["n_timestep"], schedule_opt["linear_start"],
                                   schedule_opt["linear_end"])
    return np.cumprod(1. - betas)


def respaced(schedule_opt, K: int) -> np.ndarray:
    """abar_k, k = 0 .. K - 1 (fp64)."""
    ac = alphas_cumprod(schedule_opt)
    return ac[timesteps(len(ac), K)]


def unet_eps(sd, cfg: orc.UNetConfig, cond: Optional[Tensor]) -> Callable[[Tensor, int, float], Tensor]:
    """The UNet (weights cast to fp64) conditioned on `cond` as eps_fn."""
    sd64 = {k: v.double() for k, v in sd.items()}

    def eps(x, k, nl):
        inp = x if cond is None else torch.cat([cond.double(), x], dim=1)
        return orc.unet_forward(sd64, cfg, inp, torch.full((x.shape[0], 1), nl, dtype=torch.float64))
    return eps


def predict_x0(eps_fn, x: Tensor, k: int, abar: float, clip: bool = True) -> Tensor:
    nl = float(np.float32(math.sqrt(abar)))
    x0 = math.sqrt(1. / abar) * x - math.sqrt(1. / abar - 1.) * eps_fn(x, k, nl)
    return x0.clamp(-1., 1.) if clip else x0


def canvas_x0(sd, cfg: orc.UNetConfig, cond: Optional[Tensor], window: Tuple[int, int], overlap: Tuple[int, int]):
    """x0_fn(x, k, abar) of a canvas: every window's clipped x0 (fp64 UNet) blended with windowed_oracle's weights."""
    eps = unet_eps(sd, cfg, None)
    wh, ww = window

    def x0_fn(x, k, abar):
        B, C, H, W = x.shape
        crops = [(slice(b, b + 1), slice(None), slice(y0, y0 + wh), slice(x0, x0 + ww))
                 for b in range(B) for y0 in worc.window_grid(H, wh, overlap[0]) for x0 in worc.window_grid(W, ww, overlap[1])]
        xs = torch.cat([x[c] for c in crops]).double()
        inp_cond = None if cond is None else torch.cat([cond[c] for c in crops]).double()
        e = (lambda xx, kk, nl: eps(torch.cat([inp_cond, xx], 1) if inp_cond is not None else xx, kk, nl))
        x0s = predict_x0(e, xs, k, abar)
        return worc.merge_means(list(x0s), tuple(x.shape), window, overlap).double()
    return x0_fn


def sample(x0_fn: Callable[[Tensor, int, float], Tensor], abars: Sequence[float], spec: dict, x_T: Tensor,
           noises: Optional[Sequence[Tensor]] = None, keep_states: bool = False):
    """Run `spec` ({"sampler": "ddim", "steps": K, "eta": eta} or {"sampler": "dpmpp_2m", "steps": K}) from x_T through the K steps of
    abars = abar_0 .. abar_{K-1}.  x0_fn(x, k, abar_k) -> x0 (clipped, e.g. lambda x, k, a: predict_x0(eps_fn, x, k, a)).  noises[k] is z
    at step k (DDIM with eta > 0).  Returns x_{-1}, or (x_{-1}, [x_{K-2}, ..., x_{-1}]) with keep_states (the state after every step)."""
    K = len(abars)
    x = x_T.double()
    states = []
    x0_next = None                      # x0 of step k + 1
    for k in reversed(range(K)):
        a = float(abars[k])
        ap = 1. if k == 0 else float(abars[k - 1])
        x0 = x0_fn(x, k, a).double()
        if spec["sampler"] == "ddim":
            eta = float(spec.get("eta", 0.0))
            sigma = eta * math.sqrt((1. - ap) / (1. - a)) * math.sqrt(max(1. - a / ap, 0.))
            eps = (x - math.sqrt(a) * x0) / math.sqrt(1. - a)
            x = math.sqrt(ap) * x0 + math.sqrt(max(1. - ap - sigma * sigma, 0.)) * eps
            if sigma > 0:
                x = x + sigma * noises[k].double()
        elif k == 0:
            x = x0
        else:
            lam = lambda ab: math.log(math.sqrt(ab) / math.sqrt(1. - ab))
            h = lam(ap) - lam(a)
            if x0_next is None:
                D = x0
            else:
                r = (lam(a) - lam(float(abars[k + 1]))) / h
                D = (1. + 1. / (2. * r)) * x0 - x0_next / (2. * r)
            x = (math.sqrt(1. - ap) / math.sqrt(1. - a)) * x + math.sqrt(ap) * (1. - math.exp(-h)) * D
        x0_next = x0
        states.append(x)
    return (x, states) if keep_states else x


def sample_loop(sd, cfg: orc.UNetConfig, schedule_opt, spec: dict, x_in: Optional[Tensor], x_T: Tensor,
                noises: Optional[Sequence[Tensor]] = None, continous: bool = False, window=None, overlap=(0, 0)) -> Tensor:
    """p_sample_loop(sampler=spec) with the draws injected: [x_in or x_T ; x after every step k with k % (1 | K // 10) == 0] when
    continous, else the last image of the batch.  `window`: run as a canvas of such windows (canvas_x0), default one window = the image."""
    K = int(spec["steps"])
    abars = respaced(schedule_opt, K)
    if window is None:
        eps = unet_eps(sd, cfg, x_in)
        x0_fn = lambda x, k, a: predict_x0(eps, x, k, a)
    else:
        x0_fn = canvas_x0(sd, cfg, x_in, tuple(window), tuple(overlap))
    _, states = sample(x0_fn, abars, spec, x_T, noises, keep_states=True)
    inter = 1 | (K // 10)
    ret = (x_in if x_in is not None else x_T).double()
    for i, k in enumerate(reversed(range(K))):
        if k % inter == 0:
            ret = torch.cat([ret, states[i]], dim=0)
    return ret if continous else ret[-1]

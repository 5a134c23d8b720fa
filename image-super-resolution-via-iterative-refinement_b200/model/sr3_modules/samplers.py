"""Few-step samplers on the trained noise schedule (DESIGN.md 3.11): respaced DDIM and DPM-Solver++(2M), as tables the native samplers read.

A sampler spec is a dict, {"sampler": "ddim", "steps": K, "eta": eta} (1 <= K <= T, 0 <= eta <= 1) or {"sampler": "dpmpp_2m", "steps": K}
(2 <= K <= T), and always respaces the schedule of set_new_noise_schedule (T steps).  The K steps sit at the trained timesteps
tau_k = round(k (T - 1) / (K - 1)), k = 0 .. K - 1 (tau = [T - 1] for K = 1); the engine's step index k runs from K - 1 down to 0, and step k
conditions the UNet on the trained noise level sqrt(abar_k) = sqrt_alphas_cumprod_prev[tau_k + 1], so the model only sees levels it was
trained on.  abar_k = alphas_cumprod[tau_k], abar_{-1} = 1.

Every table is computed in fp64 and rounded once to fp32, like noise_schedule_buffers.  Both samplers run on the existing update of every
native sampler, x0 = clamp(c1 x_k - c2 eps), with the per-step rows c1 = sqrt(1 / abar_k), c2 = sqrt(1 / abar_k - 1):
* DDIM: x_{k-1} = pc1 x0 + pc2 x_k + sigma_k z, i.e. sqrt(abar') x0 + sqrt(1 - abar' - sigma^2) eps(x0) + sigma z with the eps re-derived from
  the clipped x0, eps(x0) = (x_k - sqrt(abar_k) x0) / sqrt(1 - abar_k), abar' = abar_{k-1}.  sigma_k = eta sqrt((1 - abar') / (1 - abar_k))
  sqrt(1 - abar_k / abar'); the last factor is computed from the betas between the two timesteps (-expm1(sum log1p(-beta))), not from a
  quotient of the rounded cumulative products, and the rows are rearranged so that nothing cancels (ddim_tables64): K = T, eta = 1 gives
  the DDPM posterior to rounding.  logvar = log sigma^2 is -inf
  where sigma = 0 (eta = 0, and k = 0, where abar' = 1 makes the step return x0): exp(0.5 logvar) is then exactly 0 and no noise is added.
* DPM-Solver++(2M) (Lu et al. 2022, data prediction, multistep): the engine's rows are pc1 = 1, pc2 = 0, so its "posterior mean" is the clipped
  x0, and the canvas merge applies x_{k-1} = A x_k + B x0_k + C x0_{k+1} with alpha = sqrt(abar), sigma = sqrt(1 - abar),
  lambda = log(alpha / sigma), h_k = lambda_{k-1} - lambda_k, r_k = h_{k+1} / h_k, A = sigma_{k-1} / sigma_k,
  B = alpha_{k-1} (1 - e^-h)(1 + 1 / 2r), C = -alpha_{k-1} (1 - e^-h) / 2r; the first step (k = K - 1) is first order (C = 0,
  B = alpha_{k-1} (1 - e^-h)), the last (k = 0, to abar = 1) returns x0_0 (A = 0, B = 1, C = 0).  No noise."""
import numbers

import numpy as np
import torch

SAMPLER_NAMES = ("ddim", "dpmpp_2m")


def check_sampler_spec(spec, T, what="sampler"):
    """The canonical (name, steps, eta) of a sampler spec for a trained schedule of T steps (eta is None for dpmpp_2m), or ValueError naming
    `what` and the offending key."""
    if not isinstance(spec, dict):
        raise ValueError("%s: a sampler spec is a dict with keys 'sampler', 'steps' (and 'eta' for ddim), got %r" % (what, type(spec)))
    name = spec.get("sampler")
    if name not in SAMPLER_NAMES:
        raise ValueError("%s: unknown 'sampler' %r (one of %s)" % (what, name, ", ".join(SAMPLER_NAMES)))
    extra = sorted(set(spec) - {"sampler", "steps", "eta"})
    if extra:
        raise ValueError("%s: unknown key %s in a %s spec" % (what, ", ".join(repr(k) for k in extra), name))
    if "steps" not in spec:
        raise ValueError("%s: the %s spec has no 'steps'" % (what, name))
    K, lo = spec["steps"], 1 if name == "ddim" else 2
    if isinstance(K, bool) or not isinstance(K, numbers.Integral) or not lo <= K <= T:
        raise ValueError("%s: 'steps' %r out of range [%d, %d] for %s on the %d-step trained schedule" % (what, K, lo, T, name, T))
    if name == "dpmpp_2m":
        if "eta" in spec:
            raise ValueError("%s: 'eta' is a ddim option; dpmpp_2m adds no noise" % what)
        return (name, int(K), None)
    eta = spec.get("eta", 0.0)
    if isinstance(eta, bool) or not isinstance(eta, numbers.Real) or not 0.0 <= float(eta) <= 1.0:
        raise ValueError("%s: 'eta' %r out of range [0, 1]" % (what, eta))
    return (name, int(K), float(eta))


def respaced_timesteps(T, K):
    """tau_k = round(k (T - 1) / (K - 1)) for k = 0 .. K - 1 (round half up, exact integer arithmetic); [T - 1] for K = 1."""
    if K == 1:
        return np.array([T - 1], dtype=np.int64)
    k = np.arange(K, dtype=np.int64)
    return (2 * k * (T - 1) + (K - 1)) // (2 * (K - 1))


def _respaced(betas, K):
    """fp64 (tau, abar [K], abar' [K] = abar_{k-1} with abar_{-1} = 1, 1 - abar_k / abar' [K]) of the betas of the trained schedule."""
    betas = np.asarray(betas, dtype=np.float64)
    T = betas.shape[0]
    tau = respaced_timesteps(T, K)
    ac = np.cumprod(1. - betas, axis=0)                   # noise_schedule_buffers' alphas_cumprod
    abar = ac[tau]
    abar_prev = np.append(1., abar[:-1])
    # 1 - prod_{tau_{k-1} < j <= tau_k} (1 - beta_j), with tau_{-1} = -1
    log_alpha = np.log1p(-betas)
    edges = np.append(-1, tau)
    one_minus_ratio = -np.expm1(np.array([log_alpha[edges[k] + 1:edges[k + 1] + 1].sum() for k in range(K)]))
    return tau, abar, abar_prev, one_minus_ratio


def ddim_tables64(betas, K, eta):
    """fp64 rows {c1, c2, pc1, pc2, var} [K] of respaced DDIM (var = sigma^2).  With u = 1 - abar_k, u' = 1 - abar', m = 1 - abar_k / abar'
    and r = 1 - m, the definitions become sums of positive terms (abar_k = r abar' gives 1 - abar' - sigma^2 = u' (r u' + (1 - eta^2) m) / u):
        sigma^2 = eta^2 u' m / u,   pc2 = S / u with S = sqrt(u' (r u' + (1 - eta^2) m)),
        pc1 = sqrt(abar') - pc2 sqrt(abar_k) = sqrt(abar') m (u + eta^2 r u') / (u (u + sqrt(r) S)),
    so nothing cancels, and K = T, eta = 1 gives the DDPM posterior's own expressions (pc1 = beta sqrt(abar') / u, pc2 = u' sqrt(alpha) / u)
    to rounding.  The last step (k = 0, abar' = 1) is pc1 = 1, pc2 = 0, sigma = 0: it returns x0."""
    _, abar, abar_prev, m = _respaced(betas, K)
    u, up, r, e2 = 1. - abar, 1. - abar_prev, 1. - m, eta * eta
    S = np.sqrt(up * (r * up + (1. - e2) * m))
    pc2 = S / u
    pc1 = np.sqrt(abar_prev) * m * (u + e2 * r * up) / (u * (u + np.sqrt(r) * S))
    pc1[0], pc2[0] = 1., 0.
    return {"c1": np.sqrt(1. / abar), "c2": np.sqrt(1. / abar - 1), "pc1": pc1, "pc2": pc2, "var": e2 * up * m / u}


def dpmpp_2m_tables64(betas, K):
    """fp64 rows {c1, c2, A, B, C} [K] of DPM-Solver++(2M)."""
    _, abar, abar_prev, _ = _respaced(betas, K)
    alpha, sigma = np.sqrt(abar), np.sqrt(1. - abar)
    alpha_p, sigma_p = np.sqrt(abar_prev), np.sqrt(1. - abar_prev)
    lam = np.log(alpha) - np.log(sigma)
    with np.errstate(divide="ignore"):
        lam_p = np.log(alpha_p) - np.log(sigma_p)         # +inf at k = 0
    A, B, C = np.zeros(K), np.zeros(K), np.zeros(K)
    for k in range(1, K):
        h = lam_p[k] - lam[k]
        one_m_eh = -np.expm1(-h)
        A[k] = sigma_p[k] / sigma[k]
        if k == K - 1:
            B[k] = alpha_p[k] * one_m_eh
        else:
            r = (lam_p[k + 1] - lam[k + 1]) / h
            B[k] = alpha_p[k] * one_m_eh * (1. + 1. / (2. * r))
            C[k] = -alpha_p[k] * one_m_eh / (2. * r)
    B[0] = 1.
    return {"c1": np.sqrt(1. / abar), "c2": np.sqrt(1. / abar - 1), "A": A, "B": B, "C": C}


def sampler_schedule(spec, betas, device="cpu"):
    """(buffers, sqrt_alphas_cumprod_prev [K + 1] fp64, solver [3, K] fp32 or None) of a canonical spec (check_sampler_spec) on the trained
    betas: the fp32 rows the native samplers read under the names noise_schedule_buffers gives them (betas = the respaced step's
    1 - abar_k / abar', then sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1, posterior_mean_coef2,
    posterior_log_variance_clipped), ready for Engine.set_schedule and WindowedStreamSampler.add_schedule; `solver` holds A, B, C of
    DPM-Solver++(2M) for WindowedSampler.set_solver."""
    name, K, eta = spec
    to_torch = lambda a: torch.tensor(a, dtype=torch.float32, device=device)
    tau, abar, _, omr = _respaced(betas, K)
    if name == "ddim":
        t = ddim_tables64(betas, K, eta)
        with np.errstate(divide="ignore"):
            logvar = np.log(t["var"])                      # -inf where sigma = 0: exp(0.5 logvar) = 0 exactly
        pc1, pc2, solver = t["pc1"], t["pc2"], None
    else:
        t = dpmpp_2m_tables64(betas, K)
        pc1, pc2, logvar = np.ones(K), np.zeros(K), np.full(K, -np.inf)
        solver = to_torch(np.stack([t["A"], t["B"], t["C"]]))
    bufs = {"betas": to_torch(omr), "sqrt_recip_alphas_cumprod": to_torch(t["c1"]), "sqrt_recipm1_alphas_cumprod": to_torch(t["c2"]),
            "posterior_mean_coef1": to_torch(pc1), "posterior_mean_coef2": to_torch(pc2), "posterior_log_variance_clipped": to_torch(logvar)}
    return bufs, np.sqrt(np.append(1., abar)), solver

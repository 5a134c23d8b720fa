"""Generate tests/golden/sr3_lowres_golden.pt: UNets whose lowest level is 4x4, run by the UNMODIFIED reference (imported from
/root/reference, CPU fp32).  Run once in the build container:

    python tests/golden/make_lowres_golden.py

As in make_golden.py, weights are never stored: both implementations draw them from torch.manual_seed(seed) in the reference's
construction order, checked here bit for bit against oracle.sr3_oracle.init_state_dict before anything is written.  The inputs are not
stored either: tests/_lowres_inputs.py draws them from seeded generators.  The fixture keeps what the tests compare, small: eps and
p_mean_variance of whole images for the small nets, a 16x16 crop for the 16->64 config, the per-layer outputs around the 4x4 level for
one image, and two snapshots of the sampling loop.
"""
import os
import sys

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _lowres_inputs as li  # noqa: E402
from make_golden import build_ref, check_init  # noqa: E402  (puts the reference and the repository on sys.path)


def eps_and_pmv(g, cond, xt, crop=(slice(None),)):
    eps, pmv = {}, {}
    with torch.no_grad():
        for t in li.T_EVAL:
            nl = torch.FloatTensor([g.sqrt_alphas_cumprod_prev[t + 1]]).repeat(xt.shape[0], 1)
            eps[t] = g.denoise_fn(torch.cat([cond, xt], 1) if cond is not None else xt, nl)[crop].clone()
            if cond is not None:
                m, lv = g.p_mean_variance(xt, t, True, condition_x=cond)
                pmv[t] = (m[crop].clone(), lv.clone())
    return eps, pmv


def main():
    out = {}
    # ---- tiny 16x16 net: per-layer outputs around the 4x4 level, eps, p_mean_variance, a 10-step loop, p_losses
    g = build_ref(li.TINY4, 16, 0)
    check_init(g, li.TINY4, 16, 0)
    inp = li.tiny4()
    taps, hooks = {}, []
    for coll in ("downs", "mid", "ups"):
        for i, m in enumerate(getattr(g.denoise_fn, coll)):
            name = f"{coll}.{i}"
            if name in li.TAPS:
                hooks.append(m.register_forward_hook(lambda mod, x, o, n=name: taps.__setitem__(n, o[:1].detach().clone())))
    with torch.no_grad():
        eps = g.denoise_fn(inp["x"], inp["noise_level"]).clone()
    for h in hooks:
        h.remove()
    assert sorted(taps) == sorted(li.TAPS)
    eps_t, pmv = eps_and_pmv(g, inp["cond"], inp["x_t"])
    out["tiny4"] = {"seed": 0, "eps": eps, "taps": taps, "eps_t": eps_t, "pmv": pmv}

    g.set_new_noise_schedule(li.SCHED10, "cpu")
    d = li.tiny4_diffusion()
    draws = iter([d["x_T"]] + [d["noises"][i] for i in reversed(range(1, 10))])
    orig_randn, orig_randn_like = torch.randn, torch.randn_like
    torch.randn = lambda *a, **k: next(draws)
    torch.randn_like = lambda *a, **k: next(draws)
    try:
        with torch.no_grad():
            loop = g.super_resolution(inp["cond"], continous=True)
    finally:
        torch.randn, torch.randn_like = orig_randn, orig_randn_like
    assert loop.shape == (3 * 11, 3, 16, 16)
    np.random.seed(d["np_seed"])
    with torch.no_grad():
        loss = g.p_losses({"HR": d["hr"], "SR": inp["cond"]}, noise=d["noise"])
    # loop snapshots: rows [3 (1 + k), 3 (2 + k)) hold the images after the k-th recorded step; k = 4 (t = 5) and the finished images
    out["tiny4_diffusion"] = {"loop_mid": loop[15:18].clone(), "loop_last": loop[-3:].clone(), "loss": loss.clone()}

    # ---- unconditional 32x32 net with (1, 2, 4, 8)
    g = build_ref(li.UNCOND32, 32, 1, conditional=False)
    check_init(g, li.UNCOND32, 32, 1)
    eps_u, _ = eps_and_pmv(g, None, li.uncond32()["x_t"])
    out["uncond32"] = {"seed": 1, "eps": eps_u}

    # ---- the 16->64 config at batch 2 (16x16 centre crop)
    g = build_ref(li.SR16_64, 64, 0)
    check_init(g, li.SR16_64, 64, 0)
    s = li.sr16_64()
    e64, p64 = eps_and_pmv(g, s["cond"], s["x_t"], li.CROP)
    out["sr16_64"] = {"seed": 0, "eps": e64, "pmv": p64}

    path = os.path.join(HERE, "sr3_lowres_golden.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

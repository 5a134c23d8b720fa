"""Generate tests/golden/sr3_sizes_golden.pt: nets run on images of another size than their image_size (non-square included), by the
UNMODIFIED reference (imported from /root/reference, CPU fp32).  Run once in the build container:

    python tests/golden/make_sizes_golden.py

As in make_golden.py, weights are never stored: both implementations draw them from torch.manual_seed(seed) in the reference's
construction order, checked here bit for bit against oracle.sr3_oracle.init_state_dict before anything is written.  The inputs are not
stored either: tests/_sizes_inputs.py draws them from seeded generators and names the cases.  Per case the fixture keeps eps of one
forward (over the case's crop) and the per-layer outputs of image 0 over small crops; for the 16->128 config at 128x256 also eps and
p_mean_variance at three timesteps and two snapshots of a 10-step sampling loop with injected noise.
"""
import os
import sys

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402

import _sizes_inputs as si  # noqa: E402
from make_golden import build_ref, check_init  # noqa: E402  (puts the reference and the repository on sys.path)


def run_case(name):
    unet, image_size, seed, b, h, w, _, taps_spec = si.CASES[name]
    g = build_ref(unet, image_size, seed)
    check_init(g, unet, image_size, seed)
    inp = si.inputs(name)
    taps, hooks = {}, []
    for coll in ("downs", "mid", "ups"):
        for i, m in enumerate(getattr(g.denoise_fn, coll)):
            layer = f"{coll}.{i}"
            if layer in taps_spec:
                hooks.append(m.register_forward_hook(lambda mod, x, o, n=layer: taps.__setitem__(n, si.tap_crop(name, n, o).clone())))
    with torch.no_grad():
        eps = g.denoise_fn(inp["x"], inp["noise_level"])
    for hk in hooks:
        hk.remove()
    assert eps.shape == (b, 3, h, w) and sorted(taps) == sorted(taps_spec), (eps.shape, sorted(taps))
    out = {"seed": seed, "eps": si.eps_crop(name, eps).clone(), "taps": taps}
    if name != si.LOOP_CASE:
        return out
    out["eps_t"], out["pmv"] = {}, {}
    with torch.no_grad():
        for t in si.T_EVAL:
            nl = torch.FloatTensor([g.sqrt_alphas_cumprod_prev[t + 1]]).repeat(b, 1)
            out["eps_t"][t] = si.eps_crop(name, g.denoise_fn(torch.cat([inp["cond"], inp["x_t"]], 1), nl)).clone()
            m, lv = g.p_mean_variance(inp["x_t"], t, True, condition_x=inp["cond"])
            out["pmv"][t] = (si.eps_crop(name, m).clone(), lv.clone())
    g.set_new_noise_schedule(si.SCHED10, "cpu")
    d = si.loop_inputs()
    draws = iter([d["x_T"]] + [d["noises"][i] for i in reversed(range(1, 10))])
    orig_randn, orig_randn_like = torch.randn, torch.randn_like
    torch.randn = lambda *a, **k: next(draws)
    torch.randn_like = lambda *a, **k: next(draws)
    try:
        with torch.no_grad():
            loop = g.super_resolution(inp["cond"], continous=True)
    finally:
        torch.randn, torch.randn_like = orig_randn, orig_randn_like
    assert loop.shape == (b * 11, 3, h, w), loop.shape
    # rows [b (1 + k), b (2 + k)) hold the images after the k-th recorded step: k = 4 is t = 5; the last b rows are x_0
    out["loop_mid"] = si.eps_crop(name, loop[5 * b:6 * b]).clone()
    out["loop_last"] = si.eps_crop(name, loop[-b:]).clone()
    return out


def main():
    out = {name: run_case(name) for name in si.CASES}
    path = os.path.join(HERE, "sr3_sizes_golden.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

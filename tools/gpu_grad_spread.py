"""Run-to-run spread of the differentiable denoiser's backward next to its error against the oracle, for one case of
tests/_unet_grad_inputs.py.  The backward is not bit-reproducible (fp32 atomics, DESIGN.md §3.6), so a bound on any gradient has to sit
above both.  Runs the case's forward and backward N times (each backward needs its own forward: the engine backpropagates a forward
once) and prints, for every parameter tensor, for dtau per image (sr3_test_train_film_state) and for d noise_level per image:
  * spread: the largest relative L2 difference between run k and run 0;
  * err min / max: the relative L2 error against the oracle's fp32 autograd over the N runs;
and for d noise_level also the conditioned ratio |error| / (||c_b|| ||dtau_b^ref||) of tests/test_gpu_unet_grad.py compare().  The GPU's
name and power limit are printed with it: every number is a measurement on that card.

    python tools/gpu_grad_spread.py [--case tiny_32x32] [--runs 5]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default="tiny_32x32")
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import torch
    import _train_util as tu
    import _unet_grad_inputs as ui
    from test_gpu_noise_level_grad import run
    from test_gpu_unet_grad import build, dnl_bounds, oracle_of

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    net, unet = build(args.case)
    x, nl, G = ui.inputs(args.case)
    b = x.shape[0]
    runs = []
    for _ in range(args.runs):
        dnl, grads, _, st = run(net, x, nl, G)
        grads = dict(grads, **{f"dtau[{i}]": st["dtau"][i] for i in range(b)}, **{f"dnl[{i}]": dnl[i:i + 1] for i in range(b)})
        runs.append(grads)
    r = oracle_of(net, unet, args.case, x, nl, G)
    ref = dict(r[3], **{f"dtau[{i}]": r[4][i] for i in range(b)}, **{f"dnl[{i}]": r[2].view(-1)[i:i + 1] for i in range(b)})
    sd = {k: v.detach().cpu() for k, v in net.denoise_fn.state_dict().items()}
    _, scale = dnl_bounds(sd, nl, r[4])
    print(f"case {args.case}, batch {b}, {args.runs} runs, GPU: {gpu}")
    print(f"{'tensor':60s} {'spread':>9s} {'err min':>9s} {'err max':>9s}")
    rows = []
    for k in ref:
        spread = max(tu.rel(g[k], runs[0][k]) for g in runs[1:]) if len(runs) > 1 else 0.0
        errs = [tu.rel(g[k], ref[k]) for g in runs]
        rows.append((k, spread, min(errs), max(errs)))
    for k, s, lo, hi in sorted(rows, key=lambda row: -row[3]):
        print(f"{k:60s} {s:9.2e} {lo:9.2e} {hi:9.2e}")
    for i in range(b):
        ratios = [abs(float(g[f"dnl[{i}]"]) - float(ref[f"dnl[{i}]"])) / float(scale[i]) for g in runs]
        print(f"dnl[{i}] conditioned |error| / (|c| |dtau|): max {max(ratios):.2e} over {len(ratios)} runs")
    params = [row for row in rows if not row[0].startswith(("dtau[", "dnl["))]
    print(f"parameters: largest spread {max(r[1] for r in params):.2e}, largest error {max(r[3] for r in params):.2e}")


if __name__ == "__main__":
    main()

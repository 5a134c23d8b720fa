"""Generate tests/golden/sr3_unet_grad_golden.pt: gradients of the denoiser alone -- loss = sum(G * denoise_fn(x, noise_level)) for a fixed
seeded upstream gradient G, backpropagated by autograd through the UNMODIFIED reference UNet (CPU fp32) to
x, the noise level and every parameter.  The reference checkout is found as make_golden.py finds it.  Run once:

    python tests/golden/make_unet_grad_golden.py

Weights are never stored: both implementations draw them from torch.manual_seed(seed) in the reference's construction order (train phase:
orthogonal init, checked against the oracle's before anything is written).  Cases and inputs come from tests/_unet_grad_inputs.py.  Per case
the fixture keeps eps, dx and d noise_level whole and a signature (norm, sum, 16 strided samples) of every parameter gradient; for the
Dropout case (train() mode) also the reference's own keep-masks, bit-packed.
"""
import os
import sys

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import _unet_grad_inputs as ui  # noqa: E402
from make_golden import build_ref, check_init  # noqa: E402  (puts the reference and the repository on sys.path)


def run(name, dropout=0.0, torch_seed=None):
    unet, image_size, conditional, b, h, w = ui.CASES[name]
    unet = dict(unet, dropout=dropout)
    g = build_ref(unet, image_size, ui.SEED, conditional=conditional, phase="train")
    check_init(g, unet, image_size, ui.SEED, orthogonal=True)
    net = g.denoise_fn
    net.train(bool(dropout))
    masks, hooks = {}, []
    for mname, m in net.named_modules():
        if isinstance(m, nn.Dropout):
            key = mname[: -len(".block.2")]          # "downs.1.res_block.block2.block.2" -> "downs.1.res_block.block2"

            def hook(mod, inp, outp, key=key):
                keep = (outp != 0) | (inp[0] == 0)     # where the input is 0 the mask is unobservable (and irrelevant)
                masks[key] = keep.clone()
            hooks.append(m.register_forward_hook(hook))
    x, nl, G = ui.inputs(name)
    x.requires_grad_(True)
    nl.requires_grad_(True)
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    eps = net(x, nl)                                   # unet.py:235-259
    (G * eps).sum().backward()
    for hk in hooks:
        hk.remove()
    out = {"eps": eps.detach().clone(), "dx": x.grad.clone(), "dnl": nl.grad.clone(),
           "grads": {k: ui.signature(p.grad) for k, p in net.named_parameters()}}
    if dropout:
        assert len(masks) > 0
        out["p"] = dropout
        out["masks"] = {k: (torch.from_numpy(np.packbits(v.numpy().reshape(-1))), tuple(v.shape)) for k, v in masks.items()}
    print(name, "dropout" if dropout else "", "|eps|", eps.norm().item(), "|dx|", x.grad.norm().item(), "dnl", nl.grad.flatten().tolist(),
          flush=True)
    return out


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {"seed": ui.SEED, "cases": {name: run(name) for name in ui.CASES}}
    name, p, tseed = ui.DROPOUT_CASE
    out["dropout"] = dict(run(name, p, tseed), case=name, torch_seed=tseed)
    path = os.path.join(HERE, "sr3_unet_grad_golden.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

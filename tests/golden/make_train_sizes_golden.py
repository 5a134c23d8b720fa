"""Generate tests/golden/sr3_train_sizes_golden.pt: one training iteration head of DDPM.optimize_parameters (model/model.py:48-53:
p_losses -> sum / (b c h w) -> backward) on images of another size than the net's image_size (non-square included), by the UNMODIFIED
reference (imported from /root/reference, CPU fp32).  Run once in the build container:

    python tests/golden/make_train_sizes_golden.py

As in make_train_golden.py, weights are never stored: both implementations draw them from torch.manual_seed(seed) in the reference's
construction order (train phase: orthogonal init).  Inputs come from tests/_train_sizes_inputs.py.  Per case the fixture keeps the L1 loss
and a signature (norm, sum, 16 strided samples) of every parameter gradient; for the Dropout case also the reference's own keep-masks,
bit-packed.  Each loss is checked against the oracle before anything is written.
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

import _train_sizes_inputs as ti  # noqa: E402
from make_golden import build_ref, check_init  # noqa: E402  (puts the reference and the repository on sys.path)
from oracle import sr3_oracle as orc  # noqa: E402


def oracle_cfg(unet, image_size):
    return orc.UNetConfig(in_channel=unet["in_channel"], out_channel=unet["out_channel"], inner_channel=unet["inner_channel"], norm_groups=32,
                          channel_mults=tuple(unet["channel_multiplier"]), attn_res=tuple(unet["attn_res"]), res_blocks=unet["res_blocks"],
                          dropout=unet["dropout"], image_size=image_size)


def run(name, dropout=0.0, torch_seed=None):
    unet, image_size, b, h, w = ti.CASES[name]
    unet = dict(unet, dropout=dropout)
    g = build_ref(unet, image_size, ti.SEED, phase="train", sched=ti.SCHED)
    check_init(g, unet, image_size, ti.SEED, orthogonal=True)
    g.train()
    masks, hooks = {}, []
    for mname, m in g.denoise_fn.named_modules():
        if isinstance(m, nn.Dropout):
            key = mname[: -len(".block.2")]          # "downs.1.res_block.block2.block.2" -> "downs.1.res_block.block2"

            def hook(mod, inp, outp, key=key):
                keep = (outp != 0) | (inp[0] == 0)     # where the input is 0 the mask is unobservable (and irrelevant)
                masks[key] = keep.clone()
            hooks.append(m.register_forward_hook(hook))
    hr, sr, noise = ti.case_batch(name)
    np.random.seed(ti.NP_SEED)
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    l_pix = g.p_losses({"HR": hr, "SR": sr}, noise=noise)            # diffusion.py:221-246, L1
    l_pix = l_pix.sum() / int(b * 3 * h * w)                            # model/model.py:50-53
    l_pix.backward()
    for hk in hooks:
        hk.remove()
    out = {"loss": l_pix.item(), "grads": {k[len("denoise_fn."):]: ti.signature(p.grad) for k, p in g.named_parameters()}}
    if dropout:
        out["p"] = dropout
        out["masks"] = {k: (torch.from_numpy(np.packbits(v.numpy().reshape(-1))), tuple(v.shape)) for k, v in masks.items()}
    # the oracle's loss on the same draws (and masks) before anything is written
    sch = orc.make_schedule(ti.SCHED)
    _, gamma = orc.draw_gamma(sch, b, np.random.RandomState(ti.NP_SEED))
    om = {k: v.float() / (1.0 - dropout) for k, v in masks.items()} if dropout else None
    sd = orc.init_state_dict(oracle_cfg(unet, image_size), ti.SEED, orthogonal=True)
    with torch.no_grad():
        lo = orc.train_loss(sd, oracle_cfg(unet, image_size), sch, hr, sr, gamma, noise, "l1", om).item()
    print(name, "dropout" if dropout else "", "loss", out["loss"], "oracle", lo, flush=True)
    assert abs(lo - out["loss"]) <= 1e-5 * abs(out["loss"]), (lo, out["loss"])
    return out


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {"sched": ti.SCHED, "seed": ti.SEED, "np_seed": ti.NP_SEED, "cases": {name: run(name) for name in ti.CASES}}
    name, p, tseed = ti.DROPOUT_CASE
    out["dropout"] = dict(run(name, p, tseed), case=name, torch_seed=tseed)
    path = os.path.join(HERE, "sr3_train_sizes_golden.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

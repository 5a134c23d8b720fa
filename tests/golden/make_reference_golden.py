"""Regenerates tests/golden/reference_tiny.pt: what the UNMODIFIED reference computes for the tiny conditional config of
tests/test_oracle.py::test_live_reference_matches_oracle (define_G with torch.manual_seed(11), then p_mean_variance at t = 19, 7, 0).

    python tests/golden/make_reference_golden.py <reference checkout>

Stored: per parameter tensor its shape, fp64 sum and sum of squares and a fixed, seeded sample of 16 values (the full state dict is
megabytes); the inputs and the posterior means / log variances (small)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref_root):
    sys.dont_write_bytecode = True
    sys.path.insert(0, ref_root)
    import model.networks as ref_networks
    sched = {"schedule": "linear", "n_timestep": 20, "linear_start": 1e-6, "linear_end": 1e-2}
    opt = {"phase": "val", "gpu_ids": None, "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False,
                     "unet": dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0),
                     "beta_schedule": {"train": sched, "val": sched},
                     "diffusion": {"image_size": 32, "channels": 3, "conditional": True}}}
    torch.manual_seed(11)
    g = ref_networks.define_G(opt)
    g.set_new_noise_schedule(sched, "cpu")
    g.eval()
    params = {}
    for k, v in g.denoise_fn.state_dict().items():
        flat = v.detach().flatten()
        idx = torch.randint(0, flat.numel(), (16,), generator=torch.Generator().manual_seed(len(k)))
        params[k] = {"shape": tuple(v.shape), "sum": flat.double().sum().item(), "sumsq": (flat.double() ** 2).sum().item(), "idx": idx, "vals": flat[idx].clone()}
    torch.manual_seed(5)
    x, c = torch.randn(3, 3, 32, 32), torch.rand(3, 3, 32, 32) * 2 - 1
    pmv = {}
    with torch.no_grad():
        for t in (19, 7, 0):
            m, lv = g.p_mean_variance(x, t, True, condition_x=c)
            pmv[t] = (m.clone(), float(lv))
    torch.save({"params": params, "x": x, "c": c, "pmv": pmv}, os.path.join(HERE, "reference_tiny.pt"))


if __name__ == "__main__":
    main(sys.argv[1])

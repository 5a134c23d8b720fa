"""CPU-side checks: the C-ABI library loads and exports every symbol of include/sr3_b200.h, the Python mirror reproduces the
reference's state_dict / schedule layout, and the host logic fails loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import sr3_b200
from oracle import sr3_oracle as orc
from sr3_b200 import _native
from sr3_b200.model.sr3_modules import diffusion as diff
from sr3_b200.model.sr3_modules.unet import UNet, layer_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}


def make_opt(unet, image_size, conditional=True, phase="val"):
    return {"phase": phase, "gpu_ids": None, "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}


FULL = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.2)


def test_library_exports_every_header_symbol_and_its_abi_version():
    header = open(os.path.join(ROOT, "include", "sr3_b200.h")).read()
    declared = set(re.findall(r"\b(sr3_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    lib = ctypes.CDLL(_native.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in sr3_b200.h but not exported by the library"
    assert declared == set(_native.EXPORTED_SYMBOLS), declared ^ set(_native.EXPORTED_SYMBOLS)
    assert _native.lib().sr3_abi_version() == 5          # v5: the single-size stream entry points are gone


def test_state_dict_layout_matches_reference_names_and_init():
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt(FULL, 128))
    sd = net.state_dict()
    ref = orc.init_state_dict(orc.UNetConfig(), 0)
    keys = [k for k in sd if k.startswith("denoise_fn.")]
    assert [k[len("denoise_fn."):] for k in keys] == list(ref.keys())
    assert len(keys) == 362 and sum(sd[k].numel() for k in keys) == 97807491
    for k in keys:
        assert torch.equal(sd[k], ref[k[len("denoise_fn."):]]), k
    net.set_loss("cpu")
    assert net.__class__.__name__ == "GaussianDiffusion"


def test_orthogonal_train_phase_init():
    torch.manual_seed(3)
    net = sr3_b200.define_G(make_opt(FULL, 128, phase="train"))
    ref = orc.init_state_dict(orc.UNetConfig(), 3, orthogonal=True)
    for k, v in ref.items():
        assert torch.equal(net.state_dict()["denoise_fn." + k], v), k


def test_schedule_buffers_and_strict_loading(golden_schedules):
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt(dict(FULL, channel_multiplier=[1, 2], res_blocks=1), 32))
    for name, g in golden_schedules.items():
        net.set_new_noise_schedule(g["opt"], "cpu")
        assert net.num_timesteps == g["opt"]["n_timestep"]
        for k, v in g["buffers"].items():
            assert torch.equal(getattr(net, k), v) or torch.allclose(getattr(net, k), v, rtol=0, atol=0, equal_nan=True), (name, k)
        assert np.array_equal(net.sqrt_alphas_cumprod_prev, g["sqrt_alphas_cumprod_prev"].numpy())
    sd = net.state_dict()
    assert len([k for k in sd if not k.startswith("denoise_fn.")]) == 12
    net.load_state_dict(sd, strict=True)
    with pytest.raises(NotImplementedError):
        diff.make_beta_schedule("nope", 10)


def test_layer_table_matches_survey_appendix():
    t = layer_table(6, 64, [1, 2, 4, 8, 8], [16], 2, 128)
    kinds = [(n, k) for n, k, *_ in t]
    assert kinds[:5] == [("downs.0", "conv"), ("downs.1", "res"), ("downs.2", "res"), ("downs.3", "down"), ("downs.4", "res")]
    assert ("ups.18", "res") in kinds and len([k for _, k in kinds if k == "up"]) == 4
    ups = {n: (ci, co, a) for n, k, ci, co, a in t if n.startswith("ups.") and k == "res"}
    assert ups["ups.6"] == (768, 512, True) and ups["ups.16"] == (192, 64, False)
    big = layer_table(6, 64, [1, 2, 4, 8, 16], [], 1, 512)
    assert [x for x in big if x[0] == "ups.0"][0][2:4] == (2048, 1024)


def test_no_cpu_fallback_and_unsupported_variants():
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt(dict(FULL, channel_multiplier=[1, 2], res_blocks=1), 32))
    net.set_new_noise_schedule({"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}, "cpu")
    with pytest.raises(_native.NativeLibraryError):
        net.denoise_fn(torch.zeros(1, 6, 32, 32), torch.zeros(1, 1))          # parameters on CPU -> loud failure
    with pytest.raises(_native.NativeLibraryError):
        net.super_resolution(torch.zeros(1, 3, 32, 32))
    opt = make_opt(FULL, 128)
    opt["model"]["which_model_G"] = "ddpm"
    with pytest.raises(NotImplementedError):
        sr3_b200.define_G(opt)
    with pytest.raises(NotImplementedError):
        UNet(with_noise_level_emb=False)
    # nn.DataParallel (networks.py:113-115) is replaced by one process per GPU: the factory says so instead of wrapping
    opt = make_opt(FULL, 128)
    opt["gpu_ids"], opt["distributed"] = [0, 1], True
    with pytest.raises(NotImplementedError, match="parallel"):
        sr3_b200.define_G(opt)


def test_q_sample_and_helpers_match_oracle():
    torch.manual_seed(0)
    net = sr3_b200.define_G(make_opt(dict(FULL, channel_multiplier=[1, 2], res_blocks=1), 32))
    net.set_new_noise_schedule(SCHED, "cpu")
    sch = orc.make_schedule(SCHED)
    x0, n = torch.randn(2, 3, 8, 8), torch.randn(2, 3, 8, 8)
    g = torch.tensor([0.3, 0.9]).view(-1, 1, 1, 1)
    assert torch.equal(net.q_sample(x0, g, n), orc.q_sample(x0, g, n))
    for t in (0, 7, 1999):
        assert torch.equal(net.predict_start_from_noise(x0, t, n), orc.predict_start_from_noise(sch, x0, t, n))
        m, lv = net.q_posterior(x0, n, t)
        om, olv = orc.q_posterior(sch, x0, n, t)
        assert torch.equal(m, om) and torch.equal(lv, olv)

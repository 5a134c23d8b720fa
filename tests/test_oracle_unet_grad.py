"""Gradients of the denoiser alone on the CPU: the oracle's fp32 autograd (oracle/sr3_oracle.py unet_forward) pinned to the unmodified
reference's in tests/golden/sr3_unet_grad_golden.pt (tests/golden/make_unet_grad_golden.py; cases and inputs in tests/_unet_grad_inputs.py).
tests/test_gpu_unet_grad.py holds the native backward of UNet.forward to the same oracle."""
import os

import numpy as np
import pytest
import torch

import _unet_grad_inputs as ui
from oracle import sr3_oracle as orc
from test_oracle_train import _check_signature

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1e-5


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "sr3_unet_grad_golden.pt"), map_location="cpu", weights_only=False)


def cfg_of(unet, image_size, dropout=0.0):
    return orc.UNetConfig(in_channel=unet["in_channel"], out_channel=unet["out_channel"], inner_channel=unet["inner_channel"], norm_groups=32,
                          channel_mults=tuple(unet["channel_multiplier"]), attn_res=tuple(unet["attn_res"]), res_blocks=unet["res_blocks"],
                          dropout=dropout, image_size=image_size)


def unpack_masks(d):
    """{block: keep mask as 0 / 1 uint8 [B, C, H, W]} of the fixture's bit-packed reference masks."""
    return {k: torch.from_numpy(np.unpackbits(bits.numpy())[: int(np.prod(shape))].reshape(shape).astype(np.uint8))
            for k, (bits, shape) in d["masks"].items()}


def oracle_grads(sd, cfg, x, nl, G, masks=None, p=0.0):
    """eps and the gradients of sum(G * eps) for x, the noise level and every entry of sd (fp32 autograd).  masks: 0 / 1 keep masks."""
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    x = x.detach().clone().requires_grad_(True)
    nl = nl.detach().clone().requires_grad_(True)
    om = None if masks is None else {k: m.float() / (1.0 - p) for k, m in masks.items()}
    eps = orc.unet_forward(sd, cfg, x, nl, dropout_masks=om)
    (G * eps).sum().backward()
    return eps.detach(), x.grad, nl.grad, {k: v.grad for k, v in sd.items()}


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def check_case(rec, name, masks=None, p=0.0):
    unet, image_size, _, _, _, _ = ui.CASES[name]
    cfg = cfg_of(unet, image_size, p)
    sd = orc.init_state_dict(cfg, ui.SEED, orthogonal=True)
    x, nl, G = ui.inputs(name)
    eps, dx, dnl, grads = oracle_grads(sd, cfg, x, nl, G, masks, p)
    assert rel(eps, rec["eps"]) <= TOL
    assert rel(dx, rec["dx"]) <= TOL
    assert dnl.shape == rec["dnl"].shape and rel(dnl, rec["dnl"]) <= TOL, (dnl, rec["dnl"])
    assert set(grads) == set(rec["grads"])
    for k, sig in rec["grads"].items():
        _check_signature(grads[k], sig, TOL)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(ui.CASES))
def test_oracle_unet_gradients_match_reference(golden, name):
    torch.set_num_threads(min(16, torch.get_num_threads()))
    check_case(golden["cases"][name], name)


def test_oracle_unet_gradients_with_reference_dropout_masks(golden):
    """train() mode: the reference's own nn.Dropout masks of one forward, injected into the oracle."""
    d = golden["dropout"]
    masks = unpack_masks(d)
    unet, image_size, _, _, _, _ = ui.CASES[d["case"]]
    downs, mid, ups = orc.unet_topology(cfg_of(unet, image_size))
    assert sorted(masks) == sorted(s.name + ".res_block.block2" for s in downs + mid + ups if s.kind == "res")
    check_case(d, d["case"], masks, d["p"])
    assert rel(d["dx"], golden["cases"][d["case"]]["dx"]) > 1e-3          # the masks matter

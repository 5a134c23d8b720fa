"""Training at image sizes other than a net's image_size (non-square included), on the CPU.

The oracle's loss and gradients (oracle/sr3_oracle.py, fp32 autograd) are pinned to the unmodified reference's in
tests/golden/sr3_train_sizes_golden.pt (tests/golden/make_train_sizes_golden.py, cases and inputs in tests/_train_sizes_inputs.py); the GPU
tests (tests/test_gpu_train_sizes.py) compare the native backward against the same oracle.  Also: the library's training entry point refuses
the sizes the inference plan refuses, with the same message and before it touches a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import _train_sizes_inputs as ti
from oracle import sr3_oracle as orc
from test_oracle_sizes import REFUSED
from test_oracle_train import _check_signature

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "sr3_train_sizes_golden.pt"), map_location="cpu", weights_only=False)


def cfg_of(unet, image_size, dropout=0.0):
    return orc.UNetConfig(in_channel=unet["in_channel"], out_channel=unet["out_channel"], inner_channel=unet["inner_channel"], norm_groups=32,
                          channel_mults=tuple(unet["channel_multiplier"]), attn_res=tuple(unet["attn_res"]), res_blocks=unet["res_blocks"],
                          dropout=dropout, image_size=image_size)


def unpack_masks(d):
    """{block: keep mask as 0 / 1 uint8 [B, C, H, W]} of the fixture's bit-packed reference masks."""
    return {k: torch.from_numpy(np.unpackbits(bits.numpy())[: int(np.prod(shape))].reshape(shape).astype(np.uint8))
            for k, (bits, shape) in d["masks"].items()}


def oracle_step(name, masks=None, p=0.0):
    unet, image_size, b, h, w = ti.CASES[name]
    cfg = cfg_of(unet, image_size, p)
    sd = orc.init_state_dict(cfg, ti.SEED, orthogonal=True)
    for v in sd.values():
        v.requires_grad_(True)
    sch = orc.make_schedule(ti.SCHED)
    _, gamma = orc.draw_gamma(sch, b, np.random.RandomState(ti.NP_SEED))
    hr, sr, noise = ti.case_batch(name)
    om = None if masks is None else {k: m.float() / (1.0 - p) for k, m in masks.items()}
    loss = orc.train_loss(sd, cfg, sch, hr, sr, gamma, noise, "l1", om)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in sd.items()}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", sorted(ti.CASES))
def test_oracle_loss_and_gradients_match_reference(golden, name):
    torch.set_num_threads(min(16, torch.get_num_threads()))
    rec = golden["cases"][name]
    loss, grads = oracle_step(name)
    assert abs(loss - rec["loss"]) <= 2e-6 * abs(rec["loss"]), (loss, rec["loss"])
    assert set(grads) == set(rec["grads"])
    for k, sig in rec["grads"].items():
        _check_signature(grads[k], sig, 2e-4)


def test_oracle_dropout_step_matches_reference(golden):
    """The reference's own Dropout masks at a non-square size: they have the shape of each block2 activation, [B, C, h, w] with h != w."""
    d = golden["dropout"]
    masks = unpack_masks(d)
    unet, image_size, b, h, w = ti.CASES[d["case"]]
    downs, mid, ups = orc.unet_topology(cfg_of(unet, image_size))
    assert sorted(masks) == sorted(s.name + ".res_block.block2" for s in downs + mid + ups if s.kind == "res")
    assert any(m.shape[2] != m.shape[3] for m in masks.values())
    loss, grads = oracle_step(d["case"], masks, d["p"])
    assert abs(loss - d["loss"]) <= 2e-6 * abs(d["loss"]), (loss, d["loss"])
    for k, sig in d["grads"].items():
        _check_signature(grads[k], sig, 2e-4)
    assert abs(loss - golden["cases"][d["case"]]["loss"]) > 1e-5          # the masks matter


@pytest.mark.parametrize("levels,h,w,msg", REFUSED)
def test_training_entry_point_refuses_the_same_sizes_before_touching_a_device(levels, h, w, msg):
    """sr3_engine_create_train_sized applies sr3_engine_create_sized's rule first: the same message, also on a machine without a GPU."""
    from sr3_b200 import _native
    c = _native.UNetConfigC()
    c.in_channel, c.out_channel, c.inner_channel, c.norm_groups, c.n_mults = 6, 3, 64, 32, levels
    for i in range(levels):
        c.channel_mults[i] = 1
    c.res_blocks, c.image_size, c.channels, c.conditional = 1, 16, 3, 1
    h_ = ctypes.c_void_p()
    assert _native.lib().sr3_engine_create_train_sized(ctypes.byref(c), 1, h, w, 0, 0.0, ctypes.byref(h_)) != 0
    err = _native.lib().sr3_last_error().decode()
    assert msg in err and f"{h}x{w}" in err, err
    assert not h_.value


def test_training_sized_entry_point_is_exported():
    from sr3_b200 import _native
    assert "sr3_engine_create_train_sized" in _native.EXPORTED_SYMBOLS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "sr3_engine_create_train_sized")

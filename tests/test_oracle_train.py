"""The training row (SURVEY.md 8f rank 1) of the oracle, pinned to the unmodified reference: loss, gradients of all parameters, three
Adam iterations of DDPM.optimize_parameters (model/model.py:39-58) and a training-mode (Dropout) forward/backward with the reference's
masks.  Fixture: tests/golden/sr3_train_golden.pt (tests/golden/make_train_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import sr3_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def train_golden():
    return torch.load(os.path.join(HERE, "golden", "sr3_train_golden.pt"), weights_only=False)


def _cfg(g, dropout):
    u = g["unet_dropout"] if dropout else g["unet"]
    return orc.UNetConfig(in_channel=u["in_channel"], out_channel=u["out_channel"], inner_channel=u["inner_channel"], norm_groups=32,
                          channel_mults=tuple(u["channel_multiplier"]), attn_res=tuple(u["attn_res"]), res_blocks=u["res_blocks"],
                          dropout=u["dropout"], image_size=g["res"])


def _batch(g, i):
    gen = torch.Generator().manual_seed(1000 + i)
    B, R = g["batch"], g["res"]
    hr = torch.rand(B, 3, R, R, generator=gen) * 2 - 1
    sr = torch.rand(B, 3, R, R, generator=gen) * 2 - 1
    noise = torch.randn(B, 3, R, R, generator=gen)
    return hr, sr, noise


def _check_signature(t, sig, rtol):
    f = t.detach().flatten()
    assert f.numel() == sig["numel"]
    stride = max(1, f.numel() // 16)
    scale = max(sig["norm"] / max(f.numel(), 1) ** 0.5, 1e-12)          # rms of the tensor: absolute floor for tiny entries
    assert abs(f.norm().item() - sig["norm"]) <= rtol * max(sig["norm"], 1e-12) + 1e-12
    assert torch.allclose(f[::stride][:16], sig["samples"], rtol=rtol, atol=rtol * 10 * scale)


def test_three_adam_steps_match_reference(train_golden):
    g = train_golden
    cfg = _cfg(g, False)
    sd = orc.init_state_dict(cfg, g["seed"], orthogonal=True)
    sch = orc.make_schedule(g["sched"])
    opt = orc.make_adam(sd, g["lr"])
    for i, rec in enumerate(g["steps"]):
        hr, sr, noise = _batch(g, i)
        _, gamma = orc.draw_gamma(sch, g["batch"], np.random.RandomState(rec["np_seed"]))
        if i == 0:      # gradients of the first iteration, before the update
            opt.zero_grad()
            loss = orc.train_loss(sd, cfg, sch, hr, sr, gamma, noise)
            loss.backward()
            assert abs(loss.item() - rec["loss"]) <= 1e-6 * abs(rec["loss"])
            assert set(rec["grads"]) == set(sd)
            for k, sig in rec["grads"].items():
                _check_signature(sd[k].grad, sig, 2e-4)
        l = orc.train_step(sd, opt, cfg, sch, hr, sr, gamma, noise)
        assert abs(l - rec["loss"]) <= 2e-6 * abs(rec["loss"]), (i, l, rec["loss"])
    for k, sig in g["params_after"].items():
        _check_signature(sd[k], sig, 1e-5)


def test_training_mode_dropout_forward_backward(train_golden):
    g = train_golden
    d = g["dropout"]
    cfg = _cfg(g, True)
    sd = orc.init_state_dict(cfg, g["seed"], orthogonal=True)
    for v in sd.values():
        v.requires_grad_(True)
    sch = orc.make_schedule(g["sched"])
    masks = {}
    for k, (bits, shape) in d["masks"].items():
        keep = np.unpackbits(bits.numpy())[: int(np.prod(shape))].reshape(shape)
        masks[k] = torch.from_numpy(keep.astype(np.float32)) / (1.0 - d["p"])
    # Dropout sits in block2 of every ResnetBlock and nowhere else (unet.py:100-101)
    downs, mid, ups = orc.unet_topology(cfg)
    assert sorted(masks) == sorted(s.name + ".res_block.block2" for s in downs + mid + ups if s.kind == "res")
    hr, sr, noise = _batch(g, d["batch_index"])
    _, gamma = orc.draw_gamma(sch, g["batch"], np.random.RandomState(d["np_seed"]))
    loss = orc.train_loss(sd, cfg, sch, hr, sr, gamma, noise, dropout_masks=masks)
    assert abs(loss.item() - d["loss"]) <= 1e-6 * abs(d["loss"]), (loss.item(), d["loss"])
    loss.backward()
    for k, sig in d["grads"].items():
        _check_signature(sd[k].grad, sig, 2e-4)
    # and the eval-mode loss differs (the masks matter)
    with torch.no_grad():
        ev = orc.train_loss(sd, cfg, sch, hr, sr, gamma, noise)
    assert abs(ev.item() - d["loss"]) > 1e-5


def test_dgrad_identity_used_by_the_gpu_test():
    """conv3x3(dY, W') with W'[ci, co, r, s] = W[co, ci, 2-r, 2-s] is the data gradient of conv3x3(X, W) (stride 1, pad 1): the
    identity behind tests/test_gpu_kernels.py::test_conv_dgrad_is_the_forward_kernel_on_mirrored_weights, checked on CPU."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 6, 9, 7, generator=g, requires_grad=True)
    w = torch.randn(5, 6, 3, 3, generator=g)
    dy = torch.randn(2, 5, 9, 7, generator=g)
    (ref,) = torch.autograd.grad(F.conv2d(x, w, None, padding=1), x, dy)
    wp = w.flip(2, 3).transpose(0, 1).contiguous()
    assert torch.allclose(F.conv2d(dy, wp, None, padding=1), ref, atol=1e-5, rtol=1e-5)


def test_downsample_dgrad_is_four_parity_phase_convs():
    """The data gradient of the stride-2 Downsample conv (unet.py:68-74) written as four 2x2-tap convolutions on the low-res dY grid, one per
    input-pixel parity (py, px) -- the op shape csrc/train_plan.inc `bwd_downsample` hands to the forward tile kernel, with the kernel-row
    table of `pack_entry` type 3 (csrc/train_kernels.cuh): R(0,0) = none, R(0,1) = 1, R(1,0) = 2, R(1,1) = 0."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 8, 12, generator=g, requires_grad=True)
    w = torch.randn(7, 5, 3, 3, generator=g)
    dy = torch.randn(2, 7, 4, 6, generator=g)
    (ref,) = torch.autograd.grad(F.conv2d(x, w, None, stride=2, padding=1), x, dy)
    R = {(0, 0): None, (0, 1): 1, (1, 0): 2, (1, 1): 0}
    dyp = F.pad(dy, (1, 1, 1, 1))                           # taps reach one low-res pixel outside the grid (zero = TMA out-of-bounds fill)
    out = torch.zeros_like(ref)
    for py in range(2):
        for px in range(2):
            acc = torch.zeros(2, 5, 4, 6)
            for a in range(2):
                for b in range(2):
                    r, s = R[(py, a)], R[(px, b)]
                    if r is None or s is None:
                        continue
                    # tap offset (py - 1 + a, px - 1 + b) on the dY grid
                    sl = dyp[:, :, py + a: py + a + 4, px + b: px + b + 6]
                    acc += torch.einsum("bohw,oc->bchw", sl, w[:, :, r, s])
            out[:, :, py::2, px::2] = acc
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4)


def test_upsample_dgrad_is_one_4x4_stride2_conv():
    """nearest-2x -> conv3x3 (unet.py:58-65): its data gradient (conv-transpose, then the 2x2 sum of the replicated pixels) equals ONE 4x4
    stride-2 convolution over dY, dX[i][j] = sum_{u,v} K[u][v] dY[2i-1+u][2j-1+v], K[u][v] = sum over (e, r): e+2-r = u, (f, s): f+2-s = v of
    W[r][s] -- the kernel `pack_entry` type 4 builds and `bwd_upsample` runs through the parity view."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 5, 6, generator=g, requires_grad=True)
    w = torch.randn(3, 4, 3, 3, generator=g)
    dy = torch.randn(2, 3, 10, 12, generator=g)
    (ref,) = torch.autograd.grad(F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, None, padding=1), x, dy)
    K = torch.zeros(4, 4, 4, 3)                              # [u][v][ci][co]
    for u in range(4):
        for v in range(4):
            for e in range(2):
                r = e + 2 - u
                if not 0 <= r <= 2:
                    continue
                for f in range(2):
                    s = f + 2 - v
                    if 0 <= s <= 2:
                        K[u, v] += w[:, :, r, s].t()
    dyp = F.pad(dy, (1, 1, 1, 1))
    out = torch.zeros_like(ref)
    for u in range(4):
        for v in range(4):
            sl = dyp[:, :, u: u + 10: 2, v: v + 12: 2]        # dY[2i-1+u][2j-1+v] with zero padding
            out += torch.einsum("bohw,co->bchw", sl, K[u, v])
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4)


def test_weight_gradient_is_a_contraction_over_pixels():
    """dW[co][ci][r][s] = sum_p dY[p][co] X[p + (r-1, s-1)][ci] (zero outside the image): the form wgrad_kernel evaluates with both operands
    MN-major; also for the stride-2 conv, whose taps read X at (2 oh + r - 1, 2 ow + s - 1)."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(2)
    for stride in (1, 2):
        x = torch.randn(2, 4, 8, 8, generator=g)
        w = torch.randn(5, 4, 3, 3, generator=g, requires_grad=True)
        oh = 8 // stride
        dy = torch.randn(2, 5, oh, oh, generator=g)
        (ref,) = torch.autograd.grad(F.conv2d(x, w, None, stride=stride, padding=1), w, dy)
        xp = F.pad(x, (1, 1, 1, 1))
        out = torch.zeros_like(ref)
        for r in range(3):
            for s in range(3):
                sl = xp[:, :, r: r + stride * oh: stride, s: s + stride * oh: stride]
                out[:, :, r, s] = torch.einsum("bohw,bchw->oc", dy, sl)
        assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4)

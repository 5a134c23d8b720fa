"""Pins the per-layer fp64 backward reference of tests/_layer_grad_ref.py on the CPU, before any GPU compares against it:

- its forward is _layer_ref's training-plan forward bit for bit, so both references describe the same plan;
- with rounded=False every layer's gradients are fp64 autograd of the oracle's own layer (oracle/sr3_oracle.py), input gradients split at
  the concat, dfilm the per-image sums of the gradient of block1's output (the oracle's block1 bias gradient of that image alone);
- with rounding on, each gradient-rounding point of the backward plan matters: turning any single one off moves its layer's gradients
  by the order of one bf16 rounding."""
import pytest
import torch
import torch.nn.functional as F

import _layer_grad_ref as gref
import _layer_ref as lref
import test_layer_ref as tlr
from oracle import sr3_oracle as orc

NETS = tlr.NETS


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


@pytest.fixture(scope="module", params=sorted(NETS))
def net(request):
    cfg, sd, nl, taps = tlr.oracle_taps(request.param)
    g = torch.Generator().manual_seed(21)
    grads = {tap: torch.randn(taps[tap].shape, generator=g, dtype=torch.float64) for tap, _, _, _, _ in lref.layer_inputs(cfg)}
    keeps = {}
    for tap, kind, spec, _, _ in lref.layer_inputs(cfg):
        if kind == "res":
            keeps[tap] = (torch.rand(taps[tap].shape, generator=g) >= 0.2).double() / 0.8
    return request.param, cfg, sd, nl, taps, grads, keeps


def oracle_layer(sd, cfg, kind, spec, x, skip, nl, keep, gy):
    """fp64 autograd of the oracle's layer: {"x", ("skip"), ("dfilm"), parameter: gradient}."""
    names = gref.layer_params(sd, kind, spec)
    psd = dict(sd)
    psd.update({n: sd[n].clone().requires_grad_(True) for n in names})
    X = x.clone().requires_grad_(True)
    S = None if skip is None else skip.clone().requires_grad_(True)
    g = cfg.norm_groups
    out = {}
    if kind == "conv":
        y = F.conv2d(X, psd["downs.0.weight"], psd["downs.0.bias"], padding=1)
    elif kind == "res":
        p = spec.name + ".res_block"
        xin = X if S is None else torch.cat([X, S], 1)
        t = orc.noise_level_mlp(sd, nl.view(-1, 1), cfg.inner_channel)
        masks = None if keep is None else {p + ".block2": keep}
        y = orc.resnet_block(psd, p, xin, t, g, masks)
        # dfilm[b]: the gradient of block1's conv bias with image b alone
        dfilm = []
        for b in range(x.shape[0]):
            one = dict(sd)
            one[p + ".block1.block.3.bias"] = sd[p + ".block1.block.3.bias"].clone().requires_grad_(True)
            yb = orc.resnet_block(one, p, xin[b:b + 1].detach(), t[b:b + 1], g, None if keep is None else {p + ".block2": keep[b:b + 1]})
            yb.backward(gy[b:b + 1])
            dfilm.append(one[p + ".block1.block.3.bias"].grad)
        out["dfilm"] = torch.stack(dfilm)
    elif kind == "attn":
        y = orc.self_attention(psd, spec.name + ".attn", X, g)
    elif kind == "down":
        y = F.conv2d(X, psd[spec.name + ".conv.weight"], psd[spec.name + ".conv.bias"], stride=2, padding=1)
    elif kind == "up":
        y = F.conv2d(F.interpolate(X, scale_factor=2, mode="nearest"), psd[spec.name + ".conv.weight"], psd[spec.name + ".conv.bias"],
                     padding=1)
    else:
        y = orc.block(psd, "final_conv", X, g)
    y.backward(gy)
    out["x"] = X.grad
    if S is not None:
        out["skip"] = S.grad
    out.update({n: psd[n].grad for n in names})
    return out


def layer_args(cfg, taps, grads, keeps, tap, kind, src, skip):
    gy = grads[tap] if kind != "final" else torch.randn(taps["eps"].shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    return taps[src], None if skip is None else taps[skip], keeps.get(tap), gy


def test_forward_is_the_layer_reference(net):
    name, cfg, sd, nl, taps, grads, keeps = net
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        x, sk, keep, gy = layer_args(cfg, taps, grads, keeps, tap, kind, src, skip)
        got = gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, keep_scale=keep)["out"]
        want = lref.layer_reference(sd, cfg, kind, spec, x, sk, nl, unfused=True, keep_scale=keep)
        assert rel(got, want) < 1e-15, (name, tap, rel(got, want))


def test_unrounded_gradients_are_the_oracle(net):
    name, cfg, sd, nl, taps, grads, keeps = net
    seen = set()
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        x, sk, keep, gy = layer_args(cfg, taps, grads, keeps, tap, kind, src, skip)
        got = gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, keep_scale=keep, rounded=False)
        want = oracle_layer(sd, cfg, kind, spec, x, sk, nl, keep, gy)
        assert set(want) <= set(got), (tap, sorted(set(want) - set(got)))
        for k, v in want.items():
            e = rel(got[k], v)
            assert e < 1e-12, (name, tap, k, e)
        seen.update(gref.layer_params(sd, kind, spec))
    # every parameter is some layer's, except those whose gradients come from dfilm (FiLM projections, block1 conv bias, noise MLP)
    rest = {k for k in sd if k not in seen}
    assert all(k.startswith("noise_level_mlp.") or ".noise_func." in k or k.endswith(".block1.block.3.bias") for k in rest), rest


# one bf16 rounding of a gradient operand moves a layer's gradients by ~2^-9 relative, diluted or summed over the products it enters;
# the attention core's points (P, dS) reach only the q / k / v part of d(qkv): 9e-5 to 8e-4 over 16 to 512 keys
MOVES = (5e-5, 2e-2)


def layer_move(a, b):
    return max(rel(a[k], b[k]) for k in b if k != "out")


def test_every_gradient_rounding_point_matters(net):
    name, cfg, sd, nl, taps, grads, keeps = net
    moves = {}
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        x, sk, keep, gy = layer_args(cfg, taps, grads, keeps, tap, kind, src, skip)
        full = gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, keep_scale=keep)
        m = {pt: layer_move(gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, keep_scale=keep, off=(pt,)), full)
             for pt in gref.POINTS[kind]}
        m["unrounded"] = layer_move(gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, keep_scale=keep, rounded=False), full)
        moves[tap] = m
    print(name, {t: {k: f"{v:.1e}" for k, v in m.items()} for t, m in moves.items()})
    for tap, m in moves.items():
        for k, v in m.items():
            assert MOVES[0] < v < MOVES[1], (name, tap, k, v)


def test_wrong_references_move():
    """The wrong references of the wiring differ from the plan's reference where they should, and only there."""
    cfg, sd, nl, taps = tlr.oracle_taps("tiny_16x16")
    g = torch.Generator().manual_seed(2)
    for tap, kind, spec, src, skip in lref.layer_inputs(cfg):
        gy = torch.randn(taps[tap if kind != "final" else "eps"].shape, generator=g, dtype=torch.float64)
        x, sk = taps[src], None if skip is None else taps[skip]
        ref = gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy)
        for wrong, applies in (("gn_per_source", kind == "res" and sk is not None and x.shape[1] % ((x.shape[1] + sk.shape[1]) // 32) != 0),
                               ("joint_softmax", kind == "attn"), ("per_tap", kind == "up")):
            w = gref.layer_grads(sd, cfg, kind, spec, x, sk, nl, gy, wrong=wrong)
            move = layer_move(w, ref)
            assert (move > 1e-3) if applies else (move < 1e-12), (tap, wrong, move)

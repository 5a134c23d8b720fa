"""fp64 references of the training backward, one layer at a time, as the native plan computes it (train_plan.inc: bwd_res_block,
bwd_attention, bwd_downsample, bwd_upsample, bwd_final, bwd_first_conv), shared by tests/test_layer_grad_ref.py and
tests/test_gpu_layer_grads.py.

layer_grads() takes a layer's input activations (NCHW; in the GPU test the engine's own fp32 taps), the state dict, the noise levels, the
scaled Dropout keep-mask and the gradient of the layer's output, and returns in fp64 the gradient of each input ("x", and "skip" for an
up-path ResnetBlock, split at the concat), every parameter gradient the layer's backward block writes (layer_params) and, for a
ResnetBlock, "dfilm" [B, cout]: the per-image channel sums of dh, the gradient of block1's conv output.

The forward is _layer_ref's training plan in bf16 (operands rounded by _layer_ref.bf, whose backward passes the gradient through), so the
data and weight gradients of each product see the same bf16 operands as the device.  The gradients are rounded where the backward plan
rounds, and nowhere else (GradRound: identity forward, bf16 rounding of the gradient):

  "gy"    y.gb = bf16(y.g), the operand of every data and weight gradient of the layer (for the final block: grad_load_kernel's bf16(deps));
          bias sums, identity shortcuts and the attention residual take the unrounded y.g
  "dh"    ResnetBlock: dh only as bf16 (ghb, the operand of conv1's gradients); dfilm from the unrounded sums
  "dO"    attention: dO is bf16 only
  "P"     attention: softmax_bwd_kernel uses the bf16 P the forward kept, dS = P (dP - sum_k P dP), segments of HW keys
  "dS"    attention: dS rounded to bf16 (after the 1 / sqrt(C) scale) before dQ = dS K and dK = dS^T Q
  "dqkv"  attention: d(qkv) rounded to bf16 before the qkv data and weight gradients
Upsample's data gradient is the 4x4 stride-2 conv with weights bf16(fp32 sum of the aliased taps) (the folded forward differentiated);
its weight gradient contracts bf16(y.g) with bf16 of the nearest-2x input.

rounded=False turns every rounding off (plain fp64); off={points} turns single gradient-rounding points off.  wrong= selects a wrong
reference of the wiring: "gn_per_source" (GroupNorm statistics of a group that straddles the concat taken per source), "joint_softmax"
(the softmax, forward and backward, over the whole 128-token attention batch instead of per image), "per_tap" (the Upsample data
gradient with per-tap rounded weights), "gn_neighbour" (every GroupNorm of the layer, forward and backward, with the statistics of image
(b + 1) mod B for image b: _layer_ref's gn_stats)."""
import math

import torch
import torch.nn.functional as F

import _layer_ref as lref

POINTS = {"conv": ("gy",), "res": ("gy", "dh"), "attn": ("gy", "dO", "P", "dS", "dqkv"), "down": ("gy",), "up": ("gy",), "final": ("gy",)}


class GradRound(torch.autograd.Function):
    """Identity forward; the gradient is rounded to bf16 on its way back."""
    @staticmethod
    def forward(ctx, v):
        return v.clone()

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


class SoftmaxRoundedP(torch.autograd.Function):
    """P = bf16(softmax(s)) as the training forward keeps it; backward dS = P' (dP - sum_k P' dP) with P' the bf16 P (rounded_p) or the
    unrounded softmax."""
    @staticmethod
    def forward(ctx, s, rounded_p):
        p = torch.softmax(s, -1)
        pb = p.to(torch.bfloat16).to(p.dtype)
        ctx.save_for_backward(pb if rounded_p else p)
        return pb

    @staticmethod
    def backward(ctx, dp):
        p, = ctx.saved_tensors
        return p * (dp - (p * dp).sum(-1, keepdim=True)), None


def layer_params(sd, kind, spec):
    """The parameters whose gradients the layer's backward block writes (block1's conv bias and the FiLM projection come from dfilm)."""
    if kind == "conv":
        return ["downs.0.weight", "downs.0.bias"]
    if kind == "res":
        p = spec.name + ".res_block"
        names = [p + s for s in (".block1.block.0.weight", ".block1.block.0.bias", ".block1.block.3.weight", ".block2.block.0.weight",
                                 ".block2.block.0.bias", ".block2.block.3.weight", ".block2.block.3.bias")]
        return names + ([p + ".res_conv.weight", p + ".res_conv.bias"] if p + ".res_conv.weight" in sd else [])
    if kind == "attn":
        return [spec.name + ".attn" + s for s in (".norm.weight", ".norm.bias", ".qkv.weight", ".out.weight", ".out.bias")]
    if kind in ("down", "up"):
        return [spec.name + ".conv.weight", spec.name + ".conv.bias"]
    return ["final_conv.block.0.weight", "final_conv.block.0.bias", "final_conv.block.3.weight", "final_conv.block.3.bias"]


def _leaf(t, device):
    return t.detach().to(device=device, dtype=torch.float64).clone().requires_grad_(True)


def gn_per_source(x, c0, gamma, beta, groups):
    """GroupNorm of x = cat(s0, s1) with the statistics of the group that straddles the concat taken over each source separately (wrong)."""
    C = x.shape[1]
    gs = C // groups
    gid = torch.arange(C) // gs
    if c0 % gs:
        gid[c0:] = torch.where(gid[c0:] == c0 // gs, torch.full_like(gid[c0:], groups), gid[c0:])
    m = F.one_hot(gid, groups + 1).to(x)                                   # [C, groups + 1]
    cnt = m.sum(0) * x.shape[2] * x.shape[3]
    mean = torch.einsum("bchw,cg->bg", x, m) / cnt.clamp_min(1)
    xc = x - (mean @ m.T)[:, :, None, None]
    var = torch.einsum("bchw,cg->bg", xc * xc, m) / cnt.clamp_min(1)
    return xc / torch.sqrt(var @ m.T + lref.EPS)[:, :, None, None] * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)


def layer_grads(sd, cfg, kind, spec, x, skip, nl, gy, keep_scale=None, rounded=True, off=(), wrong=None):
    """Gradients of one entry of _layer_ref.layer_inputs, given its input activations and the gradient gy of its output (for the final
    block: the upstream gradient of eps).  -> {"x", ("skip"), ("dfilm"), parameter name: gradient, "out": the forward output}, fp64."""
    dev = x.device
    names = layer_params(sd, kind, spec)
    psd = dict(sd)
    psd.update({n: _leaf(sd[n], dev) for n in names})
    X = _leaf(x, dev)
    S = None if skip is None else _leaf(skip, dev)

    def r(v):                                  # a forward bf16 operand
        return lref.bf(v) if rounded else v

    def gr(v, point):                          # a gradient-rounding point of the backward
        return GradRound.apply(v) if rounded and point not in off else v

    def conv(a, name, pad, stride=1):
        return F.conv2d(r(a), r(psd[name]), stride=stride, padding=pad)

    def bias(name):
        return psd[name].view(1, -1, 1, 1)

    out, extra, g = None, {}, cfg.norm_groups
    st = lref.neighbour(x.shape[0]) if wrong == "gn_neighbour" else None
    if kind == "conv":
        out = gr(conv(X, "downs.0.weight", 1), "gy") + bias("downs.0.bias")
    elif kind == "res":
        p = spec.name + ".res_block"
        xin = X if S is None else torch.cat([X, S], 1)
        if wrong == "gn_per_source":
            n1 = gn_per_source(xin, X.shape[1], psd[p + ".block1.block.0.weight"], psd[p + ".block1.block.0.bias"], g)
        else:
            n1 = lref._gn(xin, psd, p + ".block1.block.0", g, st)
        film = _leaf(lref.film_rows(sd, p, nl, cfg.inner_channel), dev)
        extra["film"] = film
        h = gr(conv(lref._silu(n1), p + ".block1.block.3.weight", 1), "dh") + film[:, :, None, None]
        a2 = lref._silu(lref._gn(h, psd, p + ".block2.block.0", g, st))
        if keep_scale is not None:
            a2 = a2 * keep_scale.to(dev, torch.float64)
        br = conv(a2, p + ".block2.block.3.weight", 1)
        if p + ".res_conv.weight" in sd:
            out = gr(br + conv(xin, p + ".res_conv.weight", 0), "gy") + bias(p + ".block2.block.3.bias") + bias(p + ".res_conv.bias")
        else:
            out = gr(br, "gy") + bias(p + ".block2.block.3.bias") + X
    elif kind == "attn":
        p = spec.name + ".attn"
        B, C, H, W = X.shape
        HW = H * W
        qkv = gr(conv(lref._gn(X, psd, p + ".norm", g, st), p + ".qkv.weight", 0), "dqkv").view(B, 3, C, HW).transpose(2, 3)
        q, k, v = r(qkv[:, 0]), r(qkv[:, 1]), r(qkv[:, 2])             # [B, HW, C]
        per = max(1, 128 // HW) if wrong == "joint_softmax" else 1     # images sharing one softmax
        os = []
        for b0 in range(0, B, per):
            qs, ks, vs = (t[b0:b0 + per].reshape(1, -1, C) for t in (q, k, v))
            s = gr(qs @ ks.transpose(1, 2), "dS") / math.sqrt(C)
            pm = SoftmaxRoundedP.apply(s, "P" not in off) if rounded else torch.softmax(s, -1)
            os.append((pm @ vs).reshape(-1, HW, C))
        o = gr(r(torch.cat(os, 0)), "dO").transpose(1, 2).reshape(B, C, H, W)
        out = gr(conv(o, p + ".out.weight", 0), "gy") + bias(p + ".out.bias") + X
    elif kind == "down":
        out = gr(conv(X, spec.name + ".conv.weight", 1, 2), "gy") + bias(spec.name + ".conv.bias")
    elif kind == "up":
        w, b = spec.name + ".conv.weight", spec.name + ".conv.bias"
        # the weight and bias gradients: bf16(y.g) against bf16 of the nearest-2x input (the forward's up_x copy)
        yw = gr(conv(F.interpolate(X.detach(), scale_factor=2, mode="nearest"), w, 1), "gy") + bias(b)
        yw.backward(gy.to(dev, torch.float64))
        # the data gradient: the folded forward's transpose, weights bf16(fp32 sums of the aliased taps); "per_tap": each tap rounded
        if wrong == "per_tap":
            out = gr(F.conv2d(r(F.interpolate(X, scale_factor=2, mode="nearest")), r(psd[w].detach()), padding=1), "gy")
        else:
            wd = sd[w].to(dev)
            B, C, h, wdt = X.shape
            parts = []
            for ph, wf in enumerate(lref.folded_weights(wd.to(torch.float32) if rounded else wd.to(torch.float64))):
                py, px = ph >> 1, ph & 1
                parts.append(F.conv2d(F.pad(r(X), (1, 1, 1, 1)), r(wf))[:, :, py:py + h, px:px + wdt])
            # interleave the four phases: out[:, :, 2 i + py, 2 j + px] = parts[2 py + px][:, :, i, j]
            out = torch.stack(parts, 2).view(B, -1, 2, 2, h, wdt).permute(0, 1, 4, 2, 5, 3).reshape(B, -1, 2 * h, 2 * wdt)
            out = gr(out, "gy")
        out.backward(gy.to(dev, torch.float64))
        res = {"x": X.grad, "out": (out + bias(b)).detach()}
        res.update({n: psd[n].grad for n in names})
        return res
    else:
        a = lref._silu(lref._gn(X, psd, "final_conv.block.0", g, st))
        out = gr(conv(a, "final_conv.block.3.weight", 1), "gy") + bias("final_conv.block.3.bias")
    out.backward(gy.to(dev, torch.float64))
    res = {"out": out.detach()}
    if S is None:
        res["x"] = X.grad
    else:
        res["x"], res["skip"] = X.grad, S.grad
    if "film" in extra:
        res["dfilm"] = extra["film"].grad
    res.update({n: psd[n].grad for n in names})
    return res


def passthrough(kind, spec, sd):
    """Whether the layer adds its output gradient y.g unrounded to its input's (identity-shortcut ResnetBlock, attention): input gradients
    are measured on the rest, the branch."""
    return kind == "attn" or (kind == "res" and spec.name + ".res_block.res_conv.weight" not in sd)

"""fp64 references of the UNet's layers as the native plan computes them, shared by tests/test_layer_ref.py and tests/test_gpu_layers.py.

Each function takes a layer's input activations (NCHW; in the GPU test the engine's own fp32 taps), the state dict and the noise levels,
and returns the layer's output in fp64.  bf16 rounding is applied where the plan (engine.cu: build_plan, add_res_block, add_attention)
makes a bf16 operand, and nowhere else:

  first conv      conv3x3(bf16(cat(cond, x)), bf16 W) + b                                   (load_nchw_kernel)
  ResnetBlock     a1 = bf16(silu(GN(cat(x, skip))))                                         (prep_kernel, groups may straddle the concat)
                  h  = conv3x3(a1, bf16 W1) + film[b],  film = W_f tau(nl) + b_f + block1.bias  (film_kernel folds block1's bias in)
                  a2 = bf16(silu(GN(h)) [* scaled keep-mask])                               (prep_kernel<true> in the training plan)
                  y  = conv3x3(a2, bf16 W2) + conv1x1(bf16(cat(x, skip)), bf16 W_res) + (b2 + b_res)   if cin != cout (one GEMM)
                  y  = conv3x3(a2, bf16 W2) + b2 + x                                        otherwise
  SelfAttention   n = bf16(GN(y)); q | k and v = bf16 of the fp32 projection; the fused core as _attention_ref (<= 256 tokens) or
                  _attention_long_ref (streaming, above); out = conv1x1(O, bf16 W_out) + b_out + y.  Images attend within themselves only
                  (at 8x8 two, at 4x4 eight images share one 128-token attention batch).
  Downsample      conv3x3 stride 2 on bf16(previous output) (the epilogue's bf16 copy)
  Upsample        the four-phase folded conv on bf16(previous output), weights bf16(fp32 sum of the aliased 3x3 taps) (pack_entry type 5)
  final block     conv3x3(bf16(silu(GN(x))), bf16 W) + b

precision="fp32" (precise mode): every bf16(v) becomes the pair hi = bf16(v), lo = bf16(v - hi), weights too, and a product is
hi.hi + hi.lo + lo.hi.  Attention is then unfused: S fp32, P the pair of the fp32 softmax (softmax_kernel), O the pair of P v.
unfused=True (the training plan in bf16): P = bf16(softmax), O = bf16(P v).

rounded=False turns every rounding off: what is left is plain fp64 arithmetic of the layer.

gn_stats (a wrong reference): every GroupNorm of the layer normalises image b with the statistics of image gn_stats[b] (neighbour(B):
those of image (b + 1) mod B), what a per-image statistics run restarted at the wrong row would give.  With the identity it is the
default reference bit for bit.

The functions run on the device of their inputs (the GPU test keeps its fp64 references on the GPU)."""
import math

import torch
import torch.nn.functional as F

import _attention_long_ref as lr
import _attention_ref as ar
from oracle import sr3_oracle as orc

EPS = 1e-5


def state_dict(cfg, seed):
    """The reference's initial weights (orc.init_state_dict) with every GroupNorm's affine parameters drawn away from (1, 0), so that a
    layer reading another layer's gamma or beta shows."""
    sd = orc.init_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(seed + 7)
    for k in sd:
        if k.endswith((".norm.weight", ".block.0.weight")):
            sd[k] = 1.0 + 0.25 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith((".norm.bias", ".block.0.bias")):
            sd[k] = 0.25 * torch.randn(sd[k].shape, generator=g)
    return sd


class _Round(torch.autograd.Function):
    """bf16 rounding of an operand, with the pass-through backward of the plan's gradients: a product's gradient reaches the unrounded
    value it was rounded from (tests/_layer_grad_ref.py differentiates these functions)."""
    @staticmethod
    def forward(ctx, v):
        ctx.dtype = v.dtype
        return v.to(torch.bfloat16).to(torch.float64)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dtype)


def bf(v):
    return _Round.apply(v)


def operand(v, mode):
    """The terms an operand enters a product as: [v] unrounded, [bf16(v)], or the precise pair [hi, lo]."""
    v = v.to(torch.float64)
    if mode is None:
        return [v]
    hi = bf(v)
    return [hi] if mode == "bf16" else [hi, bf(v - hi)]


def product(f, a, w, mode):
    """Bilinear f of two operands: one product, or in precise mode hi.hi + hi.lo + lo.hi."""
    A, W = operand(a, mode), operand(w, mode)
    if len(A) == 1:
        return f(A[0], W[0])
    return f(A[0], W[0]) + f(A[0], W[1]) + f(A[1], W[0])


def _mode(precision, rounded):
    assert precision in ("bf16", "fp32"), precision
    return precision if rounded else None


def _p(sd, name, like):
    return sd[name].to(device=like.device, dtype=torch.float64)


def _gn(x, sd, prefix, groups, stats=None):
    """GroupNorm of x; stats: image b normalised with the mean and variance of image stats[b] (a wrong reference).  That is GroupNorm of
    the stats image plus the difference of the two images in its scale, an exact zero for stats[b] == b."""
    gamma, beta = _p(sd, prefix + ".weight", x), _p(sd, prefix + ".bias", x)
    if stats is None:
        return F.group_norm(x, groups, gamma, beta, eps=EPS)
    xs = x[list(stats)]
    B, C = x.shape[:2]
    rstd = torch.rsqrt(xs.reshape(B, groups, -1).var(-1, unbiased=False) + EPS).repeat_interleave(C // groups, 1)
    return F.group_norm(xs, groups, gamma, beta, eps=EPS) + (x - xs) * (rstd * gamma)[:, :, None, None]


def neighbour(b):
    """The GroupNorm statistics of image (i + 1) mod b for image i (gn_stats)."""
    return [(i + 1) % b for i in range(b)]


def _silu(x):
    return x * torch.sigmoid(x)


def _conv(pad, stride=1):
    return lambda a, w: F.conv2d(a, w, stride=stride, padding=pad)


def _bias(sd, name, like):
    return _p(sd, name, like).view(1, -1, 1, 1)


def first_conv(sd, x, precision="bf16", rounded=True):
    """downs.0 on the UNet input x [B, in_channel, H, W] (cat(cond, x_t) for a conditional net)."""
    x = x.to(torch.float64)
    return product(_conv(1), x, _p(sd, "downs.0.weight", x), _mode(precision, rounded)) + _bias(sd, "downs.0.bias", x)


def film_rows(sd, prefix, noise_level, inner):
    """film[b] of ResnetBlock `prefix` ("downs.1.res_block"): W_f tau(nl_b) + b_f + block1.bias, [B, cout] in fp64."""
    nl = noise_level.to(torch.float64).view(-1, 1)
    sd64 = {k: sd[k].to(device=nl.device, dtype=torch.float64) for k in sd if k.startswith("noise_level_mlp.")}
    tau = orc.noise_level_mlp(sd64, nl, inner).view(nl.shape[0], inner)
    return (tau @ _p(sd, prefix + ".noise_func.noise_func.0.weight", nl).T + _p(sd, prefix + ".noise_func.noise_func.0.bias", nl)
            + _p(sd, prefix + ".block1.block.3.bias", nl))


def res_block(sd, prefix, x, skip, film, groups, precision="bf16", rounded=True, keep_scale=None, gn_stats=None):
    """ResnetBlock `prefix` on x [B, C0, H, W] (+ skip [B, C1, H, W]); film [B, cout] from film_rows; keep_scale: the scaled Dropout
    keep-mask [B, cout, H, W] of block2 (training plan), or None."""
    mode = _mode(precision, rounded)
    x = x.to(torch.float64)
    xin = x if skip is None else torch.cat([x, skip.to(torch.float64)], 1)
    a1 = _silu(_gn(xin, sd, prefix + ".block1.block.0", groups, gn_stats))
    h = product(_conv(1), a1, _p(sd, prefix + ".block1.block.3.weight", x), mode) + film.to(x.device, torch.float64)[:, :, None, None]
    a2 = _silu(_gn(h, sd, prefix + ".block2.block.0", groups, gn_stats))
    if keep_scale is not None:
        a2 = a2 * keep_scale.to(x.device, torch.float64)
    y = product(_conv(1), a2, _p(sd, prefix + ".block2.block.3.weight", x), mode) + _bias(sd, prefix + ".block2.block.3.bias", x)
    if prefix + ".res_conv.weight" in sd:
        return y + product(_conv(0), xin, _p(sd, prefix + ".res_conv.weight", x), mode) + _bias(sd, prefix + ".res_conv.bias", x)
    return y + x


def attention(sd, prefix, y, groups, precision="bf16", rounded=True, unfused=False, gn_stats=None):
    """SelfAttention `prefix` ("mid.0.attn") on its ResnetBlock's output y [B, C, H, W]."""
    mode = _mode(precision, rounded)
    y = y.to(torch.float64)
    B, C, H, W = y.shape
    n = _gn(y, sd, prefix + ".norm", groups, gn_stats)
    qkv = product(_conv(0), n, _p(sd, prefix + ".qkv.weight", y), mode).view(B, 3, C, H * W).transpose(2, 3)    # [B, 3, HW, C]
    q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
    if mode == "bf16" and not unfused:
        qk, vb = bf(torch.cat([q, k], 2)).cpu(), bf(v).cpu()      # (the attention references build their masks on the CPU)
        o = ar.fused_reference(qk, vb, H * W, H * W, C) if H * W <= 256 else lr.streaming_reference(qk, vb, C)
        o = o.to(y.device)
    else:
        s = product(lambda a, b: a @ b.transpose(1, 2), q, k, mode) / math.sqrt(C)
        o = product(lambda a, b: a @ b, torch.softmax(s, -1), v, mode)
    o = o.transpose(1, 2).reshape(B, C, H, W)
    return product(_conv(0), o, _p(sd, prefix + ".out.weight", y), mode) + _bias(sd, prefix + ".out.bias", y) + y


def downsample(sd, name, x, precision="bf16", rounded=True):
    x = x.to(torch.float64)
    return product(_conv(1, 2), x, _p(sd, name + ".conv.weight", x), _mode(precision, rounded)) + _bias(sd, name + ".conv.bias", x)


# kernel rows (columns) of a 3x3 conv on the nearest-2x image that land on low-res row offset a for output parity p: ROWS[p][a]
ROWS = (((0,), (1, 2)), ((0, 1), (2,)))


def folded_weights(w):
    """[phase = 2 py + px] -> [Cout, Cin, 2, 2]: the aliased taps summed in w's dtype, in pack_entry's order (rows outer, columns inner,
    from zero), so an fp32 w gives the packer's fp32 sums bit for bit."""
    out = []
    for py in (0, 1):
        for px in (0, 1):
            wf = torch.zeros(*w.shape[:2], 2, 2, dtype=w.dtype, device=w.device)
            for a in (0, 1):
                for b in (0, 1):
                    acc = torch.zeros_like(w[:, :, 0, 0])
                    for r in ROWS[py][a]:
                        for s in ROWS[px][b]:
                            acc = acc + w[:, :, r, s]
                    wf[:, :, a, b] = acc
            out.append(wf)
    return out


def upsample(sd, name, x, precision="bf16", rounded=True, fold=True):
    """Upsample `name` (nearest 2x, conv3x3) on x [B, C, h, w].  fold=False: conv3x3 of the upsampled operand with per-tap rounded weights
    (a wrong reference for the folded plan: it rounds each 3x3 tap instead of their fp32 sums)."""
    mode = _mode(precision, rounded)
    x = x.to(torch.float64)
    w = sd[name + ".conv.weight"].to(x.device)
    b = _bias(sd, name + ".conv.bias", x)
    if not fold:
        return product(lambda a, ww: F.conv2d(F.interpolate(a, scale_factor=2, mode="nearest"), ww, padding=1), x, w, mode) + b
    B, C, h, wd = x.shape
    out = torch.empty(B, w.shape[0], 2 * h, 2 * wd, dtype=torch.float64, device=x.device)
    # unrounded: the exact sums (fp64); rounded: the fp32 sums the packer forms, then rounded once
    phases = folded_weights(w.to(torch.float64) if mode is None else w.to(torch.float32))
    for ph, wf in enumerate(phases):
        py, px = ph >> 1, ph & 1
        o = product(lambda a, ww: F.conv2d(F.pad(a, (1, 1, 1, 1)), ww), x, wf, mode)
        out[:, :, py::2, px::2] = o[:, :, py:py + h, px:px + wd]
    return out + b


def final_block(sd, x, groups, precision="bf16", rounded=True, gn_stats=None):
    x = x.to(torch.float64)
    a = _silu(_gn(x, sd, "final_conv.block.0", groups, gn_stats))
    return product(_conv(1), a, _p(sd, "final_conv.block.3.weight", x), _mode(precision, rounded)) + _bias(sd, "final_conv.block.3.bias", x)


def layer_inputs(cfg):
    """The plan's layers in order: [(tap, kind, spec, input tap, skip tap)] with kind "conv" | "res" | "attn" | "down" | "up" | "final";
    "input" is the UNet input, the res block of an attention layer is tapped as "<layer>.res_block", skips are popped in the plan's order."""
    downs, mid, ups = orc.unet_topology(cfg)
    out, feats, prev = [], [], "input"
    for spec in downs + mid + ups:
        skip = feats.pop() if spec.name.startswith("ups.") and spec.kind == "res" else None
        if spec.kind == "res":
            rb = spec.name + ".res_block" if spec.attn else spec.name
            out.append((rb, "res", spec, prev, skip))
            if spec.attn:
                out.append((spec.name, "attn", spec, rb, None))
        else:
            out.append((spec.name, spec.kind, spec, prev, None))
        prev = spec.name
        if spec.name.startswith("downs."):
            feats.append(spec.name)
    out.append(("eps", "final", None, prev, None))
    return out


def layer_reference(sd, cfg, kind, spec, x, skip, nl, precision="bf16", rounded=True, unfused=False, keep_scale=None, film=None, gn_stats=None):
    """One entry of layer_inputs evaluated on the given input (and skip) activations."""
    g = cfg.norm_groups
    if kind == "conv":
        return first_conv(sd, x, precision, rounded)
    if kind == "res":
        p = spec.name + ".res_block"
        if film is None:
            film = film_rows(sd, p, nl, cfg.inner_channel)
        return res_block(sd, p, x, skip, film, g, precision, rounded, keep_scale, gn_stats)
    if kind == "attn":
        return attention(sd, spec.name + ".attn", x, g, precision, rounded, unfused, gn_stats)
    if kind == "down":
        return downsample(sd, spec.name, x, precision, rounded)
    if kind == "up":
        return upsample(sd, spec.name, x, precision, rounded)
    return final_block(sd, x, g, precision, rounded, gn_stats)


def residual(kind, spec, sd, x):
    """The un-rounded input a layer adds to its output (x of an identity-shortcut ResnetBlock, y of an attention layer), else None: errors
    are measured against the rest (the branch), which the residual can outweigh many times over."""
    if kind == "attn" or (kind == "res" and spec.name + ".res_block.res_conv.weight" not in sd):
        return x.to(torch.float64)
    return None

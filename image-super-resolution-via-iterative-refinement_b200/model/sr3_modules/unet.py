"""Host-side mirror of the reference's denoiser `UNet` (model/sr3_modules/unet.py:161-259).

Unlike the reference this is NOT a tree of torch.nn layers: it is a flat parameter store whose `state_dict()` has exactly
the reference's keys / shapes (so public `*_gen.pth` checkpoints load with strict=True) plus a handle to the native
engine that executes the whole forward as hand-written sm_90a kernels.  `forward(x, time)` has the reference signature.
"""
import math
from typing import Dict, List, Tuple

import torch
from torch import nn

from ... import _native


def layer_table(in_channel, inner_channel, channel_mults, attn_res, res_blocks, image_size):
    """Top-level layers in construction order: (name, kind, cin, cout, with_attn).  Follows unet.py:186-231."""
    mults = list(channel_mults)
    attn_res = tuple(attn_res) if not isinstance(attn_res, int) else (attn_res,)
    layers: List[Tuple[str, str, int, int, bool]] = []
    pre, feats, res = inner_channel, [inner_channel], image_size
    layers.append(("downs.0", "conv", in_channel, inner_channel, False))
    nd = 1
    for lvl, m in enumerate(mults):
        ch = inner_channel * m
        for _ in range(res_blocks):
            layers.append((f"downs.{nd}", "res", pre, ch, res in attn_res))
            nd += 1
            feats.append(ch)
            pre = ch
        if lvl != len(mults) - 1:
            layers.append((f"downs.{nd}", "down", pre, pre, False))
            nd += 1
            feats.append(pre)
            res //= 2
    layers.append(("mid.0", "res", pre, pre, True))
    layers.append(("mid.1", "res", pre, pre, False))
    nu = 0
    for lvl in reversed(range(len(mults))):
        ch = inner_channel * mults[lvl]
        for _ in range(res_blocks + 1):
            layers.append((f"ups.{nu}", "res", pre + feats.pop(), ch, res in attn_res))
            nu += 1
            pre = ch
        if lvl != 0:
            layers.append((f"ups.{nu}", "up", pre, pre, False))
            nu += 1
            res *= 2
    return layers


def parameter_table(in_channel, out_channel, inner_channel, channel_mults, attn_res, res_blocks, image_size):
    """[(state_dict key, shape, init kind)] in the reference's registration order."""
    tab: List[Tuple[str, Tuple[int, ...], str]] = []

    def dense(name, shape, bias=True):
        tab.append((name + ".weight", shape, "w"))
        if bias:
            tab.append((name + ".bias", (shape[0],), "b"))

    def norm(name, c):
        tab.append((name + ".weight", (c,), "one"))
        tab.append((name + ".bias", (c,), "zero"))

    dense("noise_level_mlp.1", (inner_channel * 4, inner_channel))
    dense("noise_level_mlp.3", (inner_channel, inner_channel * 4))
    for name, kind, cin, cout, attn in layer_table(in_channel, inner_channel, channel_mults, attn_res, res_blocks, image_size):
        if kind == "conv":
            dense(name, (cout, cin, 3, 3))
        elif kind in ("down", "up"):
            dense(name + ".conv", (cout, cin, 3, 3))
        else:
            rb = name + ".res_block"
            dense(rb + ".noise_func.noise_func.0", (cout, inner_channel))
            norm(rb + ".block1.block.0", cin)
            dense(rb + ".block1.block.3", (cout, cin, 3, 3))
            norm(rb + ".block2.block.0", cout)
            dense(rb + ".block2.block.3", (cout, cout, 3, 3))
            if cin != cout:
                dense(rb + ".res_conv", (cout, cin, 1, 1))
            if attn:
                norm(name + ".attn.norm", cout)
                dense(name + ".attn.qkv", (cout * 3, cout, 1, 1), bias=False)
                dense(name + ".attn.out", (cout, cout, 1, 1))
    norm("final_conv.block.0", inner_channel)
    dense("final_conv.block.3", (out_channel, inner_channel, 3, 3))
    return tab


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's dotted state_dict names."""


class _UNetFn(torch.autograd.Function):
    """UNet.forward as one autograd node on a training engine: forward = sr3_train_unet_forward (every intermediate kept), backward =
    sr3_train_unet_backward from the upstream gradient of eps -> gradients of x, of the noise level and of every parameter."""

    @staticmethod
    def forward(ctx, unet, eng, x, time, seed, *params):
        eps, ctx.fwd = eng.train_unet_forward(x, time, seed)
        ctx.eng = eng
        order = getattr(eng, "_param_order", None)          # parameters in the engine's (= the reference's state_dict) order, cached per engine
        if order is None:
            by_name = dict(unet.named_parameters())
            order = eng._param_order = [by_name[n] for n, _ in eng.param_table()]
        ctx.order = order
        ctx.params = params
        ctx.time_shape = time.shape
        return eps

    @staticmethod
    def backward(ctx, deps):
        if torch.is_grad_enabled():
            raise RuntimeError("sr3_b200: double backward (create_graph=True) through the native UNet is not supported")
        grads = {id(p): torch.empty_like(p, memory_format=torch.contiguous_format) for p in ctx.order}
        dx, dnl = ctx.eng.train_unet_backward(deps, [grads[id(p)] for p in ctx.order], want_dx=ctx.needs_input_grad[2],
                                              want_dnl=ctx.needs_input_grad[3], forward=ctx.fwd)
        return (None, None, dx, None if dnl is None else dnl.view(ctx.time_shape), None) + \
            tuple(grads[id(p)] if p.requires_grad else None for p in ctx.params)


class UNet(nn.Module):
    def __init__(self, in_channel=6, out_channel=3, inner_channel=32, norm_groups=32, channel_mults=(1, 2, 4, 8, 8), attn_res=(8),
                 res_blocks=3, dropout=0, with_noise_level_emb=True, image_size=128, precision="bf16"):
        super().__init__()
        self.precision = "bf16"
        self._engines = {}
        self.set_precision(precision)
        if not with_noise_level_emb:
            raise NotImplementedError("sr3_b200 implements the noise-level conditioned UNet only")
        out_channel = out_channel if out_channel is not None else in_channel
        attn_res = (attn_res,) if isinstance(attn_res, int) else tuple(attn_res)
        self.arch = dict(in_channel=in_channel, out_channel=out_channel, inner_channel=inner_channel, norm_groups=norm_groups,
                         channel_mults=tuple(channel_mults), attn_res=attn_res, res_blocks=res_blocks, image_size=image_size)
        self.dropout = dropout
        self._table = parameter_table(in_channel, out_channel, inner_channel, channel_mults, attn_res, res_blocks, image_size)
        for key, shape, _ in self._table:
            node = self
            parts = key.split(".")
            for part in parts[:-1]:
                if part not in node._modules:
                    node.add_module(part, _Node())
                node = node._modules[part]
            node.register_parameter(parts[-1], nn.Parameter(torch.empty(shape)))
        self.reset_parameters()
        self._engines: Dict[tuple, "_native.Engine"] = {}
        self._engine_versions: Dict[tuple, int] = {}
        self._schedule = None
        self._manual_version = 0
        self._differentiable = False

    # torch's default Conv2d / Linear initialisation, drawn in the reference's construction order so that
    # torch.manual_seed(s) yields bit-identical weights in both implementations.
    @torch.no_grad()
    def reset_parameters(self):
        sd = dict(self.named_parameters())
        for key, shape, kind in self._table:
            p = sd[key]
            if kind == "w":
                nn.init.kaiming_uniform_(p, a=math.sqrt(5))
            elif kind == "b":
                w = sd[key[:-4] + "weight"]
                fan_in = w[0].numel()
                bound = 1 / math.sqrt(fan_in) if fan_in > 0 else 0
                nn.init.uniform_(p, -bound, bound)
            elif kind == "one":
                p.fill_(1.0)
            else:
                p.zero_()

    @torch.no_grad()
    def init_orthogonal(self):
        """weights_init_orthogonal of the reference (model/networks.py:45-57) on every Conv / Linear."""
        sd = dict(self.named_parameters())
        for key, _shape, kind in self._table:
            if kind == "w":
                nn.init.orthogonal_(sd[key], gain=1)
            elif kind == "b":
                sd[key].zero_()

    def set_precision(self, precision):
        """"bf16" (default): bf16 tensor-core operands, fp32 accumulation and residual stream -- matches the reference within 1e-2 relative.
        "fp32": every operand is a (hi, lo) bf16 pair, three tensor-core passes per product -- matches the reference's fp32 nn.Conv2d /
        nn.Linear arithmetic (unet.py:87) within 1e-3 relative (measured ~1e-5) at ~1/3 of the speed.  Also: env SR3_PRECISION."""
        if precision not in _native.PRECISIONS:
            raise ValueError("precision must be one of %s, got %r" % (sorted(_native.PRECISIONS), precision))
        self.precision = precision
        return self

    # ---- native engine management
    MAX_ENGINES = 4          # distinct (batch, image size, device, ...) engines kept alive; least recently used ones are released

    def _weights_version(self):
        return sum(p._version for p in self.parameters()) + self._manual_version

    def invalidate(self):
        """Force every engine to re-pack the weights before its next use.  Needed after updates that bypass autograd's version counter
        (`p.data.copy_()`, EMA helpers, reference-style `m.weight.data` initialisers); `load_state_dict` and optimizer steps are seen
        automatically."""
        self._manual_version += 1

    def _load_from_state_dict(self, *args, **kwargs):
        super()._load_from_state_dict(*args, **kwargs)
        self._manual_version += 1

    def set_schedule(self, buffers, sqrt_alphas_cumprod_prev):
        self._schedule = ({k: v.detach().cpu().clone() for k, v in buffers.items()}, sqrt_alphas_cumprod_prev.copy())
        for eng in self._engines.values():
            eng.set_schedule(*self._schedule)

    def engine(self, batch, conditional=True, channels=3, train_dropout=None, height=None, width=None):
        """train_dropout=None: the inference plan; a float: the TRAINING plan (intermediates kept, backward recorded) with that Dropout
        probability -- see GaussianDiffusion.p_losses.  height / width: the image size the plan runs on (default image_size; any size
        _native.check_image_size accepts, for both kinds of plan).  Engines are kept per (batch, size, ...), and every one of them re-packs
        the weights before its next use once they changed."""
        dev = next(self.parameters()).device
        size = self.arch["image_size"]
        h, w = int(size if height is None else height), int(size if width is None else width)
        key = (batch, h, w, str(dev), bool(conditional), channels, self.precision, train_dropout)
        eng = self._engines.pop(key, None)
        if eng is None:
            _native.check_image_size(len(self.arch["channel_mults"]), h, w)      # before an older engine is released
            while len(self._engines) >= self.MAX_ENGINES:            # dicts keep insertion order: the first key is the least recently used
                old = next(iter(self._engines))
                del self._engines[old], self._engine_versions[old]
            if train_dropout is not None and self.precision != "bf16":
                raise NotImplementedError("sr3_b200: the training plan supports precision='bf16' only")
            cfg = dict(self.arch, channels=channels, conditional=conditional, precision=self.precision)
            eng = _native.Engine(cfg, batch, dev, train_dropout=train_dropout, height=h, width=w)
            self._engine_versions[key] = -1
            if self._schedule is not None:
                eng.set_schedule(*self._schedule)
        self._engines[key] = eng                                     # (re-)insert as most recently used
        ver = self._weights_version()
        if self._engine_versions[key] != ver:
            order = getattr(eng, "_param_order", None)
            if order is None:
                by_name = dict(self.named_parameters())
                order = eng._param_order = [by_name[n] for n, _ in eng.param_table()]
            if all(p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and p.device == dev for p in order):
                eng.load_params_fast([p.detach() for p in order])      # one native call, asynchronous (the per-step path of training)
            else:
                eng.load_state_dict(self.state_dict())
            self._engine_versions[key] = ver
        return eng

    def set_differentiable(self, flag=True):
        """Make forward() differentiable with respect to the parameters even when neither x nor time requires grad (losses on the
        parameters alone).  Off by default: see forward()."""
        self._differentiable = bool(flag)
        return self

    def forward(self, x, time):
        """x [B,in_channel,H,W] fp32, time = noise level [B,1] -> eps [B,out_channel,H,W] (unet.py:235-259).  H x W is any size
        _native.check_image_size accepts; attention stays on the levels image_size placed it on.

        With grad mode on and x or time requiring grad (or after set_differentiable(True)) eps carries a grad_fn: the forward runs on the
        bf16 training plan (intermediates kept; Dropout(self.dropout) in train() mode, seeded from torch's RNG) and backward() gives the
        gradients of x, time and every parameter that requires grad.  Otherwise it runs the inference plan and returns a plain tensor."""
        a = self.arch
        cond = a["in_channel"] != a["out_channel"]
        wants_grad = self._differentiable or x.requires_grad or (torch.is_tensor(time) and time.requires_grad)
        if torch.is_grad_enabled() and wants_grad:
            drop = float(self.dropout or 0) if self.training else 0.0
            eng = self.engine(x.shape[0], conditional=cond, channels=a["out_channel"], train_dropout=drop, height=x.shape[2], width=x.shape[3])
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            return _UNetFn.apply(self, eng, x, time, seed, *self.parameters())
        eng = self.engine(x.shape[0], conditional=cond, channels=a["out_channel"], height=x.shape[2], width=x.shape[3])
        return eng.unet_forward(x, time)

"""The differentiable denoiser on the GPU: net.denoise_fn(x, noise_level) with x / noise_level requiring grad (or after
set_differentiable(True)) runs the bf16 training plan, and backward() gives the gradients of x, the noise level and every parameter
(sr3_train_unet_forward / sr3_train_unet_backward).

Against the oracle's fp32 autograd on the CPU (itself pinned to the reference in tests/test_oracle_unet_grad.py): eps within 1e-2, dx
within 2e-2 relative L2 over the batch, d noise_level per image within the bound of dtau conditioned by Cauchy-Schwarz (compare), every
parameter gradient within tests/test_gpu_train.py's bounds.  Also: equivalence with p_losses' backward, the three new kernels against
fp64, the guards against stale or repeated backwards, and the unchanged default."""
import numpy as np
import pytest
import torch

import _train_util as tu
import _unet_grad_inputs as ui
from oracle import sr3_oracle as orc
from test_oracle_unet_grad import golden, oracle_grads, unpack_masks  # noqa: F401  (golden: module fixture)

pytestmark = pytest.mark.gpu
EPS_TOL = 1e-2
INPUT_TOL = 2e-2         # dx
# relative L2 per parameter tensor.  tests/test_gpu_train.py holds loss gradients to 2e-2 (3e-2 for five-level nets); here the upstream
# gradient is an arbitrary fp32 tensor that the load rounds to bf16 (an L1 / L2 loss gradient loses little or nothing there), and the
# backward is not run-to-run reproducible (fp32 atomics, DESIGN.md §3.6): the unconditional case measured 1.84e-2 and 2.00e-2 in two runs.
GRAD_TOL = 2.5e-2
FIVE_LEVEL_TOL = 3e-2


def build(name, dropout=0.0, loss_type="l1"):
    unet, image_size, conditional, b, h, w = ui.ALL[name]
    unet = dict(unet, dropout=dropout)
    return tu.build_train_net(unet, image_size, ui.SEED, loss_type, tu.SCHED, conditional), unet


def ours(net, x, nl, G, train_mode=False):
    """eps and the gradients of sum(G * eps) through net.denoise_fn, as a user writes it."""
    dn = net.denoise_fn
    dn.train(train_mode)
    for p in dn.parameters():
        p.grad = None
    xc = x.cuda().requires_grad_(True)
    nc = nl.cuda().requires_grad_(True)
    eps = dn(xc, nc)
    assert eps.grad_fn is not None
    (G.cuda() * eps).sum().backward()
    return eps.detach().cpu(), xc.grad.cpu(), nc.grad.cpu(), {k: p.grad.cpu() for k, p in dn.named_parameters()}


def oracle_of(net, unet, name, x, nl, G, masks=None, p=0.0):
    """oracle_grads, and dtau [B, inner]: the gradient reaching the output of the oracle's noise-level MLP (row b is what an oracle run on
    image b alone gives as grad(noise_level_mlp.3.bias): the UNet is separable per image)."""
    _, image_size, _, _, _, _ = ui.ALL[name]
    sd = {k: v.detach().cpu() for k, v in net.denoise_fn.state_dict().items()}
    torch.set_num_threads(min(16, torch.get_num_threads()))
    taus, mlp = [], orc.noise_level_mlp

    def kept(*args):
        t = mlp(*args)
        t.retain_grad()
        taus.append(t)
        return t
    orc.noise_level_mlp = kept
    try:
        r = oracle_grads(sd, tu.oracle_cfg(unet, image_size), x, nl, G, masks, p)
    finally:
        orc.noise_level_mlp = mlp
    assert len(taus) == 1
    return r + (taus[0].grad.reshape(x.shape[0], -1),)


def dnl_bounds(sd, nl, rdtau):
    """c_b = d tau_b / d noise_level_b [B, inner] in fp64 by forward-mode autograd through the oracle's noise-level MLP, and the per-image
    scale ||c_b|| ||rdtau_b|| of the conditioned d noise_level bound."""
    sd64 = {k: v.double() for k, v in sd.items() if k.startswith("noise_level_mlp.")}
    inner = rdtau.shape[1]
    n = nl.double().view(-1, 1)
    _, c = torch.func.jvp(lambda t: orc.noise_level_mlp(sd64, t, inner).reshape(n.shape[0], inner), (n,), (torch.ones_like(n),))
    return c, c.norm(dim=1) * rdtau.double().norm(dim=1)


def compare(name, net, nl, o, r, label=None):
    """eps and dx within EPS_TOL / INPUT_TOL relative L2, every parameter gradient within GRAD_TOL (FIVE_LEVEL_TOL), and d noise_level per
    image within tol ||c_b|| ||dtau_b^ref||: by Cauchy-Schwarz on d noise_level_b = c_b^T dtau_b with dtau_b held to tol
    (tests/test_gpu_noise_level_grad.py, test_noise_level_chain_matches_oracle).  A relative L2 bound over the batch's 2 or 3 scalars
    is ill-conditioned: it is larger than the error of dtau by ||c_b|| ||dtau_b|| / |c_b^T dtau_b|, which grows without bound as c_b
    and dtau_b turn orthogonal."""
    eps, dx, dnl, grads = o
    reps, rdx, rdnl, rgrads, rdtau = r
    five = len(ui.ALL[name][0]["channel_multiplier"]) == 5
    tol = FIVE_LEVEL_TOL if five else GRAD_TOL
    _, scale = dnl_bounds({k: v.detach().cpu() for k, v in net.denoise_fn.state_dict().items()}, nl, rdtau)
    dnl_ratio = (dnl.double() - rdnl.double()).abs().view(-1) / scale
    errs = {"eps": tu.rel(eps, reps), "dx": tu.rel(dx, rdx), "dnl": tu.rel(dnl, rdnl)}
    rows = tu.compare(grads, rgrads)
    worst = sorted(rows, key=lambda row: -row[1])[:3]
    print(label or name, {k: f"{v:.2e}" for k, v in errs.items()}, "d noise_level error / (|c| |dtau|):", [f"{v:.2e}" for v in dnl_ratio.tolist()],
          "worst grads:", [(n, f"{e:.2e}") for n, e, _, _ in worst])
    assert dnl.shape == rdnl.shape
    assert errs["eps"] <= EPS_TOL and errs["dx"] <= INPUT_TOL, errs
    assert (dnl_ratio <= tol).all(), (dnl_ratio, tol)
    bad = [(n, e, c) for n, e, c, _ in rows if e >= tol]
    assert not bad, bad[:10]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", sorted(ui.ALL))
def test_unet_gradients_match_oracle_with_conditioned_dnl(name):
    """The tiny net at 32x32 (256-token attention) and 32x64 (512), the 4x4-level net at batch 3, an unconditional net, the 16->64 net at
    64x64: eps, dx, d noise_level (per image, conditioned: compare) and every parameter gradient against the oracle's fp32 autograd."""
    net, unet = build(name)
    x, nl, G = ui.inputs(name)
    o = ours(net, x, nl, G)
    b, h, w = ui.ALL[name][3:]
    assert o[1].shape == x.shape and o[2].shape == (b, 1)
    compare(name, net, nl, o, oracle_of(net, unet, name, x, nl, G))


def test_unet_gradients_with_reference_dropout_masks_conditioned_dnl(golden):  # noqa: F811
    """train() mode with the reference's own nn.Dropout masks injected: against the oracle on the same masks, and eps against the golden."""
    d = golden["dropout"]
    name = d["case"]
    unet, _, conditional, b, h, w = ui.CASES[name]
    net, unet = build(name, dropout=d["p"])
    eng = net.denoise_fn.engine(b, conditional=conditional, channels=3, train_dropout=float(d["p"]), height=h, width=w)
    masks = unpack_masks(d)
    assert sorted(eng.dropout_layers()) == sorted(masks)
    for k, keep in masks.items():
        eng.set_dropout_mask(k, keep.cuda().contiguous())
    x, nl, G = ui.inputs(name)
    o = ours(net, x, nl, G, train_mode=True)
    assert tu.rel(o[0], d["eps"]) <= EPS_TOL
    compare(name, net, nl, o, oracle_of(net, unet, name, x, nl, G, masks, d["p"]), label=name + "/dropout")


def test_train_mode_dropout_follows_torch_seed():
    """Dropout(self.dropout) in train() mode, its seed drawn from torch's RNG: torch.manual_seed reproduces eps; eval() mode has no Dropout."""
    net, _ = build("tiny_32x32", dropout=0.2)
    x, nl, _ = ui.inputs("tiny_32x32")
    dn = net.denoise_fn
    dn.train(True)
    outs = []
    for s in (5, 5, 6):
        torch.manual_seed(s)
        outs.append(dn(x.cuda().requires_grad_(True), nl.cuda()).detach())
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
    dn.train(False)
    ev = dn(x.cuda().requires_grad_(True), nl.cuda()).detach()
    assert torch.equal(ev, dn(x.cuda().requires_grad_(True), nl.cuda()).detach()) and not torch.equal(ev, outs[0])


def test_parameter_gradients_match_p_losses():
    """p_losses(...).backward() against (denoise_fn(cat(SR, q_sample(HR)), gamma) - noise).abs().sum().backward() with set_differentiable(True),
    at the same HR, SR, gamma, noise and dropout seed: both run the same forward and the same recorded backward from the same +-1 operand (its
    bf16 values and integer channel sums are exact either way), and the loss agrees.  They are not bit-identical because the backward is not
    bit-reproducible even on one path: the fp32 atomics of its per-(image, channel) sums (gn_bwd_kernel, grad_combine_kernel) and of
    film_bwd_kernel's dtau add in run-dependent order, and the bf16 roundings of later gradient operands amplify that.  Measured on an H100:
    2 of 124 tensors bit-identical, worst 3.8e-3 / 5.2e-3 relative in two sessions, while two p_losses backwards differ by 5.0e-3; the bound is
    tests/test_gpu_train.py's run-to-run bound."""
    net, _ = build("tiny_32x32", dropout=0.2, loss_type="l1")
    net.train(True)
    b, h, w = 2, 32, 32
    hr, sr, noise = tu.batch(b, h, 4321)
    hr, sr, noise = hr.cuda(), sr.cuda(), noise.cuda()
    gamma = tu.draw_gamma(b, 7).cuda()
    dn = net.denoise_fn

    def grads():
        return {k: p.grad.detach().clone() for k, p in dn.named_parameters()}

    torch.manual_seed(99)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())      # what the denoise_fn path draws after torch.manual_seed(99)
    runs = []
    for _ in range(2):
        for p in dn.parameters():
            p.grad = None
        l = net.p_losses({"HR": hr, "SR": sr}, noise=noise, gamma=gamma, dropout_seed=seed)
        l.backward()
        runs.append((l.item(), grads()))
    dn.set_differentiable(True)
    try:
        for p in dn.parameters():
            p.grad = None
        x_noisy = net.q_sample(hr, gamma.view(-1, 1, 1, 1), noise)
        torch.manual_seed(99)
        eps = dn(torch.cat([sr, x_noisy], dim=1), gamma.view(b, 1))
        lo = (eps - noise).abs().sum()
        lo.backward()
        g_ours = grads()
    finally:
        dn.set_differentiable(False)
    assert abs(lo.item() - runs[0][0]) <= 1e-5 * abs(runs[0][0]), (lo.item(), runs[0][0])
    run_to_run = max(tu.rel(runs[0][1][k], runs[1][1][k]) for k in g_ours)
    diffs = {k: tu.rel(g_ours[k], runs[0][1][k]) for k in g_ours}
    identical = sum(torch.equal(g_ours[k], runs[0][1][k]) for k in g_ours)
    worst = sorted(diffs.items(), key=lambda kv: -kv[1])[:5]
    print(f"p_losses equivalence: {identical}/{len(diffs)} tensors bit-identical; worst {worst}; p_losses run-to-run {run_to_run:.2e}")
    assert max(diffs.values()) < 2e-2, worst


# ------------------------------------------------------------------------------------------------ the new kernels against fp64
@pytest.mark.parametrize("B,H,W", [(2, 32, 32), (3, 4, 4), (2, 16, 64)])
def test_grad_load_matches_fp64(B, H, W):
    """grad_load_kernel: bf16(g) exact to rounding in channels 0..2 of the 64-channel operand, the rest untouched; fp32 channel sums of the
    unrounded g."""
    from sr3_b200 import _native
    g = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(B * H + W)) * 3
    deps, bias = _native.test_grad_load(g.cuda())
    deps = deps.cpu()
    assert torch.equal(deps[..., :3], g.permute(0, 2, 3, 1).bfloat16())
    assert not deps[..., 3:].any()
    ref = g.double().sum(dim=(0, 2, 3))
    assert ((bias.cpu().double() - ref).abs() <= 1e-5 * g.double().abs().sum(dim=(0, 2, 3))).all(), (bias, ref)


@pytest.mark.parametrize("inner,B", [(64, 2), (64, 7), (128, 3)])
def test_noise_level_gradient_matches_fp64(inner, B):
    """noise_level_bwd_kernel against fp64 autograd through the positional encoding and the noise-level MLP, for a given dtau."""
    from sr3_b200 import _native
    from oracle import sr3_oracle as orc
    gen = torch.Generator().manual_seed(inner + B)
    w1 = torch.randn(4 * inner, inner, generator=gen) / inner ** 0.5
    b1 = torch.randn(4 * inner, generator=gen) * 0.1
    w2 = torch.randn(inner, 4 * inner, generator=gen) / (4 * inner) ** 0.5
    b2 = torch.zeros(inner)
    dtau = torch.randn(B, inner, generator=gen)
    nl = torch.rand(B, generator=gen)
    got = _native.test_noise_level_bwd(*[t.cuda() for t in (nl, w1, b1, w2, dtau)]).cpu()
    sd = {"noise_level_mlp.1.weight": w1.double(), "noise_level_mlp.1.bias": b1.double(), "noise_level_mlp.3.weight": w2.double(),
          "noise_level_mlp.3.bias": b2.double()}
    nld = nl.double().view(B, 1).requires_grad_(True)
    (orc.noise_level_mlp(sd, nld, inner).view(B, inner) * dtau.double()).sum().backward()
    ref = nld.grad.view(B)
    assert ((got.double() - ref).norm() / ref.norm()).item() < 1e-4, (got, ref)


@pytest.mark.parametrize("B,H,W,inner,cin", [(2, 32, 32, 64, 6), (2, 16, 64, 64, 3), (8, 8, 8, 128, 6)])
def test_input_gradient_matches_conv_transpose(B, H, W, inner, cin):
    """The data gradient of the first conv on the tile kernel (output channels padded to 64) and its NCHW store: against fp64
    conv_transpose2d of the same bf16 operands."""
    from sr3_b200 import _native
    gen = torch.Generator().manual_seed(B + H + inner + cin)
    dy = torch.randn(B, H, W, inner, generator=gen).bfloat16()
    w = torch.randn(inner, cin, 3, 3, generator=gen) * 0.1
    got = _native.test_input_grad(dy.cuda(), w.cuda()).cpu()
    ref = torch.nn.functional.conv_transpose2d(dy.double().permute(0, 3, 1, 2), w.bfloat16().double(), padding=1)
    assert got.shape == ref.shape
    err = ((got.double() - ref).norm() / ref.norm()).item()
    assert err < 2e-5, err


# ------------------------------------------------------------------------------------------------ guards and the unchanged default
def test_backward_after_a_later_forward_raises():
    net, _ = build("tiny_32x32")
    dn = net.denoise_fn
    x, nl, G = ui.inputs("tiny_32x32")
    e1 = dn(x.cuda().requires_grad_(True), nl.cuda())
    x2 = (x * 0.5).cuda().requires_grad_(True)
    e2 = dn(x2, nl.cuda())
    with pytest.raises(RuntimeError, match="later forward"):
        e1.sum().backward()
    (G.cuda() * e2).sum().backward()                      # the later forward's own backward works
    assert x2.grad is not None and torch.isfinite(x2.grad).all()
    # a p_losses forward on the same engine overwrites it as well
    e3 = dn(x.cuda().requires_grad_(True), nl.cuda())
    hr, sr, noise = tu.batch(2, 32, 1)
    net.p_losses({"HR": hr.cuda(), "SR": sr.cuda()}, noise=noise.cuda(), gamma=tu.draw_gamma(2, 7))
    with pytest.raises(RuntimeError, match="p_losses"):
        e3.sum().backward()


def test_second_backward_and_double_backward_raise():
    net, _ = build("tiny_32x32")
    dn = net.denoise_fn
    x, nl, _ = ui.inputs("tiny_32x32")
    e = dn(x.cuda().requires_grad_(True), nl.cuda())
    e.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already been backpropagated"):
        e.sum().backward()
    xc = x.cuda().requires_grad_(True)
    e = dn(xc, nl.cuda())
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(e.sum(), xc, create_graph=True)


def test_precise_mode_and_unsupported_sizes_are_refused():
    from sr3_b200 import _native
    net, _ = build("tiny_32x32")
    dn = net.denoise_fn
    x, nl, _ = ui.inputs("tiny_32x32")
    dn.set_precision("fp32")
    try:
        with pytest.raises(NotImplementedError, match="precision='bf16' only"):
            dn(x.cuda().requires_grad_(True), nl.cuda())
    finally:
        dn.set_precision("bf16")
    keys = set(dn._engines)
    xb, nb = torch.randn(2, 6, 48, 48, device="cuda", requires_grad=True), nl.cuda()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(_native.UnsupportedSizeError):
        dn(xb, nb)
    assert set(dn._engines) == keys and torch.cuda.mem_get_info()[0] == free0


def test_default_forward_is_unchanged():
    """Grad mode on, parameters requiring grad, x and time not requiring grad, flag off: the inference plan, no grad_fn, no training engine,
    the inference engine's bits."""
    net, _ = build("tiny_32x32")
    dn = net.denoise_fn
    x, nl, _ = ui.inputs("tiny_32x32")
    assert all(p.requires_grad for p in dn.parameters()) and torch.is_grad_enabled()
    eps = dn(x.cuda(), nl.cuda())
    assert eps.grad_fn is None and not eps.requires_grad
    assert all(k[-1] is None for k in dn._engines), list(dn._engines)
    ref = dn.engine(2, conditional=True, channels=3).unet_forward(x.cuda(), nl.cuda())
    assert torch.equal(eps, ref)


def test_parameter_only_loss_and_weight_updates():
    """set_differentiable(True): a loss on the parameters alone (x and time without grad); an optimizer step on those gradients reaches the
    next forward, which matches the oracle on the updated weights."""
    net, unet = build("tiny_32x32")
    dn = net.denoise_fn.set_differentiable(True)
    x, nl, G = ui.inputs("tiny_32x32")
    opt = torch.optim.SGD(dn.parameters(), lr=1e-3)
    opt.zero_grad()
    eps0 = dn(x.cuda(), nl.cuda())
    assert eps0.grad_fn is not None
    (G.cuda() * eps0).sum().backward()
    assert all(p.grad is not None for p in dn.parameters())
    opt.step()
    eps1 = dn(x.cuda(), nl.cuda()).detach().cpu()
    assert tu.rel(eps1, eps0.detach().cpu()) > 1e-3
    sd = {k: v.detach().cpu() for k, v in dn.state_dict().items()}
    ref = oracle_grads(sd, tu.oracle_cfg(unet, 32), x, nl, G)[0]
    assert tu.rel(eps1, ref) <= EPS_TOL
    dn.set_differentiable(False)
    assert dn(x.cuda(), nl.cuda()).grad_fn is None
    assert np.isfinite(eps1.numpy()).all()

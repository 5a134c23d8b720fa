"""The noise-level gradient chain of the differentiable denoiser: FiLM projections -> d tau -> noise-level MLP -> d noise_level.

film_bwd_kernel forms dtau_b = sum_l W_f,l^T dfilm_l,b over every ResnetBlock's FiLM slice l, embed_bwd_kernel the MLP's parameter
gradients from it, noise_level_bwd_kernel d noise_level_b = c_b^T dtau_b with c_b = d tau_b / d noise_level_b (train_plan.inc,
bwd_film_and_embed and train_unet_backward).  Three levels of checks:

(a) identities between the engine's own outputs of ONE backward, in fp64 (the engine's dfilm, dtau and tau come from
    sr3_test_train_film_state).  They separate the plan's wiring from bf16 noise: the run-to-run spread of the backward (DESIGN.md §3.6)
    changes dfilm, but not whether the rest of the chain is the function of it that it should be.
(b) the chain against the oracle with a bound that holds: dtau_b per image, and d noise_level conditioned by Cauchy-Schwarz.
(c) the three kernels through their test hooks at the edges the suite's other hook tests skip.

Bounds of (a) and (c) are first-order running-error bounds of the kernels' fp32 arithmetic, u = 2^-24 (see mlp64 / mlp_backward64 and
test_film_identities_on_one_backward), times 2 for the neglected higher-order terms."""
import math

import pytest
import torch

import _train_util as tu
import _unet_grad_inputs as ui
from oracle import sr3_oracle as orc
from test_gpu_backward import check, film_reference, gen
from test_gpu_unet_grad import FIVE_LEVEL_TOL, GRAD_TOL, build, dnl_bounds, oracle_of

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
SAFETY = 2.0
EDGE_NL = (0.0, 1e-4, 1.0)
# the five-level 16->128 net (config/sr_sr3_16_128.json) at its own 128x128: 27 ResnetBlocks, F = 8384 FiLM channels
CASES = dict(ui.ALL, sr16_128_128x128=(ui.SR16_64, 128, True, 1, 128, 128))


def case_inputs(name):
    if name in ui.ALL:
        return ui.inputs(name)
    unet, _, _, b, h, w = CASES[name]
    g = torch.Generator().manual_seed(3000)
    return torch.randn(b, unet["in_channel"], h, w, generator=g), torch.tensor([[0.7]]), torch.randn(b, unet["out_channel"], h, w, generator=g)


def film_layers(unet, image_size):
    """[(ResnetBlock prefix, offset in dfilm, channels)] in plan order: downs, mid, ups."""
    downs, mid, ups = orc.unet_topology(tu.oracle_cfg(unet, image_size))
    out, off = [], 0
    for s in downs + mid + ups:
        if s.kind == "res":
            out.append((s.name + ".res_block", off, s.cout))
            off += s.cout
    return out


def run(net, x, nl, G):
    """One forward + backward of sum(G * denoise_fn(x, nl)) with x and nl requiring grad.  Returns (d noise_level [B], parameter gradients,
    fp32 weights, the engine's FiLM state), all on the CPU."""
    dn = net.denoise_fn
    dn.train(False)
    for p in dn.parameters():
        p.grad = None
    b, _, h, w = x.shape
    xc, nc = x.cuda().requires_grad_(True), nl.cuda().requires_grad_(True)
    (G.cuda() * dn(xc, nc)).sum().backward()
    a = dn.arch
    eng = dn.engine(b, conditional=a["in_channel"] != a["out_channel"], channels=a["out_channel"], train_dropout=0.0, height=h, width=w)
    state = {k: v.cpu() for k, v in eng.film_state().items()}
    return (nc.grad.cpu().view(-1), {k: p.grad.cpu() for k, p in dn.named_parameters()}, {k: v.detach().cpu() for k, v in dn.state_dict().items()},
            state)


def fp32_sum(rows):
    """sum over the leading dimension in fp32, in index order from 0.f: the kernels' `a += x[b]` loops bit for bit."""
    acc = torch.zeros_like(rows[0])
    for r in rows:
        acc = acc + r
    return acc


def within(got, ref, bound, what):
    """|got - ref| <= bound element by element; returns the largest |got - ref| / bound."""
    got, ref, bound = got.double(), ref.double(), SAFETY * bound.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    bad = (err > bound).nonzero()
    if bad.numel():
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} of {err.numel()} elements past the bound, first at {i}: got {got[i].item():.9g}, want "
                    f"{ref[i].item():.9g} (bound {bound[i].item():.3g})")
    return (err / bound.clamp_min(1e-300)).max().item()


def mlp64(sd, nl):
    """tau = W2 swish(W1 PE(nl) + b1) + b2 in fp64 at the fp32 noise levels nl [B], with first-order bounds on what the kernels' fp32
    forms of each intermediate can differ by.  PE: e = nl f_i with f_i = expf(-ln(1e4) i / (inner/2)) (the rounded step, the fp32
    constant, expf and the product: <= 17 u |e|; 23 u taken), sinf / cosf within 2 ulp.  A dot product of n fp32 terms in any order:
    <= n u of the sum of the terms' magnitudes.  swish and swish' (expf, one division, products): 4 and 6 ulp, and |swish'| <= 1.1,
    |swish''| <= 0.5 carry the error of their argument."""
    W1, b1, W2, b2 = (sd["noise_level_mlp." + k].double() for k in ("1.weight", "1.bias", "3.weight", "3.bias"))
    inner = W2.shape[0]
    count = inner // 2
    f = torch.exp(-math.log(1e4) * torch.arange(count, dtype=torch.float64) / count).repeat(2)
    e = nl.double().view(-1, 1) * f
    pe = torch.cat([e[:, :count].sin(), e[:, count:].cos()], 1)
    dpe = torch.cat([f[:count] * e[:, :count].cos(), -f[count:] * e[:, count:].sin()], 1)       # d PE / d noise level
    m = {"W1": W1, "W2": W2, "pe": pe, "dpe": dpe, "pe_err": (23 * e.abs() + 2) * U, "dpe_err": (23 * e.abs() + 25) * U * f}
    m["pre"] = pe @ W1.T + b1
    m["pre_err"] = (inner + 1) * U * (pe.abs() @ W1.abs().T + b1.abs()) + m["pe_err"] @ W1.abs().T
    m["sg"] = torch.sigmoid(m["pre"])
    m["h"] = m["pre"] * m["sg"]
    m["h_err"] = 1.1 * m["pre_err"] + 4 * U * m["h"].abs()
    m["tau"] = m["h"] @ W2.T + b2
    m["tau_err"] = (4 * inner + 1) * U * (m["h"].abs() @ W2.abs().T + b2.abs()) + m["h_err"] @ W2.abs().T
    return m


def mlp_backward64(m, dtau):
    """The MLP's backward in fp64 from a given dtau [B, inner] (exact input: the engine's own), with first-order bounds on embed_bwd_kernel's
    and noise_level_bwd_kernel's fp32 forms: dh = W2^T dtau (inner terms), dpre = dh swish'(pre), dW2 = sum_b dtau_b h_b^T and
    dW1 = sum_b dpre_b pe_b^T (B terms each), db1 = sum_b dpre_b, dPE = W1^T dpre (4 inner terms), dnl = dPE . dPE/dnl (inner / 32 terms
    per lane, then 5 shuffle levels).  Returns {name: (value, bound)}."""
    dt = dtau.double()
    B, inner = dt.shape
    hid = 4 * inner
    W1, W2, pre, sg, h = m["W1"], m["W2"], m["pre"], m["sg"], m["h"]
    dh = dt @ W2
    dh_err = inner * U * (dt.abs() @ W2.abs())
    sp = sg * (1 + pre * (1 - sg))
    sp_err = 0.5 * m["pre_err"] + 6 * U * sg * (1 + pre.abs() * (1 - sg))
    dpre = dh * sp
    dpre_err = dh_err * sp.abs() + dh.abs() * sp_err + U * dpre.abs()
    dPE = dpre @ W1
    dPE_err = dpre_err @ W1.abs() + hid * U * (dpre.abs() @ W1.abs())
    dpe = m["dpe"]
    return {"noise_level_mlp.3.weight": (dt.T @ h, dt.abs().T @ (m["h_err"] + (B + 1) * U * h.abs())),
            "noise_level_mlp.1.weight": (dpre.T @ m["pe"], dpre_err.T @ m["pe"].abs() + dpre.abs().T @ (m["pe_err"] + (B + 1) * U * m["pe"].abs())),
            "noise_level_mlp.1.bias": (dpre.sum(0), dpre_err.sum(0) + B * U * dpre.abs().sum(0)),
            "dnl": ((dPE * dpe).sum(1), (dPE_err * dpe.abs()).sum(1) + (dPE.abs() * m["dpe_err"]).sum(1) +
                    (inner // 32 + 8) * U * (dPE.abs() * dpe.abs()).sum(1))}


def check_identities(layers, nl, dnl, grads, sd, st, what):
    """Every identity of the chain on one backward's outputs at the noise levels nl [B]; returns {identity: largest error / bound}."""
    B, rows = nl.numel(), st["dfilm"].shape[0]
    dfilm, dtau, tau = st["dfilm"][:B], st["dtau"][:B], st["tau"][:B]
    F = dfilm.shape[1]
    assert F == sum(c for _, _, c in layers), (what, F)
    # padded image slots (the batch rounded up for the tile kernels): nothing is summed into them
    assert not st["dfilm"][B:].any() and not st["dtau"][B:].any(), f"{what}: padded rows {B}..{rows} of dfilm / dtau are not zero"
    ratio = {}
    # film_bwd_kernel's bias sums and the film_slices copies: bit for bit
    for p, off, c in layers:
        s = fp32_sum(dfilm[:, off:off + c])
        assert torch.equal(grads[p + ".noise_func.noise_func.0.bias"], s), f"{what}: {p} FiLM bias gradient is not the sum of its dfilm slice"
        assert torch.equal(grads[p + ".block1.block.3.bias"], s), f"{what}: {p} block1 conv bias gradient is not the sum of its dfilm slice"
    assert torch.equal(grads["noise_level_mlp.3.bias"], fp32_sum(dtau)), f"{what}: noise_level_mlp.3.bias gradient is not the sum of dtau"
    # dtau_b = sum_l W_f,l^T dfilm_l,b over every slice: per block of 64 FiLM channels a shared-memory sum of 64 rounded products, then one
    # global atomic per block: <= (64 + ceil(F / 64) + 1) u of sum_j |W_f[j][i] dfilm_b[j]|
    Wf = torch.cat([sd[p + ".noise_func.noise_func.0.weight"] for p, _, _ in layers]).double()
    nblk = -(-F // 64)
    ratio["dtau"] = within(dtau, dfilm.double() @ Wf, (64 + nblk + 1) * U * (dfilm.double().abs() @ Wf.abs()), what + " dtau = W_f^T dfilm")
    # tau (embed_kernel) against fp64 from the weights and the noise level; grad(W_f) = sum_b dfilm_b tau_b^T (B fp32 products and sums)
    m = mlp64(sd, nl)
    ratio["tau"] = within(tau, m["tau"], m["tau_err"], what + " tau")
    dwf_bound = dfilm.double().abs().T @ (m["tau_err"] + (B + 1) * U * m["tau"].abs())
    for p, off, c in layers:
        ratio["dW_f"] = max(ratio.get("dW_f", 0.0), within(grads[p + ".noise_func.noise_func.0.weight"], dfilm.double()[:, off:off + c].T @ m["tau"],
                                                           dwf_bound[off:off + c], f"{what} {p} grad(W_f)"))
    # the MLP's parameter gradients and d noise_level from the engine's own dtau
    ref = mlp_backward64(m, dtau)
    for k, (v, bnd) in ref.items():
        ratio[k] = within(dnl if k == "dnl" else grads[k], v, bnd, f"{what} {k}")
    return ratio


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_film_identities_on_one_backward(name):
    """(a) On one backward, in fp64 on the engine's own outputs: the FiLM and block1 conv bias gradients are the fp32 sums of the engine's
    dfilm slices bit for bit; dtau = sum over every FiLM slice of W_f,l^T dfilm_l (every slice, at its offset, once); the engine's tau =
    the MLP in fp64; grad(W_f) = sum_b dfilm_b tau_b^T; the MLP's parameter gradients and d noise_level = the fp64 backward from the
    engine's dtau; padded image slots stay zero.  One image at a time (every per-image quantity is then a parameter gradient) at the
    case's noise levels and at 0, 1e-4 and 1, then the case's whole batch at its noise levels and at the edge levels."""
    unet, image_size, _, b, _, _ = CASES[name]
    net, _ = build(name) if name in ui.ALL else (tu.build_train_net(unet, image_size, ui.SEED, "l1", tu.SCHED, True), unet)
    layers = film_layers(unet, image_size)
    x, nl, G = case_inputs(name)
    runs = [(x[:1], torch.tensor([[v]]), G[:1]) for v in [float(t) for t in nl.view(-1)] + list(EDGE_NL)]
    if b > 1:
        runs += [(x, nl, G), (x, torch.tensor([[v] for v in (1.0, 0.0, 1e-4)][:b]), G)]
    worst = {}
    for xr, nr, gr in runs:
        dnl, grads, sd, st = run(net, xr, nr, gr)
        what = f"{name} B={xr.shape[0]} nl={[float(v) for v in nr.view(-1)]}"
        for k, v in check_identities(layers, nr.view(-1), dnl, grads, sd, st, what).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(name, f"{len(layers)} FiLM layers, {len(runs)} backwards; largest error / bound:", {k: f"{v:.2e}" for k, v in worst.items()})


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", sorted(ui.ALL))
def test_noise_level_chain_matches_oracle(name):
    """(b) dtau_b against the oracle's (the gradient reaching the output of its noise-level MLP: the UNet is separable per image, so row b
    is what an oracle run on image b alone gives as grad(noise_level_mlp.3.bias)), per image within the file-wide per-tensor bound of a
    parameter gradient (tests/test_gpu_unet_grad.py GRAD_TOL, FIVE_LEVEL_TOL for five-level nets).  Then d noise_level per image within
    tol ||c_b|| ||dtau_b^ref||, c_b = d tau_b / d noise_level_b in fp64 by autograd through oracle.sr3_oracle.noise_level_mlp: by (a) the
    engine's d noise_level_b is c_b^T dtau_b (to ~1e-6), the oracle's is c_b^T dtau_b^ref, so by Cauchy-Schwarz the two differ by at most
    ||c_b|| ||dtau_b - dtau_b^ref|| <= tol ||c_b|| ||dtau_b^ref||.  A relative bound on d noise_level itself would be larger than tol by
    ||c_b|| ||dtau_b|| / |c_b^T dtau_b|, which is unbounded when c_b and dtau_b are far from parallel."""
    net, unet = build(name)
    x, nl, G = ui.inputs(name)
    dnl, _, _, st = run(net, x, nl, G)
    r = oracle_of(net, unet, name, x, nl, G)
    rdnl, rdtau = r[2].view(-1), r[4]
    b = x.shape[0]
    tol = FIVE_LEVEL_TOL if len(unet["channel_multiplier"]) == 5 else GRAD_TOL
    errs = [tu.rel(st["dtau"][i], rdtau[i]) for i in range(b)]
    sd = {k: v.detach().cpu() for k, v in net.denoise_fn.state_dict().items()}
    c, scale = dnl_bounds(sd, nl, rdtau)
    ratio = (dnl.double() - rdnl.double()).abs() / scale
    cond = (scale / (c * rdtau.double()).sum(1).abs()).tolist()
    print(name, "dtau per image:", [f"{e:.2e}" for e in errs], "|d noise_level error| / (|c| |dtau|):", [f"{v:.2e}" for v in ratio.tolist()],
          "conditioning |c| |dtau| / |c.dtau|:", [f"{v:.1f}" for v in cond])
    assert max(errs) <= tol, errs
    assert (ratio <= tol).all(), ratio


# ------------------------------------------------------------------------------------------------ (c) the kernels at their edges
# 200 KB of shared memory hold embed_bwd_smem = 40 B inner bytes: 80 images at inner 64, 40 at 128, 20 at 256 (the next width after the
# shipped 64 and 128 that an engine accepts: a multiple of 64)
EDGE_SHAPES = [(64, 1), (64, 80), (128, 1), (128, 40), (256, 1), (256, 3), (256, 20)]


def mlp_operands(inner, B, nl_kind, scale, key):
    """Random MLP weights (b2 = 0), noise levels of the kind asked for and a dtau scaled by `scale`."""
    g = gen(inner, B, nl_kind, scale, key)
    sd = {"noise_level_mlp.1.weight": torch.randn(4 * inner, inner, generator=g) / inner ** 0.5,
          "noise_level_mlp.1.bias": torch.randn(4 * inner, generator=g) * 0.1,
          "noise_level_mlp.3.weight": torch.randn(inner, 4 * inner, generator=g) / (4 * inner) ** 0.5,
          "noise_level_mlp.3.bias": torch.zeros(inner)}
    nl = {"zero": torch.zeros(B), "one": torch.ones(B), "rand": torch.rand(B, generator=g)}[nl_kind]
    dtau = torch.randn(B, inner, generator=g) * scale
    return sd, nl, dtau, g


@pytest.mark.parametrize("scale", [1.0, 1e3, 1e-3])
@pytest.mark.parametrize("nl_kind", ["rand", "zero", "one"])
@pytest.mark.parametrize("inner,B", EDGE_SHAPES)
def test_noise_level_bwd_at_the_edges(inner, B, nl_kind, scale):
    """noise_level_bwd_kernel against the fp64 backward, each image within its running-error bound (mlp_backward64): a single scalar per
    image, so no relative bound over a few of them."""
    from sr3_b200 import _native
    sd, nl, dtau, _ = mlp_operands(inner, B, nl_kind, scale, "dnl")
    w = [sd["noise_level_mlp." + k] for k in ("1.weight", "1.bias", "3.weight")]
    got = _native.test_noise_level_bwd(nl.cuda(), *[t.cuda() for t in w], dtau.cuda()).cpu()
    ref, bound = mlp_backward64(mlp64(sd, nl), dtau)["dnl"]
    within(got, ref, bound, f"dnl inner={inner} B={B} nl={nl_kind} scale={scale}")


@pytest.mark.parametrize("scale", [1.0, 1e3, 1e-3])
@pytest.mark.parametrize("nl_kind", ["rand", "zero", "one"])
@pytest.mark.parametrize("inner,B", EDGE_SHAPES)
def test_film_and_embed_bwd_at_the_edges(inner, B, nl_kind, scale):
    """film_bwd_kernel then embed_bwd_kernel against fp64 autograd (tests/test_gpu_backward.py film_reference), within that file's bounds
    (2e-5 relative L2, 1e-4 (|ref| + rms) per element: fp32 sums of at most 4 inner = 1024 terms, ~2^-24 sqrt(n) each), at the largest
    batch the shared memory admits, one image, inner 256, noise levels 0 and 1, and dfilm (so dtau) scaled by 1e3 and 1e-3."""
    from sr3_b200 import _native
    sd, nl, _, g = mlp_operands(inner, B, nl_kind, scale, "film")
    F_ = 1000
    wf = torch.randn(F_, inner, generator=g) / inner ** 0.5
    tau = torch.randn(B, inner, generator=g)
    dfilm = torch.randn(B, F_, generator=g) * scale
    w1, b1, w2 = (sd["noise_level_mlp." + k] for k in ("1.weight", "1.bias", "3.weight"))
    got = _native.test_film_embed_bwd(*(t.cuda() for t in (wf, tau, dfilm, nl, w1, b1, w2)), gscale=0.37)
    ref = film_reference(wf, tau, dfilm, nl, w1, b1, w2, 0.37)
    for k in ref:
        check(got[k], ref[k], f"{k} inner={inner} B={B} nl={nl_kind} scale={scale}")


@pytest.mark.parametrize("inner,B", [(64, 81), (128, 41), (256, 21)])
def test_differentiable_forward_past_the_batch_limit_is_refused_before_allocating(inner, B):
    """A differentiable forward whose batch the FiLM / noise-level MLP backward cannot hold in one block's shared memory is refused when its
    training engine is created, with the kernels' message, before any device memory is taken: not at the end of the first backward."""
    unet = dict(ui.TINY, inner_channel=inner)
    net = tu.build_train_net(unet, 32, ui.SEED, "l1", tu.SCHED, True)
    dn = net.denoise_fn
    x = torch.randn(B, 6, 32, 32, device="cuda", requires_grad=True)
    nl = torch.rand(B, 1, device="cuda", requires_grad=True)
    keys = set(dn._engines)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(RuntimeError, match="batch %d too large for one block's shared memory" % B):
        dn(x, nl)
    assert set(dn._engines) == keys and torch.cuda.mem_get_info()[0] == free0

"""GPU parity of the TRAINING row (SURVEY.md 8f rank 1; reference model/model.py:48-58 optimize_parameters, diffusion.py:221-246 p_losses):
gradients of every parameter from the native backward (dgrad = forward tile kernel on re-packed weights, wgrad = wgmma MN-major GEMM,
GroupNorm / SiLU / Dropout / attention backward kernels) against the oracle's fp32 CPU autograd, Adam iterations against the golden fixture.
bf16 tensor-core operands: tolerance 1e-2 on smooth losses; the L1 loss (sign(eps - noise) is discontinuous: a forward error of 1e-2 flips
~0.1 % of the signs, each flip moving the gradient by 2/N) is held to cosine similarity instead."""
import os

import numpy as np
import pytest
import torch

import _philox
import _train_util as tu
from _lowres_inputs import TINY4
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)
THREE = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 2], attn_res=[8], res_blocks=1, dropout=0.0)
GRAD_TOL = 2e-2          # relative L2 per parameter tensor (bf16 operands in forward, dgrad and wgrad: three roundings per path)


@pytest.fixture(scope="module")
def train_golden():
    return torch.load(os.path.join(HERE, "golden", "sr3_train_golden.pt"), weights_only=False)


@pytest.mark.parametrize("name,unet,R,B", [("tiny", TINY, 32, 2), ("three_levels_8x8_attention_odd_batch", THREE, 32, 3)])
def test_gradients_match_oracle_l2(name, unet, R, B):
    net = tu.build_train_net(unet, R, 5, "l2")
    hr, sr, noise = tu.batch(B, R, 1000)
    gamma = tu.draw_gamma(B, 7)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    lr_, gr = tu.oracle_loss_and_grads(net, unet, R, hr, sr, gamma, noise, "l2")
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    rows = tu.compare(go, gr)
    assert set(go) == set(gr)
    worst = sorted(rows, key=lambda r: -r[1])[:5]
    print("worst:", [(n, f"{e:.2e}") for n, e, _, _ in worst])
    for n, e, c, _ in rows:
        assert e < GRAD_TOL, (n, e, c)


@pytest.mark.timeout(900)
def test_gradients_full_16_128_config():
    """sr_sr3_16_128.json (five levels 128..8, two ResnetBlocks per level, attention at 16x16 and in the middle block, 97.8 M parameters), two
    images: the gradient of every one of the 362 parameter tensors against the oracle's fp32 autograd."""
    full = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
    net = tu.build_train_net(full, 128, 5, "l2")
    hr, sr, noise = tu.batch(2, 128, 1000)
    gamma = tu.draw_gamma(2, 7)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    torch.set_num_threads(min(16, torch.get_num_threads()))
    lr_, gr = tu.oracle_loss_and_grads(net, full, 128, hr, sr, gamma, noise, "l2")
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    rows = tu.compare(go, gr)
    assert len(rows) == 362
    worst = sorted(rows, key=lambda r: -r[1])[:8]
    print("worst:", [(n, f"{e:.2e}", f"{c:.5f}") for n, e, c, _ in worst])
    bad = [(n, e, c) for n, e, c, _ in rows if e >= 3e-2]
    assert not bad, bad[:10]


def test_gradients_unconditional_model():
    """sample_sr3_128.json-style model (in_channel 3, no condition image: diffusion.py:238-241 feeds x_noisy alone)."""
    unet = dict(TINY, in_channel=3)
    net = tu.build_train_net(unet, 32, 5, "l2", conditional=False)
    hr, sr, noise = tu.batch(2, 32, 1000)
    gamma = tu.draw_gamma(2, 7)
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    lr_, gr = tu.oracle_loss_and_grads(net, unet, 32, hr, sr, gamma, noise, "l2")
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    for n, e, c, _ in tu.compare(go, gr):
        assert e < GRAD_TOL, (n, e, c)


def test_gradients_l1_and_reference_optimize_parameters_semantics(train_golden):
    """The loss the reference trains with (L1, sum / (b c h w)): loss value within 1e-2 of the golden, gradients of all parameters close in
    direction to the golden ones (signatures: norms and samples recorded from the unmodified reference)."""
    g = train_golden
    net = tu.build_train_net(g["unet"], g["res"], g["seed"], "l1", g["sched"])
    hr, sr, noise = tu.batch(g["batch"], g["res"], 1000)
    rec = g["steps"][0]
    sch = orc.make_schedule(g["sched"])
    _, gamma = orc.draw_gamma(sch, g["batch"], np.random.RandomState(rec["np_seed"]))
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise)
    b, c, h, w = hr.shape
    assert abs(lo / (b * c * h * w) - rec["loss"]) < 1e-2 * abs(rec["loss"]), (lo / (b * c * h * w), rec["loss"])
    assert set(go) == set(rec["grads"])
    bad = []
    for k, sig in rec["grads"].items():
        f = go[k].flatten().cpu()
        assert f.numel() == sig["numel"]
        if abs(f.norm().item() - sig["norm"]) > 0.15 * sig["norm"] + 1e-12:
            bad.append((k, f.norm().item(), sig["norm"]))
    assert not bad, bad[:5]
    # same comparison against the oracle with the SAME sign pattern the device forward produced would be exact; the direction test:
    _, gr = tu.oracle_loss_and_grads(net, g["unet"], g["res"], hr, sr, gamma, noise, "l1")
    for n, e, cs, _ in tu.compare(go, gr):
        assert cs > 0.95, (n, e, cs)


def test_dropout_masks_of_the_reference(train_golden):
    """Training-mode forward / backward with the reference's own Dropout masks injected (unet.py:86,100-101): L2-free check of the mask
    plumbing -- loss within 1e-2 of the golden value, and different from the eval-mode loss."""
    g = train_golden
    d = g["dropout"]
    net = tu.build_train_net(g["unet_dropout"], g["res"], g["seed"], "l1", g["sched"])
    hr, sr, noise = tu.batch(g["batch"], g["res"], 1000 + d["batch_index"])
    sch = orc.make_schedule(g["sched"])
    _, gamma = orc.draw_gamma(sch, g["batch"], np.random.RandomState(d["np_seed"]))
    net.train(True)
    eng = net.denoise_fn.engine(g["batch"], conditional=True, channels=3, train_dropout=float(d["p"]))
    assert sorted(eng.dropout_layers()) == sorted(d["masks"])
    for k, (bits, shape) in d["masks"].items():
        keep = np.unpackbits(bits.numpy())[: int(np.prod(shape))].reshape(shape)
        eng.set_dropout_mask(k, torch.from_numpy(keep.astype(np.uint8)).cuda().contiguous())
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True)
    b, c, h, w = hr.shape
    assert abs(lo / (b * c * h * w) - d["loss"]) < 1e-2 * abs(d["loss"]), (lo / (b * c * h * w), d["loss"])
    for k, sig in d["grads"].items():
        f = go[k].flatten().cpu()
        assert abs(f.norm().item() - sig["norm"]) <= 0.15 * sig["norm"] + 1e-12, (k, f.norm().item(), sig["norm"])
    with torch.no_grad():
        net.eval()
        ev = net.p_losses({"HR": hr.cuda(), "SR": sr.cuda()}, noise=noise.cuda(), gamma=gamma).item()
    assert abs(ev - lo) / lo > 1e-4


def dropout_shapes(unet, R, B):
    """{"downs.1.res_block.block2": (B, C, H, W), ...}: the activation each ResnetBlock's nn.Dropout masks (unet.py:86,100-101)."""
    downs, mid, ups = orc.unet_topology(tu.oracle_cfg(unet, R))
    return {s.name + ".res_block.block2": (B, s.cout, s.res, s.res) for s in downs + mid + ups if s.kind == "res"}


def check_dropout_gradients(net, unet, R, hr, sr, gamma, noise, masks, dropout_seed=0):
    lo, go = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=dropout_seed)
    lr_, gr = tu.oracle_loss_and_grads(net, unet, R, hr, sr, gamma, noise, "l2", dropout_masks=masks)
    assert abs(lo - lr_) / abs(lr_) < 1e-2, (lo, lr_)
    assert set(go) == set(gr)
    for n, e, c, _ in tu.compare(go, gr):
        assert e < GRAD_TOL, (n, e, c)
    return lo


@pytest.mark.parametrize("name,unet,R,B", [("tiny", TINY, 32, 2), ("tiny_4x4", TINY4, 16, 3)])
def test_dropout_gradients_match_oracle_on_injected_masks(name, unet, R, B):
    """Random keep-masks (p = 0.2) injected into every block2 Dropout: every gradient tensor against the oracle's fp32 autograd with the
    same masks.  A backward that evaluated a different mask from the forward's fails here (the gradient norms alone would barely move)."""
    p = 0.2
    unet = dict(unet, dropout=p)
    net = tu.build_train_net(unet, R, 5, "l2")
    hr, sr, noise = tu.batch(B, R, 1000)
    gamma = tu.draw_gamma(B, 7)
    net.train(True)
    eng = net.denoise_fn.engine(B, conditional=True, channels=3, train_dropout=p)
    shapes = dropout_shapes(unet, R, B)
    assert sorted(eng.dropout_layers()) == sorted(shapes)
    g = torch.Generator().manual_seed(21)
    masks = {}
    for k, shape in shapes.items():
        keep = (torch.rand(shape, generator=g) >= p).to(torch.uint8)
        eng.set_dropout_mask(k, keep.cuda().contiguous())
        masks[k] = _philox.scale_mask(keep, p)
    try:
        check_dropout_gradients(net, unet, R, hr, sr, gamma, noise, masks)
    finally:
        for k in shapes:
            eng.set_dropout_mask(k, None)


def test_dropout_gradients_match_oracle_on_philox_masks():
    """The device's own Philox masks (dropout_seed), reproduced bit for bit by the numpy restatement of drop_scale4 (tests/_philox.py): the
    layer index of a Dropout is its position in eng.dropout_layers() (the order the plan numbers them in, DropSpec.layer).  Every gradient
    tensor against the oracle's fp32 autograd on those masks."""
    p, B, R, seed = 0.2, 2, 32, 0x5EED0000C0FFEE
    unet = dict(TINY, dropout=p)
    net = tu.build_train_net(unet, R, 5, "l2")
    hr, sr, noise = tu.batch(B, R, 1000)
    gamma = tu.draw_gamma(B, 7)
    net.train(True)
    eng = net.denoise_fn.engine(B, conditional=True, channels=3, train_dropout=p)
    shapes = dropout_shapes(unet, R, B)
    masks = {}
    for layer, k in enumerate(eng.dropout_layers()):
        b, c, h, w = shapes[k]
        keep = _philox.keep_mask(b, c, h * w, p, seed, layer).reshape(b, c, h, w)
        masks[k] = _philox.scale_mask(keep, p)
    check_dropout_gradients(net, unet, R, hr, sr, gamma, noise, masks, dropout_seed=seed)


def test_philox_dropout_is_deterministic():
    unet = dict(TINY, dropout=0.2)
    net = tu.build_train_net(unet, 32, 5, "l2")
    hr, sr, noise = tu.batch(2, 32, 1000)
    gamma = tu.draw_gamma(2, 7)
    l1, g1 = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=11)
    l2, g2 = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=11)
    l3, _ = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=True, dropout_seed=12)
    # same seed -> same masks: identical loss.  The backward's reductions use fp32 atomics (order dependent at 1e-7); every bf16 rounding of a
    # gradient operand amplifies a perturbation d to ~2^-4 sqrt(d), so after a few layers two runs differ by the bf16 noise floor (2^-8).
    worst = sorted(((tu.rel(g1[k], g2[k]), k, float(g1[k].norm())) for k in g1), reverse=True)[:5]
    print("run-to-run:", worst)
    assert l1 == l2 and worst[0][0] < 2e-2, worst
    assert l1 != l3
    # the masks drop ~20 % of block2's activations: the loss differs from the eval-mode loss
    l0, _ = tu.ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=False)
    assert l0 != l1


def test_three_adam_steps_reference_wrapper_flow(train_golden):
    """model/model.py:39-58 with our FusedAdam in place of torch.optim.Adam: zero_grad -> netG(data) -> sum / (b c h w) -> backward -> step,
    three iterations with the golden draws; the parameter UPDATES follow the reference's (cosine of (p_after - p_init))."""
    import sr3_b200
    g = train_golden
    net = tu.build_train_net(g["unet"], g["res"], g["seed"], "l1", g["sched"])
    net.eval()                                    # the golden Adam run has dropout 0
    init = {k: v.detach().clone() for k, v in net.denoise_fn.state_dict().items()}
    opt = sr3_b200.FusedAdam(list(net.parameters()), lr=g["lr"])
    sch = orc.make_schedule(g["sched"])
    for i, rec in enumerate(g["steps"]):
        hr, sr, noise = tu.batch(g["batch"], g["res"], 1000 + i)
        _, gamma = orc.draw_gamma(sch, g["batch"], np.random.RandomState(rec["np_seed"]))
        opt.zero_grad()
        b, c, h, w = hr.shape
        l = net.p_losses({"HR": hr.cuda(), "SR": sr.cuda()}, noise=noise.cuda(), gamma=gamma)
        l = l.sum() / int(b * c * h * w)
        l.backward()
        opt.step()
        assert abs(l.item() - rec["loss"]) < 2e-2 * abs(rec["loss"]), (i, l.item(), rec["loss"])
    after = net.denoise_fn.state_dict()
    moved = 0
    for k, sig in g["params_after"].items():
        f = after[k].flatten().cpu()
        stride = max(1, f.numel() // 16)
        # the reference's parameters after three steps (samples): ours must have moved the same way (Adam's first steps are ~ lr * sign(g))
        d_ours = (f - init[k].flatten().cpu())[::stride][:16]
        d_ref = sig["samples"] - init[k].flatten().cpu()[::stride][:16]
        if d_ref.norm() > 0:
            moved += 1
            assert (d_ours - d_ref).norm() <= 0.5 * d_ref.norm() + 1e-7, (k, d_ours, d_ref)
    assert moved > 50


def test_fused_adam_matches_torch_adam():
    """sr3_b200.FusedAdam (one native launch over a device table of tensors) against torch.optim.Adam with the reference's settings
    (model/model.py:39-40: lr from the config, torch defaults otherwise), five steps on tensors of assorted shapes."""
    import sr3_b200
    g = torch.Generator().manual_seed(0)
    shapes = [(64, 6, 3, 3), (64,), (128, 64, 3, 3), (256, 64), (3, 64, 3, 3), (1,)]
    pa = [torch.nn.Parameter(torch.randn(s, generator=g).cuda()) for s in shapes]
    pb = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    oa, ob = sr3_b200.FusedAdam(pa, lr=1e-4), torch.optim.Adam(pb, lr=1e-4)
    for step in range(5):
        for x, y in zip(pa, pb):
            gr = torch.randn(x.shape, generator=g).cuda() * (10.0 ** (step - 2))
            x.grad, y.grad = gr.clone(), gr.clone()
        oa.step(); ob.step()
    for x, y in zip(pa, pb):
        assert torch.allclose(x, y, rtol=1e-5, atol=1e-7), (x.shape, (x - y).abs().max().item())
    assert oa.state_dict()["param_groups"][0]["step"] == 5

"""Images of another size than the net's image_size, non-square included (sr3_engine_create_sized).

UNet-level cases compare against the unmodified reference's outputs in tests/golden/sr3_sizes_golden.pt (tests/golden/make_sizes_golden.py,
inputs from tests/_sizes_inputs.py; tests/test_oracle_sizes.py pins the oracle to the same fixture) at the project's bf16 and precise-mode
tolerances.  The rest checks what the size must not change: the plan at image_size, bit reproducibility, batch sharding, weight updates across cached engines, and refusal of unsupported sizes before anything is allocated."""
import ctypes
import os
import sys

import pytest
import torch

import _sizes_inputs as si
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

BF16_TOL, FP32_TOL = 1e-2, 1e-3
# bf16 per-layer bound of the five-level nets, whose taps are small crops of image 0 on their 256- and 512-channel levels: measured up to
# 1.19e-2 on an H100 (16->64 at 128x128: mid.0 1.09e-2, ups.7 1.13e-2; 16->128 at 128x256: mid.0 1.19e-2, ups.5 1.00e-2), the rounding
# of up to ~20 bf16 layers; the same layers match within 6e-5 in precise mode, and eps stays within BF16_TOL (7.2e-3)
BF16_DEEP_TOL = 2e-2
KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED6 = {"schedule": "linear", "n_timestep": 6, "linear_start": 1e-4, "linear_end": 2e-2}


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def clear_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def make_opt(unet, image_size, sched):
    return {"phase": "val", "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}


def build(unet, image_size, seed, sched=si.SCHED, precision="bf16"):
    import sr3_b200
    torch.manual_seed(seed)
    net = sr3_b200.define_G(make_opt(dict(unet, precision=precision), image_size, sched)).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


@pytest.fixture(scope="module")
def sizes():
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sr3_sizes_golden.pt"), map_location="cpu",
                      weights_only=False)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("name", sorted(si.CASES))
def test_eps_and_layers_match_reference(monkeypatch, sizes, name, precision):
    """eps and the per-layer outputs (attention over 512 / 1024 tokens, an 8x8 lowest level of a net built with a 4x4 one, 128x256)."""
    clear_knobs(monkeypatch)
    unet, image_size, seed, b, h, w = si.CASES[name][:6]
    g, inp = sizes[name], si.inputs(name)
    net = build(unet, image_size, g["seed"], precision=precision)
    eps = net.denoise_fn(inp["x"].cuda(), inp["noise_level"].cuda())
    assert eps.shape == (b, 3, h, w) and torch.isfinite(eps).all()
    tol = BF16_TOL if precision == "bf16" else FP32_TOL
    eng = net.denoise_fn.engine(b, height=h, width=w)
    assert (eng.height, eng.width) == (h, w)
    deep = len(unet["channel_multiplier"]) == 5
    errs = {layer: rel(si.tap_crop(name, layer, eng.read_activation(layer)), ref) for layer, ref in g["taps"].items()}
    errs["eps"] = rel(si.eps_crop(name, eps), g["eps"])
    print(f"{name} {precision} rel err:", {k: f"{v:.2e}" for k, v in errs.items()})
    for layer, e in errs.items():
        assert e < (BF16_DEEP_TOL if precision == "bf16" and deep and layer != "eps" else tol), (layer, e)


@pytest.mark.timeout(900)
def test_pmv_and_loop_at_128x256(monkeypatch, sizes):
    """p_mean_variance at t = 1999, 1000, 1 and the reference's 10-step loop with the same draws injected, on the 16->128 config."""
    clear_knobs(monkeypatch)
    name = si.LOOP_CASE
    unet, image_size = si.CASES[name][:2]
    g, inp = sizes[name], si.inputs(name)
    net = build(unet, image_size, g["seed"])
    sch = orc.make_schedule(si.SCHED)
    cond, x_t = inp["cond"].cuda(), inp["x_t"].cuda()
    for t in si.T_EVAL:
        eps = net.denoise_fn(torch.cat([cond, x_t], 1), orc.noise_level_for_t(sch, t, 2).cuda())
        assert rel(si.eps_crop(name, eps), g["eps_t"][t]) < BF16_TOL, t
        mean, lv = net.p_mean_variance(x_t, t, True, condition_x=cond)
        assert mean.shape == (2, 3, 128, 256)
        assert rel(si.eps_crop(name, mean), g["pmv"][t][0]) < BF16_TOL and float(lv) == float(g["pmv"][t][1]), t
    net.set_new_noise_schedule(si.SCHED10, "cuda")
    d = si.loop_inputs()
    out = net.super_resolution(cond, continous=True, x_T=d["x_T"].cuda(), noises=d["noises"].cuda())
    assert out.shape == (2 * 11, 3, 128, 256)
    assert rel(si.eps_crop(name, out[10:12]), g["loop_mid"]) < BF16_TOL
    assert rel(si.eps_crop(name, out[-2:]), g["loop_last"]) < BF16_TOL


def test_sized_create_at_image_size_is_the_plain_create(monkeypatch):
    """sr3_engine_create_sized(image_size, image_size) builds the plan sr3_engine_create builds: same ops, same variant and schedule of
    every tile op, the same eps bits."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    net = build(si.FULL, 128, 0)
    unet = net.denoise_fn
    cfg = dict(unet.arch, channels=3, conditional=True, precision="bf16")
    g = torch.Generator().manual_seed(9)
    x, nl = torch.randn(4, 6, 128, 128, generator=g), torch.rand(4, 1, generator=g)
    runs = {}
    lib = _native.lib()
    for how in ("sized", "plain"):
        if how == "plain":
            monkeypatch.setattr(lib, "sr3_engine_create_sized", lambda c, b, h, w, dev, out: lib.sr3_engine_create(c, b, dev, out))
        eng = _native.Engine(cfg, 4, torch.device("cuda", 0))
        eng.load_state_dict(unet.state_dict())
        runs[how] = (eng.ops_per_step(), eng.tile_schedules(), eng.unet_forward(x, nl).cpu())
        monkeypatch.undo()
        del eng
    assert runs["sized"][0] == runs["plain"][0]
    assert runs["sized"][1] == runs["plain"][1]
    assert torch.equal(runs["sized"][2], runs["plain"][2])


@pytest.mark.parametrize("h,w", [(32, 64), (64, 32)])
def test_non_square_is_bit_reproducible(monkeypatch, h, w):
    """At a non-square size repeat runs give the same bits."""
    g = torch.Generator().manual_seed(h + w)
    B = 3
    cond, x_T = torch.rand(B, 3, h, w, generator=g) * 2 - 1, torch.randn(B, 3, h, w, generator=g)
    clear_knobs(monkeypatch)
    net = build(si.TINY, 32, 0, sched=SCHED6)
    a = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=5).cpu()
    b = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=5).cpu()
    assert a.shape == (B * 7, 3, h, w) and torch.equal(a, b) and torch.isfinite(a).all()


@pytest.mark.timeout(900)
def test_sharded_super_resolution_in_two_shards_at_128x256(monkeypatch):
    """Three 128x256 images through sharded_super_resolution: on one rank it is the whole-batch super_resolution bit for bit; as the two
    shards (two images, then one) of a two-rank group, each shard is the super_resolution of its images with the global first index bit
    for bit, and the gathered batch agrees with the whole batch within the bf16 tolerance (other batch sizes may pick other tile shapes
    and split-K factors; the Philox streams are the same)."""
    from sr3_b200 import parallel
    clear_knobs(monkeypatch)
    net = build(si.FULL, 128, 0, sched=SCHED6)
    g = torch.Generator().manual_seed(8)
    cond, x_T = torch.rand(3, 3, 128, 256, generator=g) * 2 - 1, torch.randn(3, 3, 128, 256, generator=g)
    whole = parallel.sharded_super_resolution(net, cond, x_T=x_T, seed=11).cpu()
    ref = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=11, first_index=0)[-3:].cpu()
    assert whole.shape == (3, 3, 128, 256) and torch.equal(whole, ref)
    parts = []
    for rank in (0, 1):                    # what each rank of a two-rank group samples (the all-gather only concatenates them)
        monkeypatch.setattr(parallel.dist, "is_initialized", lambda: True)
        monkeypatch.setattr(parallel.dist, "get_world_size", lambda group=None: 2)
        monkeypatch.setattr(parallel.dist, "get_rank", lambda group=None, r=rank: r)
        monkeypatch.setattr(parallel, "gather_shards", lambda local, n, group=None: local)
        parts.append(parallel.sharded_super_resolution(net, cond, x_T=x_T, seed=11).cpu())
        monkeypatch.undo()
    assert [p.shape[0] for p in parts] == [2, 1]
    for (lo, hi), part in zip(((0, 2), (2, 3)), parts):
        alone = net.super_resolution(cond[lo:hi].cuda(), continous=True, x_T=x_T[lo:hi].cuda(), seed=11, first_index=lo)[-(hi - lo):]
        assert torch.equal(part, alone.cpu()), (lo, hi)
    assert rel(torch.cat(parts), whole) < BF16_TOL


def test_two_sizes_share_one_weight_update(monkeypatch):
    """Engines of two sizes cached on one module both re-pack after an in-place optimizer-style update and after load_state_dict."""
    clear_knobs(monkeypatch)
    net = build(si.TINY, 32, 0)
    unet = net.denoise_fn
    g = torch.Generator().manual_seed(4)
    xs = {(h, w): torch.randn(2, 6, h, w, generator=g).cuda() for h, w in ((32, 64), (64, 64))}
    nl = torch.tensor([[0.3], [0.8]]).cuda()
    before = {k: unet(x, nl).cpu() for k, x in xs.items()}
    with torch.no_grad():
        for p in unet.parameters():
            p.mul_(1.01)
    after = {k: unet(x, nl).cpu() for k, x in xs.items()}
    fresh = build(si.TINY, 32, 1).denoise_fn
    fresh.load_state_dict(unet.state_dict())
    for k, x in xs.items():
        assert not torch.equal(after[k], before[k]), k
        assert torch.equal(fresh(x, nl).cpu(), after[k]), k
    unet.load_state_dict(build(si.TINY, 32, 0).denoise_fn.state_dict())
    for k, x in xs.items():
        assert torch.equal(unet(x, nl).cpu(), before[k]), k


@pytest.mark.parametrize("h,w,msg", [(16, 16, "< 4"), (96, 128, "powers of two"), (8, 8, "< 4")])
def test_unsupported_sizes_raise_before_allocating(monkeypatch, h, w, msg):
    """The 16 -> 64 config (five levels): 16x16 and 8x8 go below 4, 96x128 is not a power of two.  Nothing is allocated and no cached
    engine is released."""
    from sr3_b200 import _native
    clear_knobs(monkeypatch)
    net = build(si.SR16_64, 64, 0)
    unet = net.denoise_fn
    unet(torch.zeros(1, 6, 64, 64).cuda(), torch.full((1, 1), 0.5).cuda())
    keys = list(unet._engines)
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    with pytest.raises(_native.UnsupportedSizeError, match=msg):
        unet(torch.zeros(1, 6, h, w).cuda(), torch.full((1, 1), 0.5).cuda())
    with pytest.raises(_native.UnsupportedSizeError, match=msg):
        net.super_resolution(torch.zeros(1, 3, h, w).cuda())
    torch.cuda.synchronize()
    assert list(unet._engines) == keys
    assert torch.cuda.mem_get_info()[0] >= free - (2 << 20)         # (the two input tensors come from torch's cache)


@pytest.mark.timeout(900)
def test_reference_ddpm_test_super_resolves_128x256(monkeypatch, tmp_path):
    """model/model.py:60-78 unmodified (feed_data -> test -> get_current_visuals) over sr3_b200.define_G, with a 128x256 conditioning image
    for a net built at image_size 32 whose attention sits on its 4x4 level (16x32 = 512 tokens here)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref = os.path.join(root, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "model")):
        pytest.skip("reference sources not present (oracle/_ref is written by build())")
    clear_knobs(monkeypatch)
    sys.dont_write_bytecode = True
    monkeypatch.syspath_prepend(ref)
    for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
        monkeypatch.delitem(sys.modules, k)
    import model as ref_model
    import model.networks as ref_networks
    import sr3_b200
    monkeypatch.setattr(ref_networks, "define_G", sr3_b200.define_G)
    sched = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
    unet = dict(si.TINY, channel_multiplier=[1, 2, 2, 2], attn_res=[4])
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False, "path": {"checkpoint": str(tmp_path), "resume_state": None},
           "train": {"optimizer": {"type": "adam", "lr": 1e-4}},
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": unet, "beta_schedule": {"train": sched, "val": sched},
                     "diffusion": {"image_size": 32, "channels": 3, "conditional": True}}}
    try:
        torch.manual_seed(0)
        m = ref_model.create_model(opt)
        m.set_new_noise_schedule(sched, schedule_phase="val")
        g = torch.Generator().manual_seed(3)
        data = {"HR": torch.rand(2, 3, 128, 256, generator=g) * 2 - 1, "SR": torch.rand(2, 3, 128, 256, generator=g) * 2 - 1,
                "Index": torch.arange(2)}
        m.feed_data(data)
        m.test(continous=True)
        vis = m.get_current_visuals()
        assert vis["SR"].shape == (2 * 11, 3, 128, 256) and torch.isfinite(vis["SR"]).all()
        assert torch.equal(vis["SR"][:2], data["SR"].cpu())
        m.test(continous=False)
        last = m.get_current_visuals()["SR"]
        assert last.shape == (3, 128, 256) and torch.isfinite(last).all()
    finally:
        for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
            sys.modules.pop(k, None)

"""Few-step samplers on the device (DESIGN.md 3.11): respaced DDIM through every sampler's existing tables, and DPM-Solver++(2M) through
the canvas's solver merge (window_solver_merge_kernel, sr3_windowed_set_solver).

What is pinned: the engine against the fp64 oracle (oracle/fast_sampler_oracle.py) with injected x_T and noises, at the suite's tolerances;
DDIM with K = T and eta = 1 is the default sampler to table rounding; one window is super_resolution bit for bit and a multi-window canvas
matches the oracle's canvas-level solver; eta = 0 and DPM-Solver++ draw nothing, and runs repeat bit for bit; a default call after a spec'd
one is unchanged bit for bit; DDIM requests share a stream with DDPM and beta_schedule requests and each equals its request alone, on the
12-step schedule and on the trained 2000-step one (K = 1 .. 50 next to a 2000-step request)."""
import functools

import pytest
import torch

import _sizes_inputs as si
from oracle import fast_sampler_oracle as fso
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED12 = {"schedule": "linear", "n_timestep": 12, "linear_start": 1e-6, "linear_end": 1e-2}
LIN5 = {"schedule": "linear", "n_timestep": 5, "linear_start": 1e-4, "linear_end": 2e-2}
CONFIGS = {"tiny": (si.TINY, 32, orc.UNetConfig(6, 3, 64, 32, (1, 2), (16,), 1, 0.0, 32)),
           "sr16_64": (si.SR16_64, 64, orc.UNetConfig(6, 3, 64, 32, (1, 2, 4, 8, 8), (16,), 2, 0.0, 64))}
SPECS = [{"sampler": "ddim", "steps": 5, "eta": 0.0}, {"sampler": "ddim", "steps": 12, "eta": 0.0},
         {"sampler": "ddim", "steps": 5, "eta": 0.5}, {"sampler": "ddim", "steps": 12, "eta": 0.5},
         {"sampler": "ddim", "steps": 5, "eta": 1.0}, {"sampler": "ddim", "steps": 12, "eta": 1.0},
         {"sampler": "dpmpp_2m", "steps": 4}, {"sampler": "dpmpp_2m", "steps": 10}]
DDIM0 = {"sampler": "ddim", "steps": 6, "eta": 0.0}
DPM = {"sampler": "dpmpp_2m", "steps": 7}


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def build(monkeypatch, config, precision="bf16", sched=SCHED12):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    unet, image_size, _ = CONFIGS[config]
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet, precision=precision),
                     "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


def draws(B, H, W, seed, K=12):
    g = torch.Generator().manual_seed(seed)
    cond, x_T = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.randn(B, 3, H, W, generator=g)
    return cond, x_T, torch.randn(K, B, 3, H, W, generator=g)


@functools.lru_cache(maxsize=None)
def oracle_run(config, spec_items, window=None, overlap=(0, 0), H=None, W=None):
    """The fp64 oracle's continous output for the config's seed-0 weights (the same for both precisions)."""
    unet, image_size, cfg = CONFIGS[config]
    spec = dict(spec_items)
    H, W = H or image_size, W or image_size
    cond, x_T, noises = draws(1, H, W, 5, spec["steps"])
    import sr3_b200
    torch.manual_seed(0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                     "beta_schedule": {"train": SCHED12, "val": SCHED12},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}
    net = sr3_b200.define_G(opt)
    sd = {k[len("denoise_fn."):]: v.detach().cpu() for k, v in net.state_dict().items() if k.startswith("denoise_fn.")}
    with torch.no_grad():
        return fso.sample_loop(sd, cfg, SCHED12, spec, cond, x_T, list(noises), continous=True, window=window, overlap=overlap)


@pytest.mark.timeout(3600)
@pytest.mark.parametrize("precision,tol", [("bf16", 1e-2), ("fp32", 1e-3)])
@pytest.mark.parametrize("config", ["tiny", "sr16_64"])
def test_engine_matches_the_fp64_oracle(monkeypatch, config, precision, tol):
    net = build(monkeypatch, config, precision)
    size = CONFIGS[config][1]
    for spec in SPECS:
        cond, x_T, noises = draws(1, size, size, 5, spec["steps"])
        got = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), noises=noises.cuda(), sampler=spec).cpu()
        ref = oracle_run(config, tuple(sorted(spec.items())))
        assert got.shape == ref.shape and torch.equal(got[:1], cond), (spec, got.shape, ref.shape)
        assert rel(got[-1:], ref[-1:]) < tol and rel(got[1:2], ref[1:2]) < tol, (spec, rel(got[-1:], ref[-1:]), rel(got[1:2], ref[1:2]))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_ddim_at_K_equal_T_eta_1_is_the_default_sampler(monkeypatch, precision):
    net = build(monkeypatch, "tiny", precision)
    cond, x_T, noises = draws(2, 32, 32, 6)
    ddpm = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), noises=noises.cuda())
    ddim = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), noises=noises.cuda(),
                                sampler={"sampler": "ddim", "steps": 12, "eta": 1.0})
    assert ddim.shape == ddpm.shape and rel(ddim, ddpm) < 1e-5, rel(ddim, ddpm)
    # and with Philox noise: sigma > 0 at every t > 0, keyed by the same (seed, sample, pixel, t)
    a = net.super_resolution(cond.cuda(), x_T=x_T.cuda(), seed=9)
    b = net.super_resolution(cond.cuda(), x_T=x_T.cuda(), seed=9, sampler={"sampler": "ddim", "steps": 12, "eta": 1.0})
    assert rel(b, a) < 1e-5, rel(b, a)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_one_window_is_super_resolution_bit_for_bit(monkeypatch, precision):
    net = build(monkeypatch, "tiny", precision)
    cond, x_T, noises = draws(2, 32, 64, 7)
    for spec in (DDIM0, {"sampler": "ddim", "steps": 9, "eta": 0.7}, DPM):
        for kw in ({"seed": 3}, {"seed": 3, "continous": True}, {"noises": noises[:spec["steps"]].cuda(), "continous": True}):
            plain = net.super_resolution(cond.cuda(), x_T=x_T.cuda(), sampler=spec, **kw)
            win = net.super_resolution_windowed(cond.cuda(), window=(32, 64), x_T=x_T.cuda(), sampler=spec, **kw)
            assert torch.isfinite(win).all() and torch.equal(win, plain), (spec, kw)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision,tol", [("bf16", 1e-2), ("fp32", 1e-3)])
def test_multi_window_canvas_matches_the_oracle(monkeypatch, precision, tol):
    net = build(monkeypatch, "tiny", precision)
    H, W, window, overlap = 40, 72, (32, 32), (8, 8)
    for spec in ({"sampler": "ddim", "steps": 5, "eta": 0.5}, {"sampler": "dpmpp_2m", "steps": 6}):
        cond, x_T, noises = draws(1, H, W, 5, spec["steps"])
        got = net.super_resolution_windowed(cond.cuda(), window=window, overlap=overlap, continous=True, x_T=x_T.cuda(),
                                            noises=noises.cuda(), sampler=spec).cpu()
        ref = oracle_run("tiny", tuple(sorted(spec.items())), window, overlap, H, W)
        assert got.shape == ref.shape, (got.shape, ref.shape)
        assert rel(got[-1:], ref[-1:]) < tol and rel(got[2:3], ref[2:3]) < tol, (spec, rel(got[-1:], ref[-1:]), rel(got[2:3], ref[2:3]))


@pytest.mark.timeout(900)
def test_noise_free_samplers_ignore_the_seed_and_repeat(monkeypatch):
    net = build(monkeypatch, "tiny")
    cond, x_T, _ = draws(2, 40, 56, 8)
    for spec in (DDIM0, DPM):
        for call in (lambda s: net.super_resolution(cond[:, :, :32, :32].cuda(), x_T=x_T[:, :, :32, :32].cuda(), seed=s, sampler=spec),
                     lambda s: net.super_resolution_windowed(cond.cuda(), x_T=x_T.cuda(), seed=s, sampler=spec)):
            a, b, c = call(1), call(2 ** 50 + 7), call(1)
            assert torch.isfinite(a).all() and torch.equal(a, b) and torch.equal(a, c), spec
    # a noisy DDIM depends on the seed and repeats
    spec = {"sampler": "ddim", "steps": 6, "eta": 0.5}
    a, b, c = (net.super_resolution_windowed(cond.cuda(), x_T=x_T.cuda(), seed=s, sampler=spec) for s in (1, 2, 1))
    assert not torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.timeout(900)
def test_default_call_after_a_spec_is_unchanged(monkeypatch):
    net = build(monkeypatch, "tiny")
    cond, x_T, _ = draws(2, 32, 32, 9)
    big_c, big_x, _ = draws(1, 40, 56, 10)
    before = (net.super_resolution(cond.cuda(), x_T=x_T.cuda(), seed=4, continous=True),
              net.super_resolution_windowed(big_c.cuda(), x_T=big_x.cuda(), seed=4, continous=True))
    for spec in (DDIM0, {"sampler": "ddim", "steps": 3, "eta": 1.0}, DPM):
        net.super_resolution(cond.cuda(), x_T=x_T.cuda(), seed=4, sampler=spec)
        net.super_resolution_windowed(big_c.cuda(), x_T=big_x.cuda(), seed=4, sampler=spec)
    with pytest.raises(ValueError, match="'steps'"):                     # a refused spec changes nothing either
        net.super_resolution(cond.cuda(), x_T=x_T.cuda(), sampler={"sampler": "dpmpp_2m", "steps": 13})
    after = (net.super_resolution(cond.cuda(), x_T=x_T.cuda(), seed=4, continous=True),
             net.super_resolution_windowed(big_c.cuda(), x_T=big_x.cuda(), seed=4, continous=True))
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])


@pytest.mark.timeout(900)
def test_unconditional_sample_takes_both_samplers(monkeypatch):
    import sr3_b200
    unet, image_size, _ = CONFIGS["tiny"]
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet, in_channel=3),
                     "beta_schedule": {"train": SCHED12, "val": SCHED12},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": False}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(SCHED12, "cuda")
    for spec in (DDIM0, DPM):
        out = net.sample(batch_size=2, continous=True, sampler=spec)
        kept = len([k for k in range(spec["steps"]) if k % (1 | spec["steps"] // 10) == 0])
        assert out.shape == ((1 + kept) * 2, 3, 32, 32)          # [x_T ; the kept states], two images each
        assert torch.isfinite(out).all()


# (module schedule, request sizes, per-request schedules or sampler specs; None = the module's schedule)
STREAM_CASES = {
    "sched12": (SCHED12, [(40, 56), (32, 32), (32, 72), (32, 32), (56, 48), (40, 40)],
                [{"sampler": "ddim", "steps": 5, "eta": 0.0}, None, LIN5, {"sampler": "ddim", "steps": 7, "eta": 1.0},
                 {"sampler": "ddim", "steps": 3, "eta": 0.5}, {"sampler": "ddim", "steps": 5, "eta": 0.0}]),
    # the trained 2000-step schedule: K = 1 is admitted at t = 0 and finishes after one step, next to a 2000-step request
    "sr3_2000": (si.SCHED, [(32, 32), (40, 56), (32, 32), (32, 72), (40, 40)],
                 [{"sampler": "ddim", "steps": 1, "eta": 0.0}, None, {"sampler": "ddim", "steps": 2, "eta": 1.0},
                  {"sampler": "ddim", "steps": 10, "eta": 0.5}, {"sampler": "ddim", "steps": 50, "eta": 0.0}]),
}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision,case", [pytest.param("bf16", "sched12", id="bf16"), pytest.param("fp32", "sched12", id="fp32"),
                                            pytest.param("bf16", "sr3_2000", id="bf16-sr3_2000"),
                                            pytest.param("fp32", "sr3_2000", id="fp32-sr3_2000")])
def test_stream_ddim_requests_equal_each_request_alone(monkeypatch, precision, case):
    sched, sizes, scheds = STREAM_CASES[case]
    net = build(monkeypatch, "tiny", precision, sched=sched)
    monkeypatch.setattr(net, "WINDOW_PASS_SIZES", (8,))      # the references run on the stream's engine
    g = torch.Generator().manual_seed(21)
    reqs = [((torch.rand(3, H, W, generator=g) * 2 - 1).cuda(), torch.randn(3, H, W, generator=g).cuda()) for H, W in sizes]
    seed, first = 77, 3
    rq = [(n, c, x) if s is None else (n, c, x, s) for n, ((c, x), s) in enumerate(zip(reqs, scheds))]
    out = dict(net.super_resolution_windowed_stream(rq, slots=8, seed=seed, first_index=first))
    assert sorted(out) == list(range(len(reqs)))
    for n, ((c, x), s) in enumerate(zip(reqs, scheds)):
        if s is not None and "sampler" not in s:
            net.set_new_noise_schedule(s, "cuda")
            try:
                ref = net.super_resolution_windowed(c[None], x_T=x[None], seed=seed, first_index=first + n)
            finally:
                net.set_new_noise_schedule(sched, "cuda")
        else:
            ref = net.super_resolution_windowed(c[None], x_T=x[None], seed=seed, first_index=first + n, sampler=s)
        assert torch.isfinite(ref).all() and torch.equal(out[n], ref), (n, s)
    # a DPM-Solver++ request is refused by name before anything is admitted
    with pytest.raises(ValueError, match="request 'p'.*dpmpp_2m"):
        list(net.super_resolution_windowed_stream([("p", reqs[1][0], None, DPM)], slots=8, seed=seed))
    with pytest.raises(ValueError, match="request 'q'.*'eta'"):
        list(net.super_resolution_windowed_stream([("q", reqs[1][0], None, {"sampler": "ddim", "steps": 3, "eta": 2})], slots=8))

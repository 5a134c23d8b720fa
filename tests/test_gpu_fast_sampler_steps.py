"""Every few-step sampler update on the device against its definition, on the trained 2000-step schedule (DESIGN.md 3.11).

The whole-trajectory tests (tests/test_gpu_fast_samplers.py) run a 12-step schedule within a relative tolerance; on SR3's 2000-step schedule
neighbouring noise levels are close and c1 = sqrt(1 / abar), c2 = sqrt(1 / abar - 1) reach 151, so an off-by-one in a table index, the Philox
key or the x0 history would pass them.  Here every step is pinned on its own, on the schedule the samplers ship for:
* DDIM: the device's mean is clamp(c1 x - c2 eps) then pc1 x0 + pc2 x in torch-CPU fp32 on the engine's own eps, bit for bit, with the UNet
  conditioned on fp32(sqrt(abar[tau_k])) computed here from oracle/fast_sampler_oracle.py, not from samplers.py; the noise is the documented
  Philox stream keyed by the step index k, within test_gpu_sampling._noise_bound;
* the loops equal their chained steps at every snapshot (engine and canvas, conditional and unconditional, Philox and injected noises);
* DPM-Solver++(2M) on a canvas: the windows' clipped x0 (the engine's own per-pass means) blended in ascending window order, then
  x_{k-1} = (A x + B x0) + C x0_prev, bit for bit, with x0_prev the previous step's blended x0 (zero before the first step);
* the 16->128 config at batch 16, the shape the few-step benchmark (tools/gpu_fast_sampler_bench.py) times.
Each check also evaluates wrong references (neighbouring noise level, DDPM rows, other Philox keys, the next step's A/B/C, a stale or
missing x0_prev) and requires them to miss, so that a sampler with such a fault would fail."""
import math

import numpy as np
import pytest
import torch

import _philox
import _sizes_inputs as si
from oracle import fast_sampler_oracle as fso
from test_gpu_plan import PLAN_16_128_B16
from test_gpu_sampling import _noise_bound
from test_gpu_windowed import device_window_means

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED = si.SCHED                                   # linear, 2000 steps, 1e-6 -> 1e-2: the schedule SR3 trains on
T = SCHED["n_timestep"]
ABAR = fso.alphas_cumprod(SCHED)
SEED = 2 ** 62 + 0x1234_5678_9ABC                  # both key words set
FIRST = 2 ** 32 - 1                                # every batch of 2 or more crosses the sample index's high word
ROWS = ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2")
# config -> (unet, image_size, batch, height, width) of the DDIM step checks
STEP_CONFIGS = {"tiny": (si.TINY, 32, 3, 32, 64), "sr16_64": (si.SR16_64, 64, 2, 64, 64)}
BENCH_UNET = dict(si.SR16_64, dropout=0.2)         # tools/gpu_fast_sampler_bench.py's 16->128 UNet (run in eval mode)


def build(monkeypatch, unet, image_size, precision, conditional=True):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    unet = dict(unet, precision=precision)
    if not conditional:
        unet["in_channel"] = 3
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": unet,
                     "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(SCHED, "cuda")
    net.eval()
    return net


def draws(B, H, W, seed, K=None):
    g = torch.Generator().manual_seed(seed)
    cond, x = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.randn(B, 3, H, W, generator=g)
    noises = None if K is None else torch.randn(K, B, 3, H, W, generator=g).cuda()
    return cond.cuda(), x.cuda(), noises


def level(K, k, tau=None):
    """(tau_k, fp32(sqrt(abar[tau_k]))) of step k of K: the trained timestep and the noise level the UNet is conditioned on."""
    tau = fso.timesteps(T, K)[k] if tau is None else tau
    return tau, float(np.float32(math.sqrt(ABAR[tau])))


def eps_at(eng, cond, x, nl):
    inp = x if cond is None else torch.cat([cond, x], 1)
    return eng.unet_forward(inp, torch.full((x.shape[0], 1), nl)).cpu()


def posterior(rows, x, eps):
    """x0 = clamp(c1 x - c2 eps), mean = pc1 x0 + pc2 x in torch-CPU fp32, every product and sum rounded on its own."""
    c1, c2, pc1, pc2 = rows
    x0 = (c1 * x - c2 * eps).clamp(-1.0, 1.0)
    return pc1 * x0 + pc2 * x, x0


def kept(K):
    """The step indices whose x_{k-1} the loops keep, in order (every 1 | K // 10 steps)."""
    inter = 1 | (K // 10)
    return [k for k in reversed(range(K)) if k % inter == 0]


def frac_changed(a, b, where=None):
    d = a != b
    if where is not None:
        d = d[where]
    return d.float().mean().item(), d.numel()


# ------------------------------------------------------------------------------------------------------------------- DDIM: one step
def check_ddim_step(net, eng, tables, K, eta, k, cond, x, label, neighbours=False):
    """One DDIM step k of K at x against its definition, with its wrong references."""
    bufs = tables[0]
    B, _, H, W = x.shape
    tau, nl = level(K, k)
    assert np.float32(tables[1][k + 1]) == np.float32(nl), (label, k, tables[1][k + 1], nl)
    x_cpu = x.cpu()
    eps = eps_at(eng, cond, x, nl)
    rows = [bufs[n][k] for n in ROWS]
    ref, x0 = posterior(rows, x_cpu, eps)
    with eng.sampling_on(tables):
        mean, lv = eng.p_mean_variance(x, k, True, cond)
        step = eng.p_sample(x, k, cond, None, SEED, FIRST).cpu()
        other = eng.p_sample(x, k, cond, None, 1, 0).cpu()
    mean = mean.cpu()
    diff = (mean != ref).sum().item()
    assert diff == 0, f"{label} K={K} eta={eta} k={k}: {diff} of {ref.numel()} means differ, max |d| {(mean - ref).abs().max().item():.3e}"
    want_lv = float(bufs["posterior_log_variance_clipped"][k])
    assert lv == want_lv, (label, K, eta, k, lv, want_lv)
    if eta == 0 or k == 0:
        assert lv == -math.inf, (label, K, eta, k, lv)
        assert torch.equal(step, mean) and torch.equal(other, mean), (label, K, eta, k)
    else:
        sigma = math.exp(0.5 * lv)
        idx = FIRST + np.arange(B, dtype=np.uint64)
        m64, s64 = mean.double().numpy(), step.double().numpy()
        z = _philox.sampling_noise(SEED, idx, k, H, W)
        ratio = np.abs(s64 - (m64 + sigma * z)) / _noise_bound(m64, z, sigma)
        assert ratio.max() <= 1.0, (label, K, eta, k, ratio.max())
        keys = {"k + 1": k + 1, "k - 1": k - 1}
        if tau != k:
            keys["tau_k"] = tau
        for name, key in keys.items():
            zw = _philox.sampling_noise(SEED, idx, key, H, W)
            rw = np.median(np.abs(s64 - (m64 + sigma * zw)) / _noise_bound(m64, zw, sigma))
            print(f"{label} K={K} eta={eta} k={k}: Philox keyed by {name} misses the bound by a median {rw:.3g}x (correct key: max {ratio.max():.3f})")
            assert rw > 1e2, (label, K, eta, k, name, rw)
    if tau > 0:                               # at tau = 0 the DDPM posterior returns x0, as DDIM's last step does
        ddpm = [getattr(net, n)[tau].cpu() for n in ROWS]
        wrong, _ = posterior(ddpm, x_cpu, eps)
        f, n = frac_changed(wrong, mean)
        print(f"{label} K={K} eta={eta} k={k}: the DDPM rows at tau={tau} change {f:.1%} of {n} means")
        assert f > 0.5, (label, K, eta, k, f)
    if neighbours:
        # c1, c2 ~ 151 at tau = 1999 clip most x0; the eps reaches the means whose x0 is not clipped
        free = x0.abs() < 1
        for tn in (tau - 1, tau + 1):
            if not 0 <= tn < T:
                continue
            wrong, _ = posterior(rows, x_cpu, eps_at(eng, cond, x, level(K, k, tn)[1]))
            f, n = frac_changed(wrong, mean, free)
            print(f"{label} K={K} eta={eta} k={k}: eps at the neighbouring level tau={tn} changes {f:.1%} of the {n} means with unclipped x0")
            assert n >= 10 and f > 0.5, (label, K, eta, k, tn, f, n)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("config", sorted(STEP_CONFIGS))
def test_one_ddim_step_is_its_definition(monkeypatch, config, precision):
    """DDIM K in {1, 2, 10, 50}, eta in {0, 0.5, 1}, at steps K - 1, K - 2, K // 2, 1 and 0 on the 2000-step schedule: the mean bit for bit,
    logvar the table's (-inf where sigma = 0), the noise the Philox stream keyed by k; the wrong references miss."""
    unet, image_size, B, H, W = STEP_CONFIGS[config]
    net = build(monkeypatch, unet, image_size, precision)
    eng = net._engine(B, H, W)
    cond, x, _ = draws(B, H, W, 3 * H + W)
    for K in (1, 2, 10, 50):
        for eta in (0.0, 0.5, 1.0):
            tables = net._sampler_tables(("ddim", K, eta))
            for k in sorted({K - 1, K - 2, K // 2, 1, 0} & set(range(K)), reverse=True):
                check_ddim_step(net, eng, tables, K, eta, k, cond, x, f"{config} {precision}", neighbours=(k == K - 1 and eta == 0.0))


# ------------------------------------------------------------------------------------------------------------------- the loops
def ddim_chain(eng, tables, K, cond, x_T, noises=None, seed=SEED, first=FIRST):
    """x_{k-1} after every step k of p_sample chained from x_T under the tables: {k: state}."""
    states, x = {}, x_T
    with eng.sampling_on(tables):
        for k in reversed(range(K)):
            x = eng.p_sample(x, k, cond, None if noises is None else noises[k], seed, first)
            states[k] = x
    return states


def dpm_chain(canvas, tables, K, cond, x_T):
    """x_{k-1} after every canvas.steps(k, 1) chained from one begin under the DPM-Solver++ tables: {k: state}."""
    states = {}
    with canvas.engine.sampling_on(tables):
        canvas.set_solver(tables[2])
        try:
            canvas.begin(cond, x_T, SEED, FIRST)
            for k in reversed(range(K)):
                canvas.steps(k, 1)
                states[k] = canvas.read_state()
        finally:
            canvas.set_solver(None)
    return states


def assert_snapshots(snaps, states, K, label):
    ks = kept(K)
    assert snaps.shape[0] == len(ks), (label, K, snaps.shape, len(ks))
    for i, k in enumerate(ks):
        assert torch.equal(snaps[i], states[k]), f"{label} K={K}: snapshot {i} (step k={k}): {(snaps[i] != states[k]).sum().item()} values differ"


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_ddim_loops_are_their_steps(monkeypatch, precision):
    """Engine.p_sample_loop(sampler=tables) and super_resolution(sampler=spec, continous=True) equal p_sample chained from x_T, bit for bit at
    every snapshot, for K in {1, 2, 10, 11, 20, 50} (the snapshot interval 1 | K // 10 is 1, 1, 1, 1, 3, 5), with Philox noise and with
    injected noises [K, ...]; noises[k] is the z of step k."""
    B, H, W = 2, 32, 64
    net = build(monkeypatch, si.TINY, 32, precision)
    eng = net._engine(B, H, W)
    for K in (1, 2, 10, 11, 20, 50):
        cond, x_T, noises = draws(B, H, W, 100 + K, K)
        # Philox
        spec = {"sampler": "ddim", "steps": K, "eta": 0.5}
        tables = net._sampler_tables(net._sampler_spec(spec))
        states = ddim_chain(eng, tables, K, cond, x_T)
        final, snaps = eng.p_sample_loop(cond, x_T, None, SEED, FIRST, want_snapshots=True, sampler=tables)
        assert_snapshots(snaps, states, K, f"{precision} philox loop")
        assert torch.equal(final, states[0])
        out = net.super_resolution(cond, continous=True, x_T=x_T, seed=SEED, first_index=FIRST, sampler=spec)
        assert torch.equal(out[:B], cond)
        assert_snapshots(out[B:].view(-1, B, 3, H, W), states, K, f"{precision} philox super_resolution")
        # injected noises
        spec = {"sampler": "ddim", "steps": K, "eta": 1.0}
        tables = net._sampler_tables(net._sampler_spec(spec))
        states = ddim_chain(eng, tables, K, cond, x_T, noises)
        final, snaps = eng.p_sample_loop(cond, x_T, noises, SEED, FIRST, want_snapshots=True, sampler=tables)
        assert_snapshots(snaps, states, K, f"{precision} noises loop")
        assert torch.equal(final, states[0])
        out = net.super_resolution(cond, continous=True, x_T=x_T, noises=noises, sampler=spec)
        assert_snapshots(out[B:].view(-1, B, 3, H, W), states, K, f"{precision} noises super_resolution")
        if K >= 2:                            # the first step draws noises[K - 1]: x = mean + sigma noises[K - 1]
            k = K - 1
            with eng.sampling_on(tables):
                mean, lv = eng.p_mean_variance(x_T, k, True, cond)
            m64, s64, sigma = mean.cpu().double().numpy(), states[k].cpu().double().numpy(), math.exp(0.5 * lv)
            for j in (k, k - 1):
                n64 = noises[j].cpu().double().numpy()
                ratio = np.abs(s64 - (m64 + sigma * n64)) / _noise_bound(m64, n64, sigma)
                if j == k:
                    assert ratio.max() <= 1.0, (precision, K, ratio.max())
                else:
                    print(f"{precision} K={K}: noises[k - 1] in place of noises[k] misses the bound by a median {np.median(ratio):.3g}x")
                    assert np.median(ratio) > 1e2, (precision, K, np.median(ratio))


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_dpm_canvas_loop_is_its_steps(monkeypatch, precision):
    """WindowedSampler.sample_loop(sampler=tables) and super_resolution_windowed(sampler=spec, continous=True) equal canvas.steps(k, 1)
    chained from one begin, bit for bit at every snapshot, on a six-window canvas for K in {2, 3, 10, 20}."""
    B, H, W, window, overlap = 1, 40, 72, (32, 32), 8
    net = build(monkeypatch, si.TINY, 32, precision)
    canvas = net._windowed_sampler(B, H, W, window, overlap)
    for K in (2, 3, 10, 20):
        cond, x_T, _ = draws(B, H, W, 200 + K)
        spec = {"sampler": "dpmpp_2m", "steps": K}
        tables = net._sampler_tables(net._sampler_spec(spec))
        states = dpm_chain(canvas, tables, K, cond, x_T)
        final, snaps = canvas.sample_loop(cond, x_T, None, SEED, FIRST, want_snapshots=True, sampler=tables)
        assert_snapshots(snaps, states, K, f"{precision} canvas sample_loop")
        assert torch.equal(final, states[0])
        out = net.super_resolution_windowed(cond, window=window, overlap=overlap, continous=True, x_T=x_T, sampler=spec)
        assert_snapshots(out[B:].view(-1, B, 3, H, W), states, K, f"{precision} super_resolution_windowed")


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_unconditional_loops_are_their_steps(monkeypatch, precision):
    """net.sample(sampler=...) on the unconditional tiny net: DDIM equals p_sample chained from its x_T under its seed, DPM-Solver++ equals
    the canvas steps chained from its x_T, bit for bit at every snapshot.  sample() returns its x_T as the first rows and draws its seed
    from torch's CPU generator (x_T comes from the CUDA one), so re-seeding that generator reproduces the seed it used."""
    B = 2
    net = build(monkeypatch, si.TINY, 32, precision, conditional=False)
    eng = net._engine(B, 32, 32)
    for spec in ({"sampler": "ddim", "steps": 1, "eta": 0.5}, {"sampler": "ddim", "steps": 11, "eta": 0.5},
                 {"sampler": "ddim", "steps": 50, "eta": 1.0}, {"sampler": "dpmpp_2m", "steps": 2}, {"sampler": "dpmpp_2m", "steps": 20}):
        K = spec["steps"]
        tables = net._sampler_tables(net._sampler_spec(spec))
        torch.manual_seed(K)
        out = net.sample(batch_size=B, continous=True, sampler=spec)
        x_T = out[:B]
        if spec["sampler"] == "ddim":
            torch.manual_seed(K)
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            states = ddim_chain(eng, tables, K, None, x_T, seed=seed, first=0)
        else:
            canvas = net._windowed_sampler(B, 32, 32, (32, 32), 0)
            states = dpm_chain(canvas, tables, K, None, x_T)
        assert_snapshots(out[B:].view(-1, B, 3, 32, 32), states, K, f"{precision} unconditional {spec}")


# ------------------------------------------------------------------------------------------------------------------- DPM-Solver++: one canvas step
def blend(canvas, means, shape):
    """The windows' means blended on the canvas as window_solver_merge_kernel blends them: ascending window index, separately rounded fp32
    products and sums, then one division."""
    oy, ox, wy, wx = canvas.grid()
    B, _, H, W = shape
    oh, ow = canvas.engine.height, canvas.engine.width
    num, den = torch.zeros(shape, device="cuda"), torch.zeros(B, 1, H, W, device="cuda")
    n = 0
    for b in range(B):
        for iy in range(len(oy)):
            for ix in range(len(ox)):
                w = (wy[iy][:, None] * wx[ix][None, :]).cuda()
                c = (slice(b, b + 1), slice(None), slice(oy[iy], oy[iy] + oh), slice(ox[ix], ox[ix] + ow))
                num[c] = num[c] + w * means[n]
                den[c] = den[c] + w
                n += 1
    assert (den > 0).all()
    return num / den


def check_dpm_canvas_steps(net, canvas, cond, x_T, label, K=20):
    """DPM-Solver++(2M) K steps from one begin, each against x_{k-1} = (A_k x + B_k x0) + C_k x0_prev on the device's state x, with x0 the
    blend of the engine's own per-pass means (under the DPM tables: the windows' clipped x0) and x0_prev the previous step's blended x0,
    bit for bit; step K - 1 is first order (C = 0), K - 2 the first to read x0_prev, 1 has the largest B and |C|, 0 (A = 0, B = 1)
    returns x0.  The wrong references (the A/B/C of step k + 1, x0_prev left at zero, x0_prev of two steps back) change most values
    where their input differs from the right one: the untrained nets clip most x0 to +-1 by step 1, so x0 of steps 2 and 3 agree on
    more than nine values in ten and there a stale x0_prev is the right one."""
    tables = net._sampler_tables(("dpmpp_2m", K, None))
    A, Bc, C = (r.cuda() for r in tables[2])
    assert C[K - 1] == 0 and A[0] == 0 and Bc[0] == 1 and C[0] == 0
    assert int(torch.argmax(Bc[1:])) + 1 == 1 and int(torch.argmax(C[1:].abs())) + 1 == 1, (Bc, C)
    zero = torch.zeros_like(x_T)
    x0s = {K: zero, K + 1: zero}                  # x0 of step k; zero before the first step
    with canvas.engine.sampling_on(tables):
        canvas.set_solver(tables[2])
        try:
            canvas.begin(cond, x_T, SEED, FIRST)
            x = x_T
            for k in reversed(range(K)):
                means, _ = device_window_means(canvas, cond, x, k)
                x0 = blend(canvas, means, tuple(x.shape))
                x0s[k] = x0
                ref = (A[k] * x + Bc[k] * x0) + C[k] * x0s[k + 1]
                canvas.steps(k, 1)
                got = canvas.read_state()
                diff = (got != ref).sum().item()
                assert diff == 0, f"{label} k={k}: {diff} of {ref.numel()} values differ, max |d| {(got - ref).abs().max().item():.3e}"
                if k == 0:
                    assert torch.equal(got, x0), label
                if k in (K - 2, 1):
                    # (wrong reference, the values where its input differs from the right one: elsewhere it is the right reference)
                    wrongs = {"A/B/C of step k + 1": ((A[k + 1] * x + Bc[k + 1] * x0) + C[k + 1] * x0s[k + 1], None),
                              "x0_prev left at zero": ((A[k] * x + Bc[k] * x0) + C[k] * zero, x0s[k + 1] != 0)}
                    if k + 2 < K:
                        wrongs["x0_prev of two steps back"] = ((A[k] * x + Bc[k] * x0) + C[k] * x0s[k + 2], x0s[k + 2] != x0s[k + 1])
                    for name, (wrong, where) in wrongs.items():
                        f, n = frac_changed(wrong, got, where)
                        print(f"{label} k={k}: {name} changes {f:.1%} of the {n} values where it differs from the right input "
                              f"({n / got.numel():.1%} of all)")
                        assert n >= 100 and f > 0.5, (label, k, name, f, n)
                x = got
        finally:
            canvas.set_solver(None)


DPM_CANVASES = {  # name -> (unet, image_size, batch, H, W, window, overlap, windows per pass or None)
    "tiny_70x99_unaligned": (si.TINY, 32, 2, 70, 99, (64, 64), (5, 0), None),
    "tiny_40x72_padded_pass": (si.TINY, 32, 1, 40, 72, (32, 32), 8, (4,)),
    "tiny_one_window": (si.TINY, 32, 2, 32, 64, (32, 64), 0, None),
    "full_200x312": (si.FULL, 128, 2, 200, 312, (128, 128), None, None),
}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("case", sorted(DPM_CANVASES))
def test_one_dpm_canvas_step_is_its_definition(monkeypatch, case, precision):
    unet, image_size, B, H, W, window, overlap, passes = DPM_CANVASES[case]
    net = build(monkeypatch, unet, image_size, precision)
    if passes is not None:
        monkeypatch.setattr(type(net), "WINDOW_PASS_SIZES", passes)
    canvas = net._windowed_sampler(B, H, W, window, overlap)
    oy, ox, _, _ = canvas.grid()
    if passes is not None:                        # the last pass runs fewer windows than the engine's batch
        assert (B * len(oy) * len(ox)) % canvas.engine.batch != 0, (oy, ox, canvas.engine.batch)
    cond, x_T, _ = draws(B, H, W, 300 + H + W)
    check_dpm_canvas_steps(net, canvas, cond, x_T, f"{case} {precision}")


# ------------------------------------------------------------------------------------------------------------------- the benchmarked shape
@pytest.mark.timeout(1800)
def test_benchmarked_shape_steps_are_their_definition(monkeypatch):
    """The 16->128 config (dropout 0.2, eval) at 128x128, batch 16, bf16: DDIM K = 50 (eta 0 and 0.5) at steps 49, 25, 1 and 0, and
    DPM-Solver++ K = 20 on its one-window canvas, step by step as above; on a 132-SM part the engine runs PLAN_16_128_B16, the plan the
    few-step benchmark times."""
    B, S = 16, 128
    net = build(monkeypatch, BENCH_UNET, S, "bf16")
    eng = net._engine(B, S, S)
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        got = [(i, tuple(s["out_hwc"]), s["tall"], 128 * s["mh"], s["block_n"], s["schedule"], s["ksplit"])
               for i, s in enumerate(eng.tile_schedules()) if s is not None]
        assert got == PLAN_16_128_B16
    cond, x, _ = draws(B, S, S, 16128)
    for eta in (0.0, 0.5):
        tables = net._sampler_tables(("ddim", 50, eta))
        for k in (49, 25, 1, 0):
            check_ddim_step(net, eng, tables, 50, eta, k, cond, x, "16->128 B16", neighbours=(k == 49 and eta == 0.0))
    canvas = net._windowed_sampler(B, S, S, (S, S), 0)
    assert canvas.engine is eng
    check_dpm_canvas_steps(net, canvas, cond, x, "16->128 B16")

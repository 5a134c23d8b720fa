"""Continuous batching of canvases of any size on the device (GaussianDiffusion.super_resolution_windowed_stream,
_native.WindowedStreamSampler, sr3_wstream_*): every request's windows take slots of one engine and run at the request's own timestep
(DESIGN.md 3.10).

What is pinned, bit for bit (torch.equal): a request's image is super_resolution_windowed of that request alone on the same engine,
whatever its neighbours, whichever slots it got and whenever it was admitted; a window-sized request is super_resolution; a stream leaves
the engine as it found it; bad calls are refused with a message and change no slot."""
import pytest
import torch

import _sizes_inputs as si
from sr3_b200 import _native

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED12 = {"schedule": "linear", "n_timestep": 12, "linear_start": 1e-6, "linear_end": 1e-2}
CONFIGS = {"tiny": (si.TINY, 32), "sr16_64": (si.SR16_64, 64)}     # sr16_64 at 64x64 windows: lowest UNet level 4x4
TINY_SIZES = [(32, 32), (40, 56), (32, 72), (56, 48)]                # 1, 4, 3 and 4 windows of 32x32 at overlap 8


def build(monkeypatch, config, precision="bf16", slots=8, sched=SCHED12):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    unet, image_size = CONFIGS[config]
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet, precision=precision),
                     "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    # the windowed sampler of the references runs on the stream's engine: batch = slots, whatever the window count
    monkeypatch.setattr(net, "WINDOW_PASS_SIZES", (slots,))
    return net


def draws(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for H, W in sizes:
        out.append(((torch.rand(3, H, W, generator=g) * 2 - 1).cuda(), torch.randn(3, H, W, generator=g).cuda()))
    return out


def alone(net, cond, x_T, seed, sample_index):
    """The request's image from super_resolution_windowed of it alone (image 0 of a one-image canvas, keyed by sample_index)."""
    return net.super_resolution_windowed(cond[None], x_T=x_T[None], seed=seed, first_index=sample_index)


def check_stream(net, reqs, slots, seed, first):
    out = dict(net.super_resolution_windowed_stream([(n, c, x) for n, (c, x) in enumerate(reqs)], slots=slots, seed=seed, first_index=first))
    assert sorted(out) == list(range(len(reqs)))
    for n, (c, x) in enumerate(reqs):
        ref = alone(net, c, x, seed, first + n)
        assert torch.isfinite(ref).all()
        assert out[n].shape == x.shape
        assert torch.equal(out[n], ref), n
    return out


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("slots", [16, 8])
def test_mixed_sizes_equal_each_request_alone(monkeypatch, precision, slots):
    """12 windows of four sizes: all admitted together in 16 slots; in 8 the 56x48 canvas waits for the first ones to finish."""
    net = build(monkeypatch, "tiny", precision, slots)
    check_stream(net, draws(TINY_SIZES, 1), slots, 2 ** 40 + 7, 5)


def alone_at(net, cond, x_T, seed, sample_index, slot):
    """super_resolution_windowed of a one-window request alone with its window in `slot`: behind `slot` copies of itself (a canvas batch
    puts image b's windows after those of images 0 .. b - 1), returned as the batch's last image, keyed by sample_index."""
    c, x = cond[None].repeat(slot + 1, 1, 1, 1), x_T[None].repeat(slot + 1, 1, 1, 1)
    return net.super_resolution_windowed(c, x_T=x, seed=seed, first_index=sample_index - slot)


@pytest.mark.timeout(900)
def test_sr16_64_canvases_that_are_not_powers_of_two(monkeypatch):
    """64x64 windows of the 4x4-lowest-level config: 100x90 (2 x 2 windows, slots 0-3), 64x64 (one window, slot 4) and 70x120 (2 x 3,
    waits for free slots, then slots 0-5).  On this config a window's result depends on the slot it runs in, so each request is compared
    with the windowed sampler running its windows in the same slots; the 64x64 request against its result in slot 0 is reported."""
    net = build(monkeypatch, "sr16_64", slots=8)
    reqs = draws([(100, 90), (64, 64), (70, 120)], 2)
    seed, first = 31, 0
    plan = list(_native.windowed_stream_plan([(0, 4), (0, 1), (0, 6)], 8, SCHED12["n_timestep"]))
    assert [sl for sl, _, _ in plan] == [[0, 1, 2, 3], [4], [0, 1, 2, 3, 4, 5]]
    out = dict(net.super_resolution_windowed_stream([(n, c, x) for n, (c, x) in enumerate(reqs)], slots=8, seed=seed, first_index=first))
    assert torch.equal(out[0], alone(net, *reqs[0], seed, first))
    assert torch.equal(out[2], alone(net, *reqs[2], seed, first + 2))
    assert torch.equal(out[1], alone_at(net, *reqs[1], seed, first + 1, 4))
    at0 = alone(net, *reqs[1], seed, first + 1)
    rel = ((out[1] - at0).norm() / at0.norm()).item()
    print("sr16_64: one window in slot 4 against slot 0: max |diff| %.3e, relative L2 %.3e, %s" %
          ((out[1] - at0).abs().max().item(), rel, "bit-identical" if torch.equal(out[1], at0) else "not bit-identical"))
    assert rel < 1e-3


@pytest.mark.timeout(900)
def test_staggered_arrivals_through_the_online_interface(monkeypatch):
    """Requests arriving over the steps, driven through WindowedStreamSampler exactly as windowed_stream_plan says."""
    slots, T, seed, first = 8, SCHED12["n_timestep"], 99, 1000
    net = build(monkeypatch, "tiny", slots=slots)
    sizes = [(56, 48), (32, 32), (40, 56), (32, 32), (32, 72), (32, 32), (56, 48), (40, 56), (32, 72)]
    arrivals = [0, 0, 2, 3, 9, 15, 16, 16, 30]
    reqs = draws(sizes, 3)
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), seed, 8, 8)
    windows = [s.windows(H, W) for H, W in sizes]
    assert windows == [4, 1, 4, 1, 3, 1, 4, 4, 3]
    plan = list(_native.windowed_stream_plan(zip(arrivals, windows), slots, T))
    assert any(a > arr for (_, a, _), arr in zip(plan, arrivals)), "no request waited for slots"
    assert plan[3][1] > arrivals[3] and plan[3][1] >= plan[2][1], "the 1-window request did not wait behind the 4-window one"
    assert len({s_ for sl, _, _ in plan for s_ in sl}) == slots and sum(windows) > slots, "slots were not reused"
    ids, out = {}, {}
    for k in range(max(f for _, _, f in plan)):
        for n, (sl, a, _) in enumerate(plan):
            if a == k:
                ids[n] = s.admit(sl, reqs[n][0], reqs[n][1], first + n)
        s.step()
        done = [n for n, (_, _, f) in enumerate(plan) if f == k + 1]
        assert s.finished() == sorted(ids[n] for n in done)
        for n in done:
            out[n] = s.retire(ids[n])
    assert s.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)
    del s
    for n, (c, x) in enumerate(reqs):
        assert torch.equal(out[n], alone(net, c, x, seed, first + n)), n


@pytest.mark.timeout(900)
def test_a_window_sized_request_is_super_resolution(monkeypatch):
    slots, seed, first = 8, 17, 40
    net = build(monkeypatch, "tiny", slots=slots)
    reqs = draws([(40, 56), (32, 32), (32, 72)], 4)
    out = check_stream(net, reqs, slots, seed, first)
    # super_resolution on the same engine (batch = slots) returns its last image: put the request there, its sample index first + 1
    g = torch.Generator().manual_seed(5)
    cond = (torch.rand(slots, 3, 32, 32, generator=g) * 2 - 1).cuda()
    x_T = torch.randn(slots, 3, 32, 32, generator=g).cuda()
    cond[-1], x_T[-1] = reqs[1]
    assert torch.equal(out[1], net.super_resolution(cond, x_T=x_T, seed=seed, first_index=first + 1 - (slots - 1)))


@pytest.mark.timeout(900)
def test_a_stream_leaves_no_state_behind(monkeypatch):
    slots = 8
    net = build(monkeypatch, "tiny", slots=slots)
    eng = net._engine(slots, 32, 32)
    launches = eng.launches_per_step()
    g = torch.Generator().manual_seed(6)
    cond = (torch.rand(slots, 3, 32, 32, generator=g) * 2 - 1).cuda()
    x_T = torch.randn(slots, 3, 32, 32, generator=g).cuda()

    def lockstep():
        return eng.p_sample_loop(cond, x_T, None, 3, 0, want_snapshots=False)[0]

    before = lockstep()
    reqs = [(n, c, x) for n, (c, x) in enumerate(draws(TINY_SIZES + TINY_SIZES[::-1], 7))]
    first = list(net.super_resolution_windowed_stream(reqs, slots=slots, seed=8))
    assert eng.launches_per_step() == launches
    assert torch.equal(lockstep(), before)
    second = list(net.super_resolution_windowed_stream(reqs, slots=slots, seed=8))
    assert [k for k, _ in first] == [k for k, _ in second] and len(first) == len(reqs)
    for (_, a), (_, b) in zip(first, second):
        assert torch.equal(a, b)
    assert net._engine(slots, 32, 32) is eng


@pytest.mark.timeout(900)
def test_bad_calls_are_refused_and_change_no_slot(monkeypatch):
    slots = 8
    net = build(monkeypatch, "tiny", slots=slots)
    (c0, x0), (c1, x1) = draws([(40, 56), (32, 72)], 8)
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), 1, 8, 8)
    r = s.admit([2, 3, 5, 6], c0, x0, 0)
    s.step(3)
    state = s.slot_state()
    assert state == ([-1, -1, r, r, -1, r, r, -1], [-1, -1, 8, 8, -1, 8, 8, -1], [0, 0, 1, 1, 0, 1, 1, 0])
    with pytest.raises(RuntimeError, match="slot 3 is busy"):
        s.admit([0, 1, 3], c1, x1, 1)
    with pytest.raises(RuntimeError, match="has 3 windows .* given 2 slots"):
        s.admit([0, 1], c1, x1, 1)
    with pytest.raises(RuntimeError, match="has 3 windows .* given 4 slots"):
        s.admit([0, 1, 4, 7], c1, x1, 1)
    with pytest.raises(RuntimeError, match="slot 8 out of range"):
        s.admit([0, 1, 8], c1, x1, 1)
    with pytest.raises(RuntimeError, match="slot 1 listed twice"):
        s.admit([0, 1, 1], c1, x1, 1)
    with pytest.raises(RuntimeError, match="is still running"):
        s.retire(r)
    with pytest.raises(RuntimeError, match="request 5 is not held"):
        s.retire(5)
    with pytest.raises(ValueError, match="x_T has shape"):
        s.admit([0, 1, 4], c1, x1[:, :16], 1)
    assert s.slot_state() == state
    # a schedule change with a request in flight: the next step (and any admission) is refused, nothing moves
    net.set_new_noise_schedule(dict(SCHED12, n_timestep=10), "cuda")
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.step()
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.admit([0, 1, 4], c1, x1, 1)
    assert s.slot_state() == state
    # the generator refuses to go on once the schedule it planned with has changed
    net.set_new_noise_schedule(SCHED12, "cuda")
    del s
    gen = net.super_resolution_windowed_stream([(0, c0, x0), (1, c1, x1)], slots=4, seed=1)
    assert next(gen)[0] == 0
    net.set_new_noise_schedule(dict(SCHED12, n_timestep=10), "cuda")
    with pytest.raises(RuntimeError, match="noise schedule changed during the stream"):
        next(gen)


@pytest.mark.timeout(900)
def test_a_step_without_a_schedule_or_with_a_wrong_condition_is_refused(monkeypatch):
    slots = 4
    net = build(monkeypatch, "tiny", slots=slots)
    cfg = dict(net.denoise_fn.arch, channels=3, conditional=True, precision="bf16")
    eng = _native.Engine(cfg, slots, torch.device("cuda"), height=32, width=32)     # never given a schedule
    s = _native.WindowedStreamSampler(eng, 1, 8, 8)
    (c, x), = draws([(32, 32)], 9)
    with pytest.raises(RuntimeError, match="no noise schedule"):
        s.step()
    with pytest.raises(RuntimeError, match="no noise schedule"):
        s.admit([0], c, x, 0)
    assert s.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)
    # an unconditional model streams too, and its requests carry no condition; a conditional model's requests must
    unc = _native.WindowedStreamSampler(_native.Engine(dict(cfg, in_channel=3, conditional=False), slots, torch.device("cuda"),
                                                       height=32, width=32), 1, 8, 8)
    with pytest.raises(ValueError, match=r"condition_x must be \[0, H, W\]"):
        unc.admit([0], c, x, 0)
    assert unc.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)
    del s
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), 1, 8, 8)
    with pytest.raises(RuntimeError, match="condition_x is required by a conditional model"):
        s.admit([0], None, x, 0)
    assert s.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)

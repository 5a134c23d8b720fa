"""Continuous batching on the device (GaussianDiffusion.super_resolution_stream / sample_stream, and _native.WindowedStreamSampler with
one-window requests): every slot of the engine at its own timestep, refilled as its image finishes (DESIGN.md 3.10).

What is pinned, bit for bit (torch.equal): a request's image is the lockstep sampler's image for the same condition, x_T and sample index
at the slot stream_plan gave it, whatever the other slots hold and whenever it was admitted; a stream leaves the engine as it found it;
bad calls are refused with a message and change no slot."""
import pytest
import torch

import _sizes_inputs as si
from sr3_b200 import _native

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED12 = {"schedule": "linear", "n_timestep": 12, "linear_start": 1e-6, "linear_end": 1e-2}
CONFIGS = {"tiny": (si.TINY, 32), "sr16_64": (si.SR16_64, 64)}     # sr16_64 at 64x64: lowest UNet level 4x4
B = 4


def build(monkeypatch, config, precision="bf16", conditional=True, seed=0, sched=SCHED12):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    unet, image_size = CONFIGS[config]
    unet = dict(unet, precision=precision, in_channel=6 if conditional else 3)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": unet,
                     "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}
    torch.manual_seed(seed)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


def draws(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, H, W, generator=g) * 2 - 1).cuda(), torch.randn(n, 3, H, W, generator=g).cuda()


def lockstep(net, cond, x_T, seed, first_index):
    """All B images of the lockstep sampler (sr3_p_sample_loop) on the stream's engine."""
    final, _ = net._engine(x_T.shape[0], x_T.shape[2], x_T.shape[3]).p_sample_loop(cond, x_T, None, seed, first_index, want_snapshots=False)
    return final


def lockstep_at(net, cond, x_T, n, slot, sample_index, seed):
    """Request n's image from a lockstep batch that holds it at `slot` with `sample_index` and other requests' images around it."""
    idx = [(n + 1 + j) % cond.shape[0] for j in range(B)]
    idx[slot] = n
    out = lockstep(net, cond[idx], x_T[idx], seed, sample_index - slot)
    return out[slot]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("config,H,W", [("tiny", 32, 32), ("tiny", 32, 64), ("sr16_64", 64, 64)])
def test_all_slots_admitted_together_are_the_lockstep_sampler(monkeypatch, config, H, W, precision):
    net = build(monkeypatch, config, precision)
    cond, x_T = draws(B, H, W, 1)
    seed, first = 2 ** 40 + 7, 5
    ref = lockstep(net, cond, x_T, seed, first)
    out = dict(net.super_resolution_stream([(k, cond[k], x_T[k]) for k in range(B)], slots=B, seed=seed, first_index=first))
    assert sorted(out) == list(range(B))
    assert torch.isfinite(ref).all()
    for k in range(B):
        assert torch.equal(out[k], ref[k]), k
    # super_resolution returns the batch's last image (the reference's ret_img[-1])
    assert torch.equal(out[B - 1], net.super_resolution(cond, x_T=x_T, seed=seed, first_index=first))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_unconditional_sample_stream_is_the_lockstep_sampler(monkeypatch, precision):
    net = build(monkeypatch, "tiny", precision, conditional=False)
    seed = 11
    torch.manual_seed(123)
    out = list(net.sample_stream(B, slots=B, seed=seed))
    torch.manual_seed(123)
    x_T = torch.stack([torch.randn(3, 32, 32, device="cuda") for _ in range(B)])    # the stream draws x_T per request, in order
    ref = lockstep(net, None, x_T, seed, 0)
    assert [k for k, _ in out] == list(range(B))
    for k, img in out:
        assert torch.equal(img, ref[k]), k


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,H,W", [("tiny", 32, 32), ("sr16_64", 64, 64)])
def test_staggered_one_window_requests_are_independent_of_the_neighbours(monkeypatch, config, H, W):
    """11 requests through 4 slots, arriving over the steps; driven through the online interface exactly as stream_plan says."""
    net = build(monkeypatch, config)
    T, N, seed, first = SCHED12["n_timestep"], 11, 99, 1000
    cond, x_T = draws(N, H, W, 2)
    arrivals = [0, 0, 3, 5, 5, 9, 14, 15, 22, 30, 31]
    plan = list(_native.stream_plan(arrivals, B, T))
    assert len({a for _, a, _ in plan}) > 3 and len({s for s, _, _ in plan}) == B     # admitted at many steps, into every slot
    s = _native.WindowedStreamSampler(net._engine(B, H, W), seed, 0, 0)
    ids, out = {}, {}
    for k in range(max(f for _, _, f in plan)):
        for n, (slot, a, _) in enumerate(plan):
            if a == k:
                ids[n] = s.admit([slot], cond[n], x_T[n], first + n)
        s.step()
        done = [n for n, (_, _, f) in enumerate(plan) if f == k + 1]
        assert sorted(i for i, v in enumerate(s.slot_state()[2]) if v == 2) == sorted(plan[n][0] for n in done)
        assert s.finished() == sorted(ids[n] for n in done)
        for n in done:
            out[n] = s.retire(ids[n])
    assert s.slot_state() == ([-1] * B, [-1] * B, [0] * B)
    for n, (slot, _, _) in enumerate(plan):
        assert torch.equal(out[n], lockstep_at(net, cond, x_T, n, slot, first + n, seed)), n


@pytest.mark.timeout(900)
def test_generator_refills_slots_and_idle_slots_do_not_matter(monkeypatch):
    """One request through 4 slots (three idle), and 6 requests through 4 slots via the generator (two admitted when the first wave ends)."""
    net = build(monkeypatch, "tiny")
    cond, x_T = draws(6, 32, 32, 3)
    seed, first = 5, 40
    one = list(net.super_resolution_stream([("a", cond[0], x_T[0])], slots=B, seed=seed, first_index=first))
    assert [k for k, _ in one] == ["a"]
    assert torch.equal(one[0][1], lockstep_at(net, cond, x_T, 0, 0, first, seed))
    six = list(net.super_resolution_stream(((n, cond[n], x_T[n]) for n in range(6)), slots=B, seed=seed, first_index=first))
    assert [k for k, _ in six] == list(range(6))
    plan = list(_native.stream_plan([0] * 6, B, SCHED12["n_timestep"]))
    assert [p[:2] for p in plan[4:]] == [(0, 12), (1, 12)]
    for n, img in six:
        assert torch.equal(img, lockstep_at(net, cond, x_T, n, plan[n][0], first + n, seed)), n


@pytest.mark.timeout(900)
def test_a_stream_leaves_no_state_behind(monkeypatch):
    net = build(monkeypatch, "sr16_64")
    cond, x_T = draws(B, 64, 64, 4)
    eng = net._engine(B, 64, 64)
    launches = eng.launches_per_step()
    before = lockstep(net, cond, x_T, 3, 0)
    reqs = [(n, cond[(n + 1) % B], x_T[(n + 2) % B]) for n in range(6)]
    first = list(net.super_resolution_stream(reqs, slots=B, seed=8))
    assert eng.launches_per_step() == launches
    assert torch.equal(lockstep(net, cond, x_T, 3, 0), before)
    second = list(net.super_resolution_stream(reqs, slots=B, seed=8))
    assert [k for k, _ in first] == [k for k, _ in second]
    for (_, a), (_, b) in zip(first, second):
        assert torch.equal(a, b)
    assert net._engine(B, 64, 64) is eng


@pytest.mark.timeout(900)
def test_bad_one_window_calls_are_refused_and_change_no_slot(monkeypatch):
    net = build(monkeypatch, "tiny")
    cond, x_T = draws(B, 32, 32, 5)
    s = _native.WindowedStreamSampler(net._engine(B, 32, 32), 1, 0, 0)
    r = s.admit([1], cond[0], x_T[0], 0)
    s.step(3)
    state = s.slot_state()
    assert state == ([-1, r, -1, -1], [-1, 8, -1, -1], [0, 1, 0, 0])
    with pytest.raises(RuntimeError, match="slot 4 out of range"):
        s.admit([4], cond[1], x_T[1], 1)
    with pytest.raises(RuntimeError, match="slot -1 out of range"):
        s.admit([-1], cond[1], x_T[1], 1)
    with pytest.raises(RuntimeError, match="slot 1 is busy"):
        s.admit([1], cond[1], x_T[1], 1)
    with pytest.raises(RuntimeError, match="request %d is still running" % r):
        s.retire(r)
    with pytest.raises(RuntimeError, match="request %d is not held" % (r + 1)):
        s.retire(r + 1)
    with pytest.raises(RuntimeError, match="condition_x is required by a conditional model"):
        s.admit([0], None, x_T[1], 1)
    with pytest.raises(ValueError, match="x_T has shape"):
        s.admit([0], cond[1, :, :16], x_T[1], 1)
    assert s.slot_state() == state
    # a schedule change with a request in flight: the next step (and any admit) is refused, nothing moves
    net.set_new_noise_schedule(dict(SCHED12, n_timestep=10), "cuda")
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.step()
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.admit([0], cond[1], x_T[1], 1)
    assert s.slot_state() == state
    # the generator refuses to go on once the schedule it planned with has changed
    net.set_new_noise_schedule(SCHED12, "cuda")
    del s
    gen = net.super_resolution_stream([(n, cond[n], x_T[n]) for n in range(2)], slots=1, seed=1)
    assert next(gen)[0] == 0
    net.set_new_noise_schedule(dict(SCHED12, n_timestep=10), "cuda")
    with pytest.raises(RuntimeError, match="noise schedule changed during the stream"):
        next(gen)


@pytest.mark.timeout(900)
def test_a_one_window_stream_without_a_schedule_is_refused(monkeypatch):
    net = build(monkeypatch, "tiny")
    cfg = dict(net.denoise_fn.arch, channels=3, conditional=True, precision="bf16")
    eng = _native.Engine(cfg, B, torch.device("cuda"), height=32, width=32)     # never given a schedule
    s = _native.WindowedStreamSampler(eng, 1, 0, 0)
    cond, x_T = draws(1, 32, 32, 6)
    with pytest.raises(RuntimeError, match="no noise schedule"):
        s.step()
    with pytest.raises(RuntimeError, match="no noise schedule"):
        s.admit([0], cond[0], x_T[0], 0)
    assert s.slot_state() == ([-1] * B, [-1] * B, [0] * B)

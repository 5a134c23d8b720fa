"""Per-request noise schedules in continuous batching on the device (GaussianDiffusion.super_resolution_windowed_stream and
super_resolution_stream with (key, x_in, x_T, schedule) requests; _native.WindowedStreamSampler.add_schedule / admit(schedule=...);
sr3_wstream_add_schedule / sr3_wstream_admit_scheduled): every request samples on its own schedule, requests on different schedules
share the batch (DESIGN.md 3.10).

What is pinned, bit for bit (torch.equal): a request on schedule S is super_resolution_windowed of that request alone after
set_new_noise_schedule(S) on the same engine with its windows in the same slots; a request that names the module's schedule is the same
request without one; it is admitted at t = n_timestep(S) - 1 and finishes exactly n_timestep(S) steps later; a change of the module's
schedule touches no request on a schedule of its own; bad calls are refused with a message and change no slot."""
import ctypes

import pytest
import torch

import _sizes_inputs as si
from sr3_b200 import _native
from sr3_b200.model.sr3_modules import diffusion

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SCHED12 = {"schedule": "linear", "n_timestep": 12, "linear_start": 1e-6, "linear_end": 1e-2}
LIN5 = {"schedule": "linear", "n_timestep": 5, "linear_start": 1e-4, "linear_end": 2e-2}
COS9 = {"schedule": "cosine", "n_timestep": 9, "linear_start": 1e-6, "linear_end": 1e-2}
QUAD16 = {"schedule": "quad", "n_timestep": 16, "linear_start": 1e-6, "linear_end": 1e-2}
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


def alone(net, cond, x_T, seed, sample_index, sched=None, slot=0):
    """The request's image from super_resolution_windowed of it alone after set_new_noise_schedule(sched) (None: the module's SCHED12),
    keyed by sample_index.  slot > 0, for a one-window request: its window in `slot`, behind `slot` copies of itself (a canvas batch puts
    image b's windows after those of images 0 .. b - 1), returned as the batch's last image."""
    net.set_new_noise_schedule(sched or SCHED12, "cuda")
    try:
        c, x = cond[None].repeat(slot + 1, 1, 1, 1), x_T[None].repeat(slot + 1, 1, 1, 1)
        return net.super_resolution_windowed(c, x_T=x, seed=seed, first_index=sample_index - slot)
    finally:
        net.set_new_noise_schedule(SCHED12, "cuda")


def stream(net, reqs, scheds, slots, seed, first):
    """super_resolution_windowed_stream of reqs (cond, x_T) on scheds (None: name no schedule), as a dict key -> image."""
    rq = [(n, c, x) if s is None else (n, c, x, s) for n, ((c, x), s) in enumerate(zip(reqs, scheds))]
    out = dict(net.super_resolution_windowed_stream(rq, slots=slots, seed=seed, first_index=first))
    assert sorted(out) == list(range(len(reqs)))
    return out


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_mixed_schedules_and_sizes_equal_each_request_alone_tiny(monkeypatch, precision):
    """Eight canvases of four sizes on four schedules (shorter and longer than the module's 12 steps, and the module's), 8 slots: the
    later requests wait for slots, and short ones free theirs first."""
    net = build(monkeypatch, "tiny", precision, 8)
    reqs = draws(TINY_SIZES + TINY_SIZES[::-1], 11)
    scheds = [LIN5, None, COS9, QUAD16, COS9, LIN5, None, QUAD16]
    seed, first = 2 ** 40 + 3, 7
    out = stream(net, reqs, scheds, 8, seed, first)
    for n, ((c, x), s) in enumerate(zip(reqs, scheds)):
        ref = alone(net, c, x, seed, first + n, s)
        assert torch.isfinite(ref).all()
        assert torch.equal(out[n], ref), (n, s)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_mixed_schedules_and_sizes_equal_each_request_alone_sr16_64(monkeypatch, precision):
    """64x64 windows of the 4x4-lowest-level config, where the slot a window runs in matters: 100x90 on quad 16 (slots 0-3), 64x64 on
    linear 5 (slot 4, so compared in slot 4) and 70x120 on cosine 9, which waits until slots 0-5 are all free."""
    net = build(monkeypatch, "sr16_64", precision, 8)
    reqs = draws([(100, 90), (64, 64), (70, 120)], 12)
    scheds = [QUAD16, LIN5, COS9]
    plan = list(_native.windowed_stream_plan([(0, 4, 16), (0, 1, 5), (0, 6, 9)], 8, 12))
    assert plan == [([0, 1, 2, 3], 0, 16), ([4], 0, 5), ([0, 1, 2, 3, 4, 5], 16, 25)]
    seed, first = 31, 0
    out = stream(net, reqs, scheds, 8, seed, first)
    assert torch.equal(out[0], alone(net, *reqs[0], seed, first, QUAD16))
    assert torch.equal(out[1], alone(net, *reqs[1], seed, first + 1, LIN5, slot=4))
    assert torch.equal(out[2], alone(net, *reqs[2], seed, first + 2, COS9))


@pytest.mark.timeout(900)
def test_naming_the_modules_schedule_is_naming_none(monkeypatch):
    net = build(monkeypatch, "tiny", slots=8)
    reqs = draws(TINY_SIZES, 13)
    plain = stream(net, reqs, [None] * 4, 8, 5, 3)
    named = stream(net, reqs, [SCHED12] * 4, 8, 5, 3)
    mixed = stream(net, reqs, [SCHED12, None, dict(SCHED12), None], 8, 5, 3)
    for n in range(4):
        assert torch.equal(named[n], plain[n]) and torch.equal(mixed[n], plain[n]), n


@pytest.mark.timeout(900)
def test_online_interface_schedules_added_while_requests_run(monkeypatch):
    """A request on the module's schedule runs 3 steps; then cosine 9 and quad 16 are registered and requests on them admitted: slot_state
    shows t = T_S - 1 at admission and each finishes after exactly T_S steps."""
    slots, seed, first = 8, 41, 100
    net = build(monkeypatch, "tiny", slots=slots)
    reqs = draws([(40, 56), (32, 32), (32, 72)], 14)
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), seed, 8, 8)
    r0 = s.admit([0, 1, 2, 3], *reqs[0], first)
    s.step(3)
    ids = {}
    for n, (sched, sl) in enumerate(((COS9, [4]), (QUAD16, [5, 6, 7])), start=1):
        sid = s.add_schedule(*diffusion.noise_schedule_buffers(sched))
        assert sid == n - 1
        ids[n] = s.admit(sl, *reqs[n], first + n, schedule=sid)
        req, t, st = s.slot_state()
        assert [t[k] for k in sl] == [sched["n_timestep"] - 1] * len(sl) and [st[k] for k in sl] == [1] * len(sl)
    assert s.slot_state()[1][0] == 12 - 1 - 3
    out, finish = {}, {0: 12, 1: 3 + 9, 2: 3 + 16}
    ids[0] = r0
    for k in range(3, 3 + 16):
        s.step()
        done = sorted(ids[n] for n, f in finish.items() if f == k + 1)
        assert s.finished() == done, k
        for n, f in finish.items():
            if f == k + 1:
                out[n] = s.retire(ids[n])
    assert s.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)
    del s
    assert torch.equal(out[0], alone(net, *reqs[0], seed, first))
    assert torch.equal(out[1], alone(net, *reqs[1], seed, first + 1, COS9))
    assert torch.equal(out[2], alone(net, *reqs[2], seed, first + 2, QUAD16))


@pytest.mark.timeout(900)
def test_module_schedule_changed_mid_stream(monkeypatch):
    """Requests on schedules of their own finish correctly across a change of the module's schedule; a request on the module's schedule
    in flight across a change still makes the next step raise."""
    slots, seed, first = 8, 43, 20
    net = build(monkeypatch, "tiny", slots=slots)
    reqs = draws([(40, 56), (32, 72), (32, 32)], 15)
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), seed, 8, 8)
    lin5 = s.add_schedule(*diffusion.noise_schedule_buffers(LIN5))
    cos9 = s.add_schedule(*diffusion.noise_schedule_buffers(COS9))
    a = s.admit([0, 1, 2, 3], *reqs[0], first, schedule=lin5)
    b = s.admit([4, 5, 6], *reqs[1], first + 1, schedule=cos9)
    s.step(2)
    net.set_new_noise_schedule(dict(SCHED12, n_timestep=10), "cuda")
    s.step(3)
    assert s.finished() == [a]
    out_a = s.retire(a)
    s.step(4)
    assert s.finished() == [b]
    out_b = s.retire(b)
    # a request on the module's (new) schedule, then another change while it is in flight
    c = s.admit([7], *reqs[2], first + 2)
    assert s.slot_state()[1][7] == 9
    s.step()
    state = s.slot_state()
    net.set_new_noise_schedule(SCHED12, "cuda")
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.step()
    with pytest.raises(RuntimeError, match="noise schedule changed while requests are in flight"):
        s.admit([0], *reqs[2], first + 3, schedule=lin5)
    assert s.slot_state() == state
    assert c in state[0]
    del s
    assert torch.equal(out_a, alone(net, *reqs[0], seed, first, LIN5))
    assert torch.equal(out_b, alone(net, *reqs[1], seed, first + 1, COS9))


@pytest.mark.timeout(900)
def test_bad_schedule_calls_are_refused_and_change_no_slot(monkeypatch):
    slots = 8
    net = build(monkeypatch, "tiny", slots=slots)
    (c0, x0), (c1, x1) = draws([(40, 56), (32, 72)], 16)
    s = _native.WindowedStreamSampler(net._engine(slots, 32, 32), 1, 8, 8)
    sid = s.add_schedule(*diffusion.noise_schedule_buffers(LIN5))
    r = s.admit([2, 3, 5, 6], c0, x0, 0, schedule=sid)
    s.step(2)
    state = s.slot_state()
    assert state == ([-1, -1, r, r, -1, r, r, -1], [-1, -1, 2, 2, -1, 2, 2, -1], [0, 0, 1, 1, 0, 1, 1, 0])
    with pytest.raises(RuntimeError, match=r"unknown schedule 1 \(1 registered\)"):
        s.admit([0, 1, 4], c1, x1, 1, schedule=1)
    with pytest.raises(RuntimeError, match="unknown schedule -2"):
        s.admit([0, 1, 4], c1, x1, 1, schedule=-2)
    # straight to the C ABI: T out of range and a null table
    T, host, sp = _native._schedule_host(*diffusion.noise_schedule_buffers(LIN5))
    ptrs = [ctypes.c_void_p(h.data_ptr()) for h in host] + [ctypes.c_void_p(sp.ctypes.data)]
    out = ctypes.c_int(-7)
    for bad_T, bad_ptrs, match in ((0, ptrs, "n_timestep 0 out of range"), (4097, ptrs, "n_timestep 4097 out of range"),
                                   (T, ptrs[:2] + [ctypes.c_void_p()] + ptrs[3:], "null schedule table")):
        with torch.cuda.device(0):
            assert _native.lib().sr3_wstream_add_schedule(s._h, bad_T, *bad_ptrs, ctypes.byref(out), None) != 0
        assert match in _native.lib().sr3_last_error().decode() and out.value == -7
    assert s.slot_state() == state
    # nothing was registered by the refused calls: the next schedule is id 1
    assert s.add_schedule(*diffusion.noise_schedule_buffers(COS9)) == 1
    s.step(3)
    assert s.finished() == [r]
    s.retire(r)
    assert s.slot_state() == ([-1] * slots, [-1] * slots, [0] * slots)


@pytest.mark.timeout(900)
def test_a_mixed_schedule_stream_repeats_bit_for_bit(monkeypatch):
    net = build(monkeypatch, "tiny", slots=8)
    reqs = draws(TINY_SIZES + TINY_SIZES[::-1], 17)
    scheds = [QUAD16, COS9, None, LIN5, LIN5, None, COS9, QUAD16]
    a = stream(net, reqs, scheds, 8, 9, 0)
    b = stream(net, reqs, scheds, 8, 9, 0)
    for n in range(len(reqs)):
        assert torch.equal(a[n], b[n]), n


@pytest.mark.timeout(900)
def test_single_size_stream_with_mixed_schedules(monkeypatch):
    """super_resolution_stream: one-window 32x32 requests on four schedules, 4 slots."""
    net = build(monkeypatch, "tiny", slots=4)
    reqs = draws([(32, 32)] * 6, 18)
    scheds = [COS9, None, LIN5, QUAD16, None, LIN5]
    rq = [(n, c, x) if s is None else (n, c, x, s) for n, ((c, x), s) in enumerate(zip(reqs, scheds))]
    seed, first = 77, 50
    out = dict(net.super_resolution_stream(rq, slots=4, seed=seed, first_index=first))
    # the slots windowed_stream_plan gives each request: compare it in that slot (a one-window request on this config is slot-independent,
    # but the reference is taken where it ran)
    plan = list(_native.windowed_stream_plan([(0, 1, (s or SCHED12)["n_timestep"]) for s in scheds], 4, 12))
    for n, ((c, x), s) in enumerate(zip(reqs, scheds)):
        assert torch.equal(out[n], alone(net, c, x, seed, first + n, s, slot=plan[n][0][0])), (n, s)

"""Per-request noise schedules in continuous batching, without a GPU: the slot plan when requests run different numbers of steps
(_native.windowed_stream_plan with (arrival, windows, steps)), against hand cases and a step-by-step simulator; the schedule buffers the
streams build (diffusion.noise_schedule_buffers) against set_new_noise_schedule's; and the refusal of a malformed schedule, which comes
before anything native is touched."""
import numpy as np
import pytest
import torch

import sr3_b200
from sr3_b200 import _native
from sr3_b200.model.sr3_modules import diffusion

SCHED = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)


def simulate(requests, slots):
    """The plan by brute force: at every step, admit the earliest arrived request while its windows fit in the free slots (the lowest
    ones); a request of `steps` steps holds its slots for that many steps."""
    busy_until = [0] * slots
    out, queue, k, i = [], [], 0, 0
    while len(out) < len(requests):
        while i < len(requests) and requests[i][0] <= k:
            queue.append(i)
            i += 1
        while queue:
            _, n, steps = requests[queue[0]]
            free = [s for s in range(slots) if busy_until[s] <= k]
            if len(free) < n:
                break
            for s in free[:n]:
                busy_until[s] = k + steps
            out.append((free[:n], k, k + steps))
            queue.pop(0)
        k += 1
    return out


def traffic(seed, trials):
    rng = np.random.default_rng(seed)
    for _ in range(trials):
        slots = int(rng.integers(1, 17))
        n = int(rng.integers(1, 40))
        tiers = rng.integers(1, 40, size=int(rng.integers(1, 4)))
        steps = rng.choice(tiers, size=n)
        wins = rng.integers(1, slots + 1, size=n)
        gaps = rng.poisson(rng.uniform(0.05, 2.0) * steps.mean() * wins.mean() / slots, size=n)
        yield slots, list(zip(np.cumsum(gaps).tolist(), wins.tolist(), steps.tolist()))


def test_a_short_request_frees_its_slots_first():
    # 4 slots.  A 2-step and a 10-step request start together; the 2-window request arriving at step 1 takes the short request's slots at
    # step 2, long before the long request finishes.
    plan = list(_native.windowed_stream_plan([(0, 2, 2), (0, 2, 10), (1, 2, 5)], 4, 7))
    assert plan == [([0, 1], 0, 2), ([2, 3], 0, 10), ([0, 1], 2, 7)]


def test_a_blocked_large_request_still_stops_a_later_small_one():
    # 4 slots.  The 4-window request waits for the 20-step request to finish; the 1-step, 1-window request behind it waits too although
    # slots 2 and 3 are free from step 3 on.
    plan = list(_native.windowed_stream_plan([(0, 2, 20), (0, 2, 3), (1, 4, 5), (1, 1, 1)], 4, 7))
    assert plan == [([0, 1], 0, 20), ([2, 3], 0, 3), ([0, 1, 2, 3], 20, 25), ([0], 25, 26)]


def test_the_plan_is_the_step_by_step_simulation():
    for slots, reqs in traffic(3, 300):
        assert list(_native.windowed_stream_plan(reqs, slots, 7)) == simulate(reqs, slots), (slots, reqs)


def test_steps_equal_to_T_is_todays_plan():
    for slots, reqs in traffic(4, 200):
        T = reqs[0][2]
        old = [(a, n) for a, n, _ in reqs]
        assert list(_native.windowed_stream_plan([(a, n, T) for a, n in old], slots, T)) == list(_native.windowed_stream_plan(old, slots, T))
    # a request without steps runs T of them, next to requests with their own
    mixed = list(_native.windowed_stream_plan([(0, 1), (0, 2, 4), (3, 1)], 2, 6))
    assert mixed == list(_native.windowed_stream_plan([(0, 1, 6), (0, 2, 4), (3, 1, 6)], 2, 6))
    assert mixed == [([0], 0, 6), ([0, 1], 6, 10), ([0], 10, 16)]


def test_the_plan_refuses_a_request_of_no_steps():
    with pytest.raises(ValueError, match="a request of 0 steps"):
        list(_native.windowed_stream_plan([(0, 1, 0)], 2, 5))


@pytest.mark.parametrize("name", diffusion.SCHEDULE_NAMES)
def test_schedule_buffers_are_set_new_noise_schedules(name):
    opt = {"schedule": name, "n_timestep": 37, "linear_start": 1e-5, "linear_end": 2e-2}
    net = make_net()
    net.set_new_noise_schedule(opt, "cpu")
    bufs, sp = diffusion.noise_schedule_buffers(opt)
    assert sorted(bufs) == sorted(diffusion._BUFFERS)
    for k, v in bufs.items():
        ref = getattr(net, k)
        assert v.dtype == ref.dtype == torch.float32 and torch.equal(v, ref), k
    assert sp.dtype == np.float64 and np.array_equal(sp, net.sqrt_alphas_cumprod_prev)
    # the host arrays both native calls receive
    T, host, spn = _native._schedule_host(bufs, sp)
    assert T == 37 and spn.shape == (38,) and all(h.dtype == torch.float32 and h.shape == (37,) for h in host)


def make_net(conditional=True):
    opt = {"phase": "val", "gpu_ids": None, "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(TINY, in_channel=6 if conditional else 3),
                     "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": 32, "channels": 3, "conditional": conditional}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt)
    net.set_new_noise_schedule(SCHED, "cpu")
    return net


def no_native(*args, **kwargs):
    raise AssertionError("the native side was reached before the requests were checked")


X = torch.zeros(3, 32, 32)


@pytest.mark.parametrize("schedule,match", [
    ([("schedule", "linear")], r"request 'b': a schedule is a dict"),
    ({"schedule": "linear", "n_timestep": 5, "linear_start": 1e-6}, r"request 'b': the schedule has no 'linear_end'"),
    ({"n_timestep": 5}, r"request 'b': the schedule has no 'schedule', 'linear_start', 'linear_end'"),
    (dict(SCHED, schedule="sigmoid"), r"request 'b': unknown schedule 'sigmoid'"),
    (dict(SCHED, n_timestep=0), r"request 'b': n_timestep 0 out of range \[1, 4096\]"),
    (dict(SCHED, n_timestep=4097), r"request 'b': n_timestep 4097 out of range \[1, 4096\]"),
    (dict(SCHED, n_timestep=5.0), r"request 'b': n_timestep 5.0 out of range"),
    (dict(SCHED, n_timestep=True), r"request 'b': n_timestep True out of range"),
])
@pytest.mark.parametrize("stream", ["windowed", "single_size"])
def test_a_malformed_schedule_is_refused_before_anything_native(monkeypatch, schedule, match, stream):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_native)
    monkeypatch.setattr(_native, "WindowedStreamSampler", no_native)
    requests = [("a", X, None, dict(SCHED, n_timestep=5)), ("b", X, None, schedule)]
    run = net.super_resolution_windowed_stream if stream == "windowed" else net.super_resolution_stream
    with pytest.raises(ValueError, match=match):
        list(run(requests, slots=4))


def test_the_request_forms_are_named_in_the_refusal(monkeypatch):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_native)
    for bad in [(0,), (0, X, None, SCHED, 1)]:
        with pytest.raises(ValueError, match=r"a request is \(key, x_in\).*\(key, x_in, x_T or None, schedule\)"):
            list(net.super_resolution_windowed_stream([bad], slots=4))
    # a 4-tuple is checked like a 3-tuple otherwise
    with pytest.raises(ValueError, match=r"request 'a': x_T must be \(3, 32, 32\)"):
        list(net.super_resolution_windowed_stream([("a", X, torch.zeros(3, 32, 16), SCHED)], slots=4))

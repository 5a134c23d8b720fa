"""Continuous batching without a GPU: the slot plan (_native.stream_plan) over random arrival sequences, and the argument checks of
GaussianDiffusion.super_resolution_stream / sample_stream, which refuse a bad request before anything is admitted."""
import numpy as np
import pytest
import torch

import sr3_b200
from sr3_b200 import _native

SCHED = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)


def arrival_sequences():
    rng = np.random.default_rng(0)
    for trial in range(300):
        slots = int(rng.integers(1, 9))
        T = int(rng.integers(1, 30))
        n = int(rng.integers(1, 40))
        gaps = rng.poisson(rng.uniform(0.05, 2.0) * T / slots, size=n)
        gaps[0] = rng.integers(0, 5)
        yield slots, T, np.cumsum(gaps).tolist()


def busy(plan, k):
    """Requests that occupy a slot during step k."""
    return [i for i, (_, a, f) in enumerate(plan) if a <= k < f]


@pytest.mark.parametrize("case", list(range(3)))
def test_stream_plan_properties(case):
    for j, (slots, T, arrivals) in enumerate(arrival_sequences()):
        if j % 3 != case:
            continue
        plan = list(_native.stream_plan(arrivals, slots, T))
        assert len(plan) == len(arrivals)
        admits = [a for _, a, _ in plan]
        assert admits == sorted(admits), "first come first served"
        last = max(f for _, _, f in plan)
        for n, ((slot, a, f), arr) in enumerate(zip(plan, arrivals)):
            assert 0 <= slot < slots
            assert a >= arr, "admitted before it arrived"
            assert f == a + T, "every request runs exactly T steps"
            # the lowest slot that is free at the admit step (earlier requests of the same step took theirs first)
            taken = {plan[m][0] for m in busy(plan, a) if m != n and (plan[m][1] < a or m < n)}
            assert slot not in taken
            assert all(s in taken for s in range(slot)), (n, slot, taken)
        for k in range(last + 1):
            occ = [plan[i][0] for i in busy(plan, k)]
            assert len(occ) == len(set(occ)), "two requests share a slot"
            waiting = [n for n, arr in enumerate(arrivals) if arr <= k < plan[n][1]]
            if waiting:
                assert len(occ) == slots, "a slot idles while request %d waits at step %d" % (waiting[0], k)


@pytest.mark.parametrize("slots,T,N", [(1, 1, 1), (4, 10, 4), (4, 10, 3), (16, 2000, 16), (16, 20, 1)])
def test_stream_plan_all_at_once_is_the_lockstep_schedule(slots, T, N):
    assert list(_native.stream_plan([0] * N, slots, T)) == [(i, 0, T) for i in range(N)]


def test_stream_plan_refuses_bad_arguments():
    with pytest.raises(ValueError, match="non-decreasing"):
        list(_native.stream_plan([0, 3, 2], 2, 5))
    with pytest.raises(ValueError, match="slots >= 1"):
        list(_native.stream_plan([0], 0, 5))
    with pytest.raises(ValueError, match="T >= 1"):
        list(_native.stream_plan([0], 2, 0))


def test_stream_plan_reads_arrivals_lazily():
    read = []

    def arrivals():
        for k in (0, 0, 7):
            read.append(k)
            yield k

    plan = _native.stream_plan(arrivals(), 2, 5)
    assert next(plan) == (0, 0, 5) and read == [0]
    assert next(plan) == (1, 0, 5) and read == [0, 0]
    assert next(plan) == (0, 7, 12) and read == [0, 0, 7]


def make_net(conditional=True, image_size=32):
    opt = {"phase": "val", "gpu_ids": None, "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(TINY, in_channel=6 if conditional else 3),
                     "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt)
    net.set_new_noise_schedule(SCHED, "cpu")
    return net


def no_engine(*args, **kwargs):
    raise AssertionError("an engine was requested before the requests were checked")


@pytest.mark.parametrize("requests,match", [
    ([(0, torch.zeros(3, 32, 32)), (1, torch.zeros(3, 64, 32))], "is 64x32; this stream runs 32x32"),
    ([(0, torch.zeros(3, 32, 32)), (1, torch.zeros(3, 32, 32)), (2, torch.zeros(3, 32, 64))], "is 32x64; this stream runs 32x32"),
    ([(0, torch.zeros(4, 32, 32))], r"x_in must be \[3, H, W\]"),
    ([(0, torch.zeros(3, 32, 32)), (1, torch.zeros(1, 3, 32, 32))], r"x_in must be \[3, H, W\]"),
    ([(0, torch.zeros(3, 32, 32), torch.zeros(3, 32, 16))], r"x_T must be \(3, 32, 32\)"),
    ([(0,)], r"a request is \(key, x_in\)"),
])
def test_stream_refuses_a_bad_request_before_anything_is_admitted(monkeypatch, requests, match):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_engine)
    with pytest.raises(ValueError, match=match):
        list(net.super_resolution_stream(requests, slots=4))


def test_stream_refuses_an_unsupported_size_and_the_wrong_model_kind(monkeypatch):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_engine)
    with pytest.raises(_native.UnsupportedSizeError):
        list(net.super_resolution_stream([(0, torch.zeros(3, 48, 48))], slots=2))
    with pytest.raises(ValueError, match="slots must be >= 1"):
        list(net.super_resolution_stream([(0, torch.zeros(3, 32, 32))], slots=0))
    with pytest.raises(ValueError, match="needs an unconditional model"):
        net.sample_stream(2)
    unc = make_net(conditional=False)
    with pytest.raises(ValueError, match="needs a conditional model"):
        unc.super_resolution_stream([])


def test_stream_without_a_gpu_fails_loudly():
    net = make_net()
    with pytest.raises((_native.NativeLibraryError, RuntimeError)):
        list(net.super_resolution_stream([(0, torch.zeros(3, 32, 32))], slots=2))


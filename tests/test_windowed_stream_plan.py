"""Continuous batching of canvases of any size without a GPU: the slot plan (_native.windowed_stream_plan) over random traffic, its
agreement with stream_plan when every request is one window, the request checks of GaussianDiffusion.super_resolution_windowed_stream
(which refuse a bad request before anything native is touched), and the ptxas report of the stream's kernels."""
import numpy as np
import pytest
import torch

import sr3_b200
from sr3_b200 import _native

SCHED = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)


def traffic():
    rng = np.random.default_rng(1)
    for trial in range(300):
        slots = int(rng.integers(1, 17))
        T = int(rng.integers(1, 30))
        n = int(rng.integers(1, 40))
        wins = rng.integers(1, slots + 1, size=n)
        if trial % 4 == 0:
            wins[:] = 1
        gaps = rng.poisson(rng.uniform(0.05, 2.0) * T * wins.mean() / slots, size=n)
        gaps[0] = rng.integers(0, 5)
        yield slots, T, list(zip(np.cumsum(gaps).tolist(), wins.tolist()))


def busy(plan, k):
    """Requests that hold slots during step k."""
    return [i for i, (_, a, f) in enumerate(plan) if a <= k < f]


@pytest.mark.parametrize("case", list(range(3)))
def test_windowed_stream_plan_properties(case):
    for j, (slots, T, reqs) in enumerate(traffic()):
        if j % 3 != case:
            continue
        plan = list(_native.windowed_stream_plan(reqs, slots, T))
        assert len(plan) == len(reqs)
        admits = [a for _, a, _ in plan]
        assert admits == sorted(admits), "first come first served: no request overtakes an earlier one"
        for n, ((sl, a, f), (arr, w)) in enumerate(zip(plan, reqs)):
            assert len(sl) == w and len(set(sl)) == w and all(0 <= s < slots for s in sl)
            assert a >= arr, "admitted before it arrived"
            assert f == a + T, "every request runs exactly T steps"
            # the lowest slots free at the admit step (earlier requests of the same step took theirs first)
            taken = {s for m in busy(plan, a) if m != n and (plan[m][1] < a or m < n) for s in plan[m][0]}
            assert not taken & set(sl), (n, sl, taken)
            free = [s for s in range(slots) if s not in taken]
            assert sl == free[:w], (n, sl, free)
            # admitted at the first step at which it has arrived, every earlier request is in and enough slots are free
            if a > max(arr, plan[n - 1][1] if n else 0):
                held = {s for m in busy(plan, a - 1) if m < n for s in plan[m][0]}
                assert slots - len(held) < w, "request %d could have started at step %d" % (n, a - 1)
        last = max(f for _, _, f in plan)
        for k in range(last + 1):
            occ = [s for i in busy(plan, k) for s in plan[i][0]]
            assert len(occ) == len(set(occ)), "two running requests share a slot at step %d" % k


def test_head_of_line_blocking_and_lowest_free_slots():
    # 4 slots, T = 5.  The 4-window request waits for every slot; the 1-window request behind it waits too although slot 3 is free from
    # step 1 on; the last 2-window request waits for two free slots although slot 3 is free from step 10 on.
    plan = list(_native.windowed_stream_plan([(0, 3), (1, 4), (1, 1), (2, 2), (2, 2)], 4, 5))
    assert plan == [([0, 1, 2], 0, 5), ([0, 1, 2, 3], 5, 10), ([0], 10, 15), ([1, 2], 10, 15), ([0, 1], 15, 20)]


def test_one_window_requests_are_stream_plan():
    rng = np.random.default_rng(2)
    for _ in range(200):
        slots, T, n = int(rng.integers(1, 9)), int(rng.integers(1, 30)), int(rng.integers(1, 40))
        arrivals = np.cumsum(rng.poisson(rng.uniform(0.05, 2.0) * T / slots, size=n)).tolist()
        want = list(_native.stream_plan(arrivals, slots, T))
        got = [(sl[0], a, f) for sl, a, f in _native.windowed_stream_plan([(a, 1) for a in arrivals], slots, T)]
        assert got == want


def test_windowed_stream_plan_refuses_bad_arguments():
    with pytest.raises(ValueError, match="non-decreasing"):
        list(_native.windowed_stream_plan([(0, 1), (3, 1), (2, 1)], 2, 5))
    with pytest.raises(ValueError, match="5 windows cannot run on 4 slots"):
        list(_native.windowed_stream_plan([(0, 1), (0, 5)], 4, 5))
    with pytest.raises(ValueError, match="0 windows"):
        list(_native.windowed_stream_plan([(0, 0)], 4, 5))
    with pytest.raises(ValueError, match="slots >= 1"):
        list(_native.windowed_stream_plan([(0, 1)], 0, 5))
    with pytest.raises(ValueError, match="T >= 1"):
        list(_native.windowed_stream_plan([(0, 1)], 2, 0))


def test_windowed_stream_plan_reads_requests_lazily():
    read = []

    def reqs():
        for r in ((0, 2), (0, 1), (0, 2)):
            read.append(r)
            yield r

    plan = _native.windowed_stream_plan(reqs(), 3, 5)
    assert next(plan) == ([0, 1], 0, 5) and len(read) == 1
    assert next(plan) == ([2], 0, 5) and len(read) == 2
    assert next(plan) == ([0, 1], 5, 10) and len(read) == 3


def make_net(conditional=True, image_size=32):
    opt = {"phase": "val", "gpu_ids": None, "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(TINY, in_channel=6 if conditional else 3),
                     "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                     "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt)
    net.set_new_noise_schedule(SCHED, "cpu")
    return net


def no_native(*args, **kwargs):
    raise AssertionError("the native side was reached before the requests were checked")


@pytest.mark.parametrize("requests,match", [
    ([("a", torch.zeros(3, 32, 32)), ("b", torch.zeros(3, 31, 64))], r"request 'b': canvas 31x64 is smaller than the window 32x32"),
    ([("a", torch.zeros(3, 32, 20))], r"request 'a': canvas 32x20 is smaller"),
    ([("a", torch.zeros(4, 40, 40))], r"request 'a': x_in must be \[3, H, W\]"),
    ([("a", torch.zeros(3, 32, 32)), ("b", torch.zeros(1, 3, 40, 40))], r"request 'b': x_in must be \[3, H, W\]"),
    ([("a", torch.zeros(3, 40, 40), torch.zeros(3, 40, 32))], r"request 'a': x_T must be \(3, 40, 40\)"),
    # 4 slots, overlap 8: 32x56 has 1 x 2 windows, 80x80 has 3 x 3; every request read at step 0 is checked before the first is admitted
    ([("a", torch.zeros(3, 32, 32)), ("b", torch.zeros(3, 32, 56)), ("c", torch.zeros(3, 80, 80))],
     r"request 'c': a 80x80 canvas has 9 windows, more than the stream's 4"),
    ([(0,)], r"a request is \(key, x_in\)"),
])
def test_windowed_stream_refuses_a_bad_request_before_anything_native(monkeypatch, requests, match):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_native)
    monkeypatch.setattr(_native, "WindowedStreamSampler", no_native)
    with pytest.raises(ValueError, match=match):
        list(net.super_resolution_windowed_stream(requests, slots=4))


def test_windowed_stream_refuses_bad_arguments_when_called(monkeypatch):
    net = make_net()
    monkeypatch.setattr(net, "_engine", no_native)
    with pytest.raises(_native.UnsupportedSizeError):
        net.super_resolution_windowed_stream([], window=(48, 48))
    with pytest.raises(ValueError, match="overlap 32 must be at least 0 and below the window side 32"):
        net.super_resolution_windowed_stream([], overlap=32)
    with pytest.raises(ValueError, match="slots must be >= 1"):
        net.super_resolution_windowed_stream([], slots=0)
    unc = make_net(conditional=False)
    monkeypatch.setattr(unc, "_engine", no_native)
    with pytest.raises(ValueError, match="needs a conditional model"):
        unc.super_resolution_windowed_stream([(0, torch.zeros(3, 40, 40))])


def test_windowed_stream_without_a_gpu_fails_loudly():
    net = make_net()
    with pytest.raises((_native.NativeLibraryError, RuntimeError)):
        list(net.super_resolution_windowed_stream([(0, torch.zeros(3, 40, 40))], slots=4))


def test_windowed_stream_kernels_do_not_spill():
    """ptxas -v of the three wstream kernels (lib/build.log, built first if needed: nvcc needs no GPU): no stack frame, no spills."""
    import importlib.util
    import os
    import re
    pkg = os.path.dirname(_native.__file__)
    spec = importlib.util.spec_from_file_location("sr3_b200_build_for_wstream_test", os.path.join(pkg, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build(force=False)
    log = open(os.path.join(pkg, "lib", "build.log")).read()
    for k in ("wstream_gather_kernel", "wstream_means_kernel", "wstream_merge_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % k,
                           log)
        assert props, "%s not found in the ptxas report" % k
        assert all(p == ("0", "0", "0") for p in props), (k, props)

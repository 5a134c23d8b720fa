"""SSIM at the exit of the sampling path (core/metrics.py:52-93, sr.py:216-217).

CPU: the oracle's numpy restatement against what the unmodified reference (cv2.filter2D in float64) computed for the pairs of
tests/golden/sr3_ssim_golden.pt (written by tests/golden/make_ssim_golden.py), and against the reference itself where its core/metrics.py
imports.  GPU: the device ssim / calculate_ssim / psnr_ssim of sr3_b200.core.metrics against the oracle, their determinism, and the
evaluation lines of sr.py run on a sampled batch."""
import importlib.util
import math
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import sr3_oracle as orc
from oracle import ssim_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TOL = 1e-12              # fp64 filtering in a different summation order than cv2: agreement to a few 1e-16, bound kept meaningful


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _load("make_ssim_golden", os.path.join(HERE, "golden", "make_ssim_golden.py"))      # numpy only at import: the pair recipe


@pytest.fixture(scope="module")
def ssim_golden():
    return torch.load(os.path.join(HERE, "golden", "sr3_ssim_golden.pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def pairs(ssim_golden):
    """name -> (a, b) uint8 arrays: the stored raw arrays, or the seeded draw checked against the stored digest."""
    out = {}
    for name, rec in ssim_golden.items():
        if "a" in rec:
            a, b = rec["a"].numpy(), rec["b"].numpy()
        else:
            a, b = GEN.pair(rec["seed"], rec["shape1"], rec["shape2"], rec["kind"], rec["amplitude"])
        assert GEN.digest(a, b) == rec["sha256"], name
        out[name] = (a, b)
    return out


def _run(fn, a, b):
    try:
        v = fn(a, b)
    except ValueError as e:
        return "error", str(e)
    return "value", None if v is None else float(v)


def _same(got, want, tol=TOL):
    """Both the same ValueError message, both None, both nan, or two floats within tol."""
    (gk, gv), (wk, wv) = got, want
    if gk != wk or (gv is None) != (wv is None):
        return False
    if gk == "error" or gv is None:
        return gv == wv
    if math.isnan(wv):
        return math.isnan(gv)
    return abs(gv - wv) <= tol


_ORACLE = {}


def _oracle(name, fn_name, a, b):
    key = (name, fn_name)
    if key not in _ORACLE:
        _ORACLE[key] = _run(getattr(so, fn_name), a, b)
    return _ORACLE[key]


def _live_reference():
    path = os.path.join(ROOT, "oracle", "_ref", "core", "metrics.py")
    if not os.path.exists(path):
        pytest.skip("the reference is not vendored under oracle/_ref")
    try:
        return _load("ref_core_metrics", path)
    except ImportError as e:                     # core/metrics.py imports cv2 and torchvision
        pytest.skip(f"the reference's core/metrics.py does not import here: {e}")


# ------------------------------------------------------------------------------------------------------------------------------ CPU


def test_golden_covers_every_behaviour(ssim_golden):
    kinds = {rec["calculate_ssim"][0] for rec in ssim_golden.values()}
    values = [rec["calculate_ssim"][1] for rec in ssim_golden.values() if rec["calculate_ssim"][0] == "value"]
    assert kinds == {"value", "error"}
    assert None in values and any(v is not None and math.isnan(v) for v in values) and 1.0 in values
    assert {rec["calculate_ssim"][1] for rec in ssim_golden.values() if rec["calculate_ssim"][0] == "error"} == {
        "Input images must have the same dimensions.", "Wrong input image dimensions."}


def test_oracle_matches_reference_golden(ssim_golden, pairs):
    for name, rec in ssim_golden.items():
        a, b = pairs[name]
        got = _oracle(name, "calculate_ssim", a, b)
        assert _same(got, rec["calculate_ssim"]), (name, got, rec["calculate_ssim"])
        if "ssim" in rec:
            got = _oracle(name, "ssim", a, b)
            assert _same(got, rec["ssim"]), (name, got, rec["ssim"])
    assert _oracle("identical_96x80x3", "calculate_ssim", *pairs["identical_96x80x3"]) == ("value", 1.0)


def test_oracle_matches_live_reference(ssim_golden, pairs):
    ref = _live_reference()
    rs = np.random.RandomState(12)
    extra = {"float_37x29x3": (rs.rand(37, 29, 3) * 255, rs.rand(37, 29, 3) * 255),
             "float32_gray_20x31": ((rs.rand(20, 31) * 255).astype(np.float32), (rs.rand(20, 31) * 255).astype(np.float32))}
    for name, (a, b) in list(pairs.items()) + list(extra.items()):
        for fn in ("calculate_ssim", "ssim"):
            if fn == "ssim" and not (a.shape == b.shape and a.ndim in (2, 3)):
                continue
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)          # np.mean of the empty crop of a too-small image
                want = _run(getattr(ref, fn), a, b)
            assert _same(_oracle(name, fn, a, b), want), (name, fn)


# ------------------------------------------------------------------------------------------------------------------------------ GPU


def _as_input(x, form, dtype):
    x = x.astype(np.float64) if dtype == "float64" else x
    return torch.from_numpy(np.ascontiguousarray(x)).cuda() if form == "cuda" else x


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["uint8", "float64"])
@pytest.mark.parametrize("form", ["numpy", "cuda"])
def test_device_ssim_matches_oracle_on_golden(ssim_golden, pairs, form, dtype):
    from sr3_b200.core import metrics
    for name, rec in ssim_golden.items():
        a, b = pairs[name]
        da, db = _as_input(a, form, dtype), _as_input(b, form, dtype)
        want = _oracle(name, "calculate_ssim", a, b)
        got = _run(metrics.calculate_ssim, da, db)
        assert _same(got, want), (name, got, want)
        if "ssim" in rec:
            want = _oracle(name, "ssim", a, b)
            got = _run(metrics.ssim, da, db)
            assert _same(got, want), (name, got, want)
    assert metrics.calculate_ssim(*[_as_input(x, form, dtype) for x in pairs["identical_96x80x3"]]) == 1.0


@pytest.mark.gpu
def test_device_ssim_of_non_integer_images_matches_oracle():
    from sr3_b200.core import metrics
    rs = np.random.RandomState(13)
    for shape in [(37, 29, 3), (20, 31), (64, 64, 1)]:
        a = rs.rand(*shape) * 255
        b = np.clip(a + rs.randn(*shape) * 9, 0, 255)
        want = so.calculate_ssim(a, b)
        assert abs(metrics.calculate_ssim(a, b) - want) <= TOL, shape
        assert abs(metrics.calculate_ssim(a.astype(np.float32), b.astype(np.float32)) - so.calculate_ssim(a.astype(np.float32), b.astype(np.float32))) <= TOL
        assert abs(metrics.calculate_ssim(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) - want) <= TOL


def _batch_ssim(a, b):
    """sr3_ssim over a batch of HWC pairs a, b (CUDA uint8 [n, H, W, C])."""
    import ctypes
    from sr3_b200 import _native
    n, H, W, C = a.shape
    out = (ctypes.c_double * n)()
    _native._check(_native.lib().sr3_ssim(_native._ptr(a), _native._ptr(b), 0, n, H, W, C, out, _native._stream()))
    return np.array(out[:], dtype=np.float64)


@pytest.mark.gpu
def test_device_ssim_is_deterministic_and_batch_independent():
    from sr3_b200.core import metrics
    rs = np.random.RandomState(14)
    for H, W in [(128, 128), (83, 61)]:
        a = rs.randint(0, 256, (16, H, W, 3)).astype(np.uint8)
        b = np.clip(a.astype(np.int32) + rs.randint(-30, 31, a.shape), 0, 255).astype(np.uint8)
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        batch = _batch_ssim(da, db)
        assert np.array_equal(batch, _batch_ssim(da, db))
        for i in (0, 5, 15):
            alone = metrics.ssim(a[i], b[i])
            assert alone == batch[i] and alone == metrics.ssim(a[i], b[i]), (H, W, i)
            assert alone == metrics.ssim(da[i], db[i])
            assert abs(alone - so.ssim(a[i], b[i])) <= TOL


def _sampled_like(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    hr = (torch.rand(B, C, H, W, generator=g) * 2 - 1)
    sr = (hr + torch.randn(B, C, H, W, generator=g) * 0.08).clamp(-1.05, 1.05)      # a few values outside [-1, 1]: tensor2img clamps
    return sr.cuda(), hr.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(16, 3, 128, 128), (4, 1, 40, 36), (3, 3, 8, 12)])
def test_psnr_ssim_of_a_batch(shape):
    from sr3_b200.core import metrics
    sr, hr = _sampled_like(*shape, seed=sum(shape))
    psnr, ssim, sr_u8, hr_u8 = metrics.psnr_ssim(sr, hr, return_images=True)
    assert psnr.dtype == np.float64 and ssim.dtype == np.float64 and psnr.shape == ssim.shape == (shape[0],)
    p2, s2 = metrics.psnr_ssim(sr, hr)
    assert np.array_equal(p2, psnr) and np.array_equal(s2, ssim, equal_nan=True)
    for i in range(shape[0]):
        a, b = metrics.tensor2img(sr[i]), metrics.tensor2img(hr[i])
        assert a.dtype == np.uint8 and np.array_equal(sr_u8[i], a) and np.array_equal(hr_u8[i], b)
        assert psnr[i] == metrics.calculate_psnr(a, b)
        want = so.calculate_ssim(a, b)
        if math.isnan(want):
            assert math.isnan(ssim[i])
        else:
            assert abs(ssim[i] - want) <= TOL, (i, ssim[i], want)
            assert ssim[i] == metrics.calculate_ssim(a, b)
    with pytest.raises(ValueError):
        metrics.psnr_ssim(sr[:, :1].expand(-1, 2, -1, -1), hr[:, :1].expand(-1, 2, -1, -1))


@pytest.mark.gpu
def test_sr_py_evaluation_lines_on_a_sampled_batch():
    """super_resolution(continous=True) of a tiny SR3 net, then sr.py:216-217 written with sr3_b200's metrics, per image of the batch."""
    import sr3_b200
    from sr3_b200.core import metrics as Metrics
    sched = {"schedule": "linear", "n_timestep": 10, "linear_start": 1e-6, "linear_end": 1e-2}
    unet = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)
    opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
           "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": unet, "beta_schedule": {"train": sched, "val": sched},
                     "diffusion": {"image_size": 32, "channels": 3, "conditional": True}}}
    torch.manual_seed(0)
    net = sr3_b200.define_G(opt).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    g = torch.Generator().manual_seed(21)
    hr = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    cond = (hr + torch.randn(2, 3, 32, 32, generator=g) * 0.2).clamp(-1, 1)
    x_T = torch.randn(2, 3, 32, 32, generator=g)
    out = net.super_resolution(cond.cuda(), continous=True, x_T=x_T.cuda(), seed=3)
    sr_last = out[-2:]
    assert torch.isfinite(sr_last).all()
    psnr, ssim = Metrics.psnr_ssim(sr_last, hr.cuda())
    for i in range(2):
        hr_img = Metrics.tensor2img(hr[i].cuda())
        eval_psnr = Metrics.calculate_psnr(Metrics.tensor2img(sr_last[i]), hr_img)        # sr.py:216
        eval_ssim = Metrics.calculate_ssim(Metrics.tensor2img(sr_last[i]), hr_img)        # sr.py:217
        sr_img = orc.tensor2img(sr_last[i].cpu())
        assert np.array_equal(sr_img, Metrics.tensor2img(sr_last[i])) and np.array_equal(orc.tensor2img(hr[i]), hr_img)
        assert eval_psnr == orc.calculate_psnr(sr_img, hr_img) == psnr[i]
        want = so.calculate_ssim(sr_img, hr_img)
        assert abs(eval_ssim - want) <= TOL and eval_ssim == ssim[i], (eval_ssim, want, ssim[i])

"""The sampler's Gaussian noise as tests/_philox.py restates it (Philox4x32-10 keyed by the seed, counter (pixel, sample index, t), then
Box-Muller; tests/test_gpu_sampling.py ties the device's draws to this restatement).  Seeds and sample indices have their high words set,
as Python's seeds in [0, 2^62) always do.  Fixed seeds: every statistic below is deterministic."""
import math

import numpy as np
import pytest
from scipy import stats

import _philox

SEEDS = (0x3A5F_1C2B_9D4E_7061, 0x0123_4567_89AB_CDEF, 2 ** 62 + 12345)
H = W = 128
IDX = np.arange(2 ** 32 - 12, 2 ** 32 + 12, 2, dtype=np.uint64)            # 12 images across the high-word boundary of the sample index
T_STEPS = (1999, 1000, 1)
ZMAX = math.sqrt(-2.0 * math.log(2.0 ** -32))                               # u1 >= 2^-32


@pytest.fixture(scope="module")
def draws():
    """(seed, t) -> z [12, 3, H, W]: 3 seeds x 3 steps x 590 K values, plus t - 1 of the first seed (time correlation): 5.9e6 values."""
    keys = [(s, t) for s in SEEDS for t in T_STEPS] + [(SEEDS[0], T_STEPS[0] - 1)]
    return {(s, t): _philox.sampling_noise(s, IDX, t, H, W) for s, t in keys}


def _all(draws):
    z = np.concatenate([v.ravel() for v in draws.values()])
    assert z.size >= 4_000_000
    return z


def test_moments_within_five_standard_errors(draws):
    z = _all(draws)
    n = z.size
    m, v = z.mean(), z.var()
    sk, ku = stats.skew(z), stats.kurtosis(z)                # (excess kurtosis)
    print(f"N={n}: mean {m:.2e} (se {1 / math.sqrt(n):.1e}), var-1 {v - 1:.2e} (se {math.sqrt(2 / n):.1e}), skew {sk:.2e} "
          f"(se {math.sqrt(6 / n):.1e}), excess kurtosis {ku:.2e} (se {math.sqrt(24 / n):.1e})")
    assert abs(m) < 5 / math.sqrt(n)
    assert abs(v - 1) < 5 * math.sqrt(2 / n)
    assert abs(sk) < 5 * math.sqrt(6 / n)
    assert abs(ku) < 5 * math.sqrt(24 / n)


def test_kolmogorov_smirnov_and_tails(draws):
    z = _all(draws)
    ks = stats.kstest(z, "norm")
    p4 = 2 * stats.norm.sf(4.0)
    frac = np.mean(np.abs(z) > 4.0)
    se = math.sqrt(p4 * (1 - p4) / z.size)
    print(f"KS D={ks.statistic:.2e} p={ks.pvalue:.3f}; |z| > 4: {frac:.3e} (expected {p4:.3e} +- {se:.1e}); max |z| {np.abs(z).max():.4f} "
          f"<= {ZMAX:.4f}")
    assert ks.pvalue > 1e-3
    assert abs(frac - p4) < 5 * se
    assert np.abs(z).max() <= ZMAX


def _corr(a, b):
    a, b = a.ravel(), b.ravel()
    r = np.corrcoef(a, b)[0, 1]
    return r, 5 / math.sqrt(a.size)


def test_no_correlation_across_channels_pixels_steps_images_and_seeds(draws):
    s0, t0 = SEEDS[0], T_STEPS[0]
    z = draws[(s0, t0)]
    pairs = {
        "channel 0/1": (z[:, 0], z[:, 1]), "channel 0/2": (z[:, 0], z[:, 2]), "channel 1/2": (z[:, 1], z[:, 2]),
        "pixel / right neighbour": (z[..., :-1], z[..., 1:]), "pixel / lower neighbour": (z[..., :-1, :], z[..., 1:, :]),
        "t / t-1": (z, draws[(s0, t0 - 1)]), "image i / i+1": (z[:-1], z[1:]),
    }
    for bit in (32, 45, 61):                              # seeds that differ in one bit of the key's high word
        pairs[f"seed bit {bit}"] = (z, _philox.sampling_noise(s0 ^ (1 << bit), IDX, t0, H, W))
    for name, (a, b) in pairs.items():
        r, bound = _corr(a, b)
        print(f"corr {name}: {r:+.2e} (bound {bound:.1e})")
        assert abs(r) < bound, name


@pytest.mark.parametrize("word", range(6))
def test_every_counter_and_key_word_changes_the_draw(word):
    """Counter (pixel, index low, t, index high) and key (seed low, seed high): adding 1 to any one word changes every value."""
    seed, idx, t = SEEDS[0], IDX, 1000

    def bump(*w):
        w = list(w)
        w[word] = (w[word] + np.uint64(1)) & np.uint64(0xFFFFFFFF) if word < 4 else (w[word] + 1) & 0xFFFFFFFF
        return tuple(w)

    a = _philox.sampling_noise(seed, idx, t, 16, 16)
    b = _philox.sampling_noise(seed, idx, t, 16, 16, words=bump)
    assert np.all(a != b)


def test_layout_is_the_documented_one():
    """Pixel oh * W + ow is word 0, the index words 1 and 3, t word 2; the same pixel of two images is two counters (no reuse across a
    batch or across the index's high-word boundary)."""
    seed = SEEDS[1]
    z = _philox.sampling_noise(seed, [2 ** 32 - 1, 2 ** 32, 7], 5, 4, 8)
    c0, c1, c2, c3 = _philox.philox4x32_10(3 * 8 + 5, 0, 5, 1, seed & 0xFFFFFFFF, seed >> 32)
    z0, z1 = _philox.box_muller(c0, c1)
    z2, _ = _philox.box_muller(c2, c3)
    assert np.array_equal(z[1, :, 3, 5], np.array([z0, z1, z2]).ravel())
    assert not np.array_equal(z[0], z[1]) and not np.array_equal(z[1], z[2])
    # u1 = 1 (word 0xffffffff rounds to 2^32 in fp32): r = 0; word 0: u1 = 2^-32, the largest radius
    r_big, _ = _philox.box_muller(np.uint64(0), np.uint64(0))
    assert r_big == pytest.approx(ZMAX, rel=1e-15)
    r0, _ = _philox.box_muller(np.uint64(0xFFFFFFFF), np.uint64(0))
    assert r0 == 0.0

"""numpy restatements of the device's two Philox4x32-10 streams (philox4x32_10 / box_muller in gemm_wgmma.cuh), so that tests can
reproduce what the device drew.

Dropout keep-mask (drop_scale4 in aux_kernels.cuh): element (b, c, pixel) of a [B][HW][C] activation belongs to the 4-channel vector
v = (b * HW + pixel) * C/4 + c/4.  Its counter is (v mod 2^32, v >> 32, layer, 0x5d0), its key (seed mod 2^32, seed >> 32); output word
c mod 4, converted to fp32 and scaled by 2^-32 in fp32, is compared with the fp32 drop probability: the element is kept when it is >= p.

Sampling noise (final_epilogue in gemm_wgmma.cuh: the z of x_{t-1} = mean + z exp(0.5 logvar) at timestep t > 0): pixel (oh, ow) of the
image with global sample index n (first_index + image of the batch) has the counter (oh * W + ow, n mod 2^32, t, n >> 32) and the key
(seed mod 2^32, seed >> 32).  Box-Muller turns the output words (w0, w1) into channels 0 and 1 and (w2, w3) into channel 2 (its sine is
unused): u1 = (fp32(a) + 1) 2^-32 in (0, 1], u2 = fp32(b) 2^-32 in [0, 1), both formed in fp32, then r = sqrt(-2 ln u1) and
z = r cos(2 pi u2), r sin(2 pi u2)."""
import numpy as np

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Ten rounds of Philox4x32 on arrays of 32-bit counters (any integer dtype); returns four uint64 arrays of 32-bit words."""
    c = [np.asarray(x).astype(np.uint64) & _M32 for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c0, c1, c2, c3 = (x.copy() for x in c)
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def keep_mask(B, C, HW, p, seed, layer):
    """uint8 keep-mask [B][C][HW] (NCHW, 1 = keep) of dropout layer `layer` for `seed` at drop probability p (rounded to fp32)."""
    assert C % 4 == 0
    vec = np.arange(B * HW * (C // 4), dtype=np.uint64)                 # [b][pixel][c/4]
    words = philox4x32_10(vec & _M32, vec >> np.uint64(32), layer, 0x5D0, seed & 0xFFFFFFFF, seed >> 32)
    u = np.stack([(w.astype(np.float64).astype(np.float32) * np.float32(2.3283064365386963e-10)) for w in words], axis=-1)   # [..][j]
    keep = (u >= np.float32(p)).reshape(B, HW, C)
    return np.ascontiguousarray(keep.transpose(0, 2, 1)).astype(np.uint8)


def _u32_to_f32(w):
    return w.astype(np.float64).astype(np.float32)          # exact in fp64, then one round-to-nearest to fp32 (cvt.rn.f32.u32)


def box_muller(a, b):
    """(r cos, r sin) in fp64 of the fp32 uniforms the device forms from words a, b."""
    u1 = (_u32_to_f32(a) + np.float32(1.0)) * np.float32(2.3283064365386963e-10)
    u2 = _u32_to_f32(b) * np.float32(2.3283064365386963e-10)
    r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    ang = 2.0 * np.pi * u2.astype(np.float64)
    return r * np.cos(ang), r * np.sin(ang)


def sampling_noise(seed, sample_index, t, H, W, words=None):
    """fp64 z [n, 3, H, W] the posterior epilogue draws at timestep t for the images with global indices `sample_index` (n of them).
    `words` (tests of the tests): a function mapping the counter / key words (c0, c1, c2, c3, k0, k1) to other ones."""
    idx = np.asarray(sample_index, dtype=np.uint64).reshape(-1, 1)
    pix = np.arange(H * W, dtype=np.uint64).reshape(1, -1)
    seed = int(seed)
    w = (pix, idx & _M32, np.uint64(t), idx >> np.uint64(32), seed & 0xFFFFFFFF, seed >> 32)
    if words is not None:
        w = words(*w)
    c0, c1, c2, c3 = philox4x32_10(*w)
    z0, z1 = box_muller(c0, c1)
    z2, _ = box_muller(c2, c3)
    return np.stack([z0, z1, z2], axis=1).reshape(idx.shape[0], 3, H, W)


def scale_mask(keep, p):
    """The scaled mask the oracle multiplies by (0 or 1 / (1 - p), both in fp32, as drop_scale4 forms them)."""
    import torch
    k = torch.as_tensor(keep).float()
    return k * (np.float32(1.0) / (np.float32(1.0) - np.float32(p)))

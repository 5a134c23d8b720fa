"""numpy restatement of the device's dropout keep-mask (philox4x32_10 in gemm_wgmma.cuh, drop_scale4 in aux_kernels.cuh), so that tests can
reproduce the masks a training forward drew and hand the same masks to the oracle.

Element (b, c, pixel) of a [B][HW][C] activation belongs to the 4-channel vector v = (b * HW + pixel) * C/4 + c/4.  Its counter is
(v mod 2^32, v >> 32, layer, 0x5d0), its key (seed mod 2^32, seed >> 32); output word c mod 4, converted to fp32 and scaled by 2^-32 in
fp32, is compared with the fp32 drop probability: the element is kept when it is >= p."""
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


def scale_mask(keep, p):
    """The scaled mask the oracle multiplies by (0 or 1 / (1 - p), both in fp32, as drop_scale4 forms them)."""
    import torch
    k = torch.as_tensor(keep).float()
    return k * (np.float32(1.0) / (np.float32(1.0) - np.float32(p)))

"""Both attention paths kernel by kernel against fp64 references (reference unet.py:129-139: S = q k^T / sqrt(C), softmax over the keys of
the same image, O = P v).

The unfused path (sr3_test_attention_unfused: the plan's S launch, softmax_kernel and P.v launch) is checked launch by launch, each on the
previous launch's actual device output, with element-wise bounds.  The fused kernel (attn_kernel) is checked against a reference that
rounds P where the kernel does, so that its bound is tight enough to see one dropped key or a mis-masked segment edge."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24           # fp32 unit roundoff
# (nz, Lt, HW, C): 8x8 and 4x4 images sharing a 128-token batch (precise mode and the training forward), 256-token batches, the batches
# of the 16->128 config at 128x256 (512 tokens) and at 512x512 (4096 tokens), and the C = 1024 middle block of the 64->512 config at
# 512x512 (1024 tokens) and at 128x128 (8x8, two images per batch)
UNFUSED = [(1, 128, 64, 128), (3, 128, 16, 256), (2, 256, 256, 512), (1, 512, 512, 512), (2, 1024, 1024, 256), (1, 4096, 4096, 512),
           (1, 1024, 1024, 1024), (2, 128, 64, 1024)]


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def split(x):
    """[hi | lo] bf16 pair of an fp32 tensor along the last dimension (lo = bf16(x - hi))."""
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


def bf16_ulp(x):
    """One bf16 ulp at |x| (x != 0)."""
    return torch.exp2(torch.floor(torch.log2(x.abs())) - 7)


def first_bad(ok, what):
    bad = (~ok).nonzero()
    if bad.numel() == 0:
        return ""
    z, r, c = bad[0].tolist()
    return f"{what}: {int((~ok).sum())} elements out of bounds, first at batch {z} row {r} column {c}"


def inputs(nz, Lt, C, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(nz, Lt, C, generator=g) for _ in range(3))
    return 2.0 * q, k, v                    # logits with a spread of a few units after the 1/sqrt(C) scaling


def seg_mask(Lt, HW):
    seg = torch.arange(Lt) // HW
    return seg[:, None] == seg[None, :]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("nz,Lt,HW,C", UNFUSED)
def test_unfused_attention_launch_by_launch(nz, Lt, HW, C, precise):
    from sr3_b200 import _native
    if precise and Lt == 4096:
        pytest.skip("precise mode runs the 16->128 config up to 128x256")
    q, k, v = inputs(nz, Lt, C, nz * 1000 + Lt + HW + C)
    if precise:
        (qh, ql), (kh, kl), (vh, vl) = split(q), split(k), split(v)
        qk = torch.cat([qh, kh, ql, kl], 2)
        vT = torch.cat([vh.transpose(1, 2), vl.transpose(1, 2)], 2)         # rows [hi | lo] of Lt keys each
        qo, ko, vo = qh.double() + ql.double(), kh.double() + kl.double(), vh.double() + vl.double()
    else:
        qk = torch.cat([q, k], 2).bfloat16()
        vT = v.bfloat16().transpose(1, 2)
        qo, ko, vo = qk[..., :C].double(), qk[..., C:2 * C].double(), v.bfloat16().double()
    S, P, O = _native.test_attention_unfused(qk.reshape(nz * Lt, -1).contiguous().cuda(), vT.reshape(nz * C, -1).contiguous().cuda(), nz, Lt,
                                             HW, C, precise)
    S, P, O = S.cpu().double().reshape(nz, Lt, Lt), P.cpu().double().reshape(nz, Lt, -1), O.cpu().double().reshape(nz, Lt, -1)
    mask = seg_mask(Lt, HW).expand(nz, Lt, Lt)

    # S on the same operands: the fp32 accumulation over C products (and, in precise mode, the dropped lo x lo pass, <= 2^-18 |q||k|)
    s_ref = qo @ ko.transpose(1, 2) / math.sqrt(C)
    s_abs = qo.abs() @ ko.abs().transpose(1, 2) / math.sqrt(C)
    s_tol = ((C + 2) * U32 + (2.0 ** -17 if precise else 0.0)) * s_abs
    e_s = rel(S, s_ref)
    ok = (S - s_ref).abs() <= s_tol
    # P: fp64 softmax of the device's S over each segment; one bf16 ulp (bf16 mode), the hi + lo pair error 2^-17 plus the fp32 error of
    # the row sum (precise mode); exactly 0 outside the segment
    p_ref = torch.softmax(S.masked_fill(~mask, float("-inf")), dim=-1)
    if precise:
        p_hi, p_lo = P[..., :Lt], P[..., Lt:]
        p_dev = p_hi + p_lo
        p_tol = (2.0 ** -17 + (HW / 32 + 8) * U32) * p_ref
        ok_p = ((p_dev - p_ref).abs() <= p_tol) & ((p_hi - p_ref).abs() <= bf16_ulp(p_ref).where(mask, torch.zeros(())))
        zero_out = (p_hi[~mask] == 0).all() and (p_lo[~mask] == 0).all()
    else:
        p_dev = P
        ok_p = (p_dev - p_ref).abs() <= torch.where(mask, bf16_ulp(p_ref.clamp_min(1e-300)), torch.zeros(()))
        zero_out = bool((p_dev[~mask] == 0).all())
    worst_p = ((p_dev - p_ref).abs()[mask] / bf16_ulp(p_ref[mask])).max().item()
    # O: fp64 product of the device's P with v; bf16 rounding of the result (2^-8 relative; precise: the pair, 2^-17) plus the fp32
    # accumulation over Lt products and the dropped lo x lo pass
    o_ref = p_dev @ vo
    o_abs = p_dev.abs() @ vo.abs()
    o_dev = O[..., :C] + O[..., C:] if precise else O
    o_tol = (2.0 ** -17 if precise else 2.0 ** -8) * o_ref.abs() + ((Lt + 2) * U32 + (2.0 ** -17 if precise else 0.0)) * o_abs
    ok_o = (o_dev - o_ref).abs() <= o_tol
    e_o = rel(o_dev, o_ref)
    print(f"unfused nz={nz} Lt={Lt} HW={HW} C={C} precise={precise}: S rel L2 {e_s:.2e} (bound 2e-5), max |dS|/tol "
          f"{((S - s_ref).abs() / s_tol).max():.2e}; P worst {worst_p:.2f} bf16 ulp (bound 1); O rel L2 {e_o:.2e}, max |dO|/tol "
          f"{((o_dev - o_ref).abs() / o_tol).max():.2e}")
    assert e_s < 2e-5, e_s
    assert ok.all(), first_bad(ok, "S")
    assert ok_p.all(), first_bad(ok_p, "P")
    assert zero_out, "P is not exactly 0 outside the segment"
    assert ok_o.all(), first_bad(ok_o, "O")

    if precise:
        # end to end against fp64 attention on the unrounded fp32 q, k, v: every operand carries the split error 2^-17, S the accumulation
        # error above; softmax turns an absolute S error d into a relative P error <= 2 d, and the O pair adds 2^-17
        d_s = ((2 * 2.0 ** -17 + 2.0 ** -17 + (C + 2) * U32) * s_abs).max().item()
        bound = 2 * d_s + 3 * 2.0 ** -17 + (Lt + 2) * U32
        full = torch.softmax((q.double() @ k.double().transpose(1, 2) / math.sqrt(C)).masked_fill(~mask, float("-inf")), -1) @ v.double()
        e = rel(o_dev, full)
        print(f"  precise end to end: O rel L2 {e:.2e} (derived bound {bound:.2e})")
        assert e < bound, (e, bound)

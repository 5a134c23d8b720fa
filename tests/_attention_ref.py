"""The reference of the fused attention kernel (attn_wgmma.cuh, attn_unit), shared by the fused-attention tests: it rounds P where the
kernel does, so the bound is far tighter than against a plain fp32 softmax."""
import math

import torch


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def seg_mask(Lt, HW):
    seg = torch.arange(Lt) // HW
    return seg[:, None] == seg[None, :]


def fused_reference(qk, vb, Lt, HW, C, drop_key=False, plain=False):
    """What attn_kernel computes, in fp64 on the same bf16 operands: per segment P~ = bf16(exp(S / sqrt(C) - max)), the row sum over the
    UNROUNDED exponentials, O = P~ v / sum rounded to bf16.  plain: the fp32 softmax of the past (P not rounded, O fp32);
    drop_key: the first key of every segment left out (a wrong reference, for the self-check)."""
    q, k, v = qk[..., :C].double(), qk[..., C:].double(), vb.double()
    mask = seg_mask(Lt, HW)
    if drop_key:
        mask = mask & (torch.arange(Lt) % HW != 0)[None, :]
    s = (q @ k.transpose(1, 2) / math.sqrt(C)).masked_fill(~mask, float("-inf"))
    if plain:
        return (torch.softmax(s.float(), -1) @ vb.float()).double()
    e = torch.exp(s - s.amax(-1, keepdim=True))
    return ((e.bfloat16().double() @ v) / e.sum(-1, keepdim=True)).bfloat16().double()


# Measured on an H100 80GB HBM3 (700 W limit) over the shapes of test_fused_attention_matches_fp32 and test_attention_16_tokens_per_image:
# 3.8e-5 to 1.05e-4 (rounding flips where the fp32 and fp64 values straddle a bf16 boundary); the plain fp32 softmax reference misses the
# kernel by 1.83e-3 to 1.93e-3 and the reference without one key per segment by 4.5e-2 or more.
FUSED_TOL = 5e-4


def check_fused(out, qk, vb, Lt, HW, C):
    ref = fused_reference(qk, vb, Lt, HW, C)
    e = rel(out, ref)
    wrong = {"fp32 softmax": rel(out, fused_reference(qk, vb, Lt, HW, C, plain=True)),
             "one key dropped": rel(out, fused_reference(qk, vb, Lt, HW, C, drop_key=True))}
    print(f"fused Lt={Lt} HW={HW} C={C}: rel L2 {e:.2e} (bound {FUSED_TOL:.0e}); wrong references: "
          + ", ".join(f"{k} {v:.2e}" for k, v in wrong.items()))
    assert torch.isfinite(out).all()
    assert e < FUSED_TOL, e
    for name, w in wrong.items():
        assert w > FUSED_TOL, (name, w)

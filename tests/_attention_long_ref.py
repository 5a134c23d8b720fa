"""References for the streaming-softmax attention kernel (attn_long_wgmma.cuh, attn_long_kernel), shared by tests/test_gpu_attention_long.py
and tests/test_attention_long_ref.py.

streaming_reference walks the keys in blocks as the kernel does, in fp64 on the same bf16 operands, and rounds where the kernel rounds:
P~ = bf16(exp(s - m)) with m the running maximum of the key blocks seen so far, the row sum over the unrounded exponentials, the output
to bf16.  plain_reference is fp64 softmax attention with no knowledge of the kernel's order."""
import math

import torch

KB = 128                  # keys per block of attn_long_kernel


def operands(q, k, v):
    """fp32 q, k, v [nz, Lt, C] -> the kernel's bf16 operands: qk [nz, Lt, 2C] and v rounded to bf16 [nz, Lt, C]."""
    return torch.cat([q, k], 2).bfloat16(), v.bfloat16()


def plain_reference(qk, vb, C):
    q, k, v = qk[..., :C].double(), qk[..., C:].double(), vb.double()
    return torch.softmax(q @ k.transpose(1, 2) / math.sqrt(C), -1) @ v


def streaming_reference(qk, vb, C, block=KB, rounded=True):
    """rounded=False switches the two bf16 roundings off: what is left is plain softmax attention in another summation order."""
    q, k, v = qk[..., :C].double(), qk[..., C:].double(), vb.double()
    nz, Lt, _ = q.shape
    s = q @ k.transpose(1, 2) / math.sqrt(C)
    m = torch.full((nz, Lt, 1), -float("inf"), dtype=torch.float64)
    l = torch.zeros(nz, Lt, 1, dtype=torch.float64)
    o = torch.zeros(nz, Lt, C, dtype=torch.float64)
    for k0 in range(0, Lt, block):
        sb = s[..., k0:k0 + block]
        m_new = torch.maximum(m, sb.amax(-1, keepdim=True))
        a = torch.exp(m - m_new)                   # 0 at the first block
        e = torch.exp(sb - m_new)
        l = a * l + e.sum(-1, keepdim=True)
        o = a * o + (e.bfloat16().double() if rounded else e) @ v[:, k0:k0 + block]
        m = m_new
    out = o / l
    return out.bfloat16().double() if rounded else out


def adversarial(kind, Lt, C, seed=0):
    """fp32 q, k, v [1, Lt, C] whose logits stress the running maximum.  k is a per-key multiple of one direction u and q a per-row multiple
    of the same u, so logit(row, key) = a_row b_key |u|^2 / sqrt(C) has the sign and the order of b_key for a_row > 0.
      rising:  b increases along the keys (every block raises the maximum)      falling: b decreases (the first block holds it)
      spike:   one key of the last block far above the rest                     equal:   all logits equal (k = 0)
      wide:    b spans more than 80 in log2 units of the scaled logit: a missing rescale overflows or zeroes the row"""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(C, generator=g).sign()                             # |u|^2 = C exactly, so logit = a b sqrt(C)
    a = 0.5 + torch.rand(Lt, generator=g)                              # per-row factor in [0.5, 1.5)
    t = torch.linspace(0, 1, Lt)
    rc = 1.0 / math.sqrt(C)
    if kind == "rising":
        b = 12.0 * t * rc
    elif kind == "falling":
        b = 12.0 * (1 - t) * rc
    elif kind == "spike":
        b = torch.randn(Lt, generator=g) * rc
        b[Lt - 37] = 30.0 * rc
    elif kind == "equal":
        b = torch.zeros(Lt)
    elif kind == "wide":
        b = 160.0 * t * rc                                             # scaled logits span 0.5 * 160 * log2(e) = 115 or more in log2 units
    else:
        raise ValueError(kind)
    q = (a[:, None] * u[None, :])[None]
    k = (b[:, None] * u[None, :])[None]
    v = torch.randn(1, Lt, C, generator=g)
    return q, k, v


ADVERSARIAL = ("rising", "falling", "spike", "equal", "wide")

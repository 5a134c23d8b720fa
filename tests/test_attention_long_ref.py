"""The streaming reference the long-row attention kernel is tested against (tests/_attention_long_ref.py) is itself softmax attention:
with its bf16 roundings switched off it equals plain fp64 softmax attention, for both block sizes and on the rows built to stress the
running maximum.  With the roundings on it stays within the bf16 rounding of P~ and of the output."""
import pytest
import torch

import _attention_long_ref as lr
from _attention_ref import rel


def _random(nz, Lt, C, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(nz, Lt, C, generator=g) for _ in range(3))
    return 2.0 * q, k, v


@pytest.mark.parametrize("block", [64, 128])
@pytest.mark.parametrize("kind", ("random",) + lr.ADVERSARIAL)
def test_streaming_reference_is_softmax_attention(kind, block):
    Lt, C = 512, 128
    q, k, v = _random(2, Lt, C, 1) if kind == "random" else lr.adversarial(kind, Lt, C)
    qk, vb = lr.operands(q, k, v)
    plain = lr.plain_reference(qk, vb, C)
    exact = lr.streaming_reference(qk, vb, C, block=block, rounded=False)
    assert torch.isfinite(exact).all()
    assert rel(exact, plain) < 1e-12, rel(exact, plain)
    rounded = lr.streaming_reference(qk, vb, C, block=block)
    assert torch.isfinite(rounded).all()
    assert rel(rounded, plain) < 2.0 ** -7, rel(rounded, plain)


def test_adversarial_rows_move_the_running_maximum_as_described():
    Lt, C = 512, 128
    blockmax = {}
    for kind in lr.ADVERSARIAL:
        q, k, v = lr.adversarial(kind, Lt, C)
        qk, _ = lr.operands(q, k, v)
        s = qk[..., :C].double() @ qk[..., C:].double().transpose(1, 2) / C ** 0.5
        blockmax[kind] = s.reshape(1, Lt, Lt // lr.KB, lr.KB).amax(-1)           # [1, row, block]
    assert (blockmax["rising"].diff(dim=-1) > 0).all()
    assert (blockmax["falling"].diff(dim=-1) < 0).all()
    assert (blockmax["spike"].argmax(-1) == Lt // lr.KB - 1).all()
    assert (blockmax["equal"] == 0).all()
    span = (blockmax["wide"][..., -1] - blockmax["wide"][..., 0]) * 1.4426950408889634
    assert (span > 80).all(), span.min()

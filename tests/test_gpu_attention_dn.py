"""attn_kernel at every channel slice (dn = 64, 128, 256 output channels per CTA) against the fp64 reference of the fused kernel, at the
attention shapes the 16->128 engines run: 16x16 images (256 tokens, one image per attention batch) and two 8x8 images sharing a
128-token batch (block-diagonal mask), C = 512, at batches 16 and 4.

dn only decides which CTA computes which output columns; every column's S, P and P v are summed in the same order.  So the slice the
library picks (dn = 0) and every forced slice must give the same bits, and each must meet the fused kernel's bound."""
import pytest
import torch

pytestmark = pytest.mark.gpu

C = 512
# (batch, Lt, HW): the 16x16 level and the 8x8 mid block of a batch of images
SHAPES = [(16, 256, 256), (16, 128, 64), (4, 256, 256), (4, 128, 64)]


def operands(B, Lt, HW):
    nz = B * HW // Lt
    g = torch.Generator().manual_seed(B * 1000 + Lt + HW)
    q = 2.0 * torch.randn(nz, Lt, C, generator=g)      # logits with a spread of a few units after the 1/sqrt(C) scaling
    k = torch.randn(nz, Lt, C, generator=g)
    v = torch.randn(nz, Lt, C, generator=g)
    qk = torch.cat([q, k], dim=2).bfloat16()
    vb = v.bfloat16()
    return nz, qk, vb


@pytest.mark.parametrize("B,Lt,HW", SHAPES)
def test_every_channel_slice_matches_fp64_and_each_other(B, Lt, HW):
    from _attention_ref import check_fused
    from sr3_b200 import _native
    nz, qk, vb = operands(B, Lt, HW)
    qk_d = qk.reshape(nz * Lt, 2 * C).cuda()
    vT_d = vb.transpose(1, 2).contiguous().reshape(nz * C, Lt).cuda()
    picked = _native.attention_dn(nz, Lt, C)
    assert picked in (64, 128, 256)
    outs = {dn: _native.test_attention_dn(qk_d, vT_d, nz, Lt, HW, C, dn).cpu() for dn in (0, 64, 128, 256)}
    print(f"B={B} Lt={Lt} HW={HW}: the library picks dn={picked}")
    check_fused(outs[0].float().reshape(nz, Lt, C), qk, vb, Lt, HW, C)
    for dn in (64, 128, 256):
        check_fused(outs[dn].float().reshape(nz, Lt, C), qk, vb, Lt, HW, C)
        assert torch.equal(outs[dn], outs[0]), f"dn={dn} differs from dn={picked} (the library's pick)"
    assert torch.equal(_native.test_attention(qk_d, vT_d, nz, Lt, HW, C).cpu(), outs[0])


def test_unsupported_channel_slices_are_refused():
    from sr3_b200 import _native
    nz, qk, vb = operands(4, 256, 256)
    qk_d = qk.reshape(nz * 256, 2 * C).cuda()
    vT_d = vb.transpose(1, 2).contiguous().reshape(nz * C, 256).cuda()
    for dn in (32, 96, 512):
        with pytest.raises(RuntimeError, match="channel slice"):
            _native.test_attention_dn(qk_d, vT_d, nz, 256, 256, C, dn)

"""The channel slice of the fused attention kernel (output channels per CTA) the library picks per shape: the fewest waves of one CTA per
SM, then the narrowest slice.  Host logic only (sr3_attention_dn with an explicit SM count): no GPU needed."""
import pytest

H100_SMS = 132


@pytest.mark.parametrize("nz,Lt,C,dn", [
    (16, 256, 512, 128),   # 16->128 at batch 16, 16x16: 128 CTAs (256 would leave half the GPU idle at 64, 64 would need two waves)
    (8, 128, 512, 64),     # its 8x8 mid block, two images per 128-token batch: 64 CTAs
    (4, 256, 512, 64),     # batch 4, 16x16: 64 CTAs
    (2, 128, 512, 64),     # batch 4, 8x8: 16 CTAs
    (32, 256, 512, 256),   # unconditional 128x128 at batch 32, 16x16: 128 CTAs (128 would need two waves)
    (16, 128, 512, 64),    # its 8x8 mid block: 128 CTAs
    (64, 256, 512, 256),   # beyond one wave at any slice: the fewest waves
    (3, 256, 384, 64),     # C not a multiple of 256
    (1, 1024, 512, 128),   # above 256 keys the streaming kernel runs its fixed 128-channel slice
])
def test_picked_channel_slice(nz, Lt, C, dn):
    from sr3_b200 import _native
    assert _native.attention_dn(nz, Lt, C, H100_SMS) == dn

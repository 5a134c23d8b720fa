"""GPU parity of the single tensor-core tile kernel (wgmma + TMA) against fp32 torch references on CPU,
called through the C ABI (sr3_test_gemm / sr3_test_conv)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("M,N,K,bn", [(128, 64, 64, 64), (128, 128, 128, 128), (256, 256, 192, 256), (384, 128, 1024, 64),
                                      (1024, 512, 4608, 128), (128, 32, 576, 32), (512, 96, 640, 32)])
def test_gemm_matches_fp32(M, N, K, bn):
    """(The 16-wide tile exists only with the posterior epilogue of the final conv: covered by the p_mean_variance / p_sample tests.)"""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).bfloat16()
    b = torch.randn(N, K, generator=g).bfloat16()
    d = _native.test_gemm(a.cuda(), b.cuda(), bn).cpu()
    ref = a.float() @ b.float().t()
    assert rel(d, ref) < 2e-5, rel(d, ref)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,s", [
    (2, 16, 16, 64, 64, 1, 1), (2, 16, 16, 64, 64, 3, 1), (2, 8, 8, 128, 128, 3, 1), (1, 32, 32, 64, 128, 3, 1),
    (2, 32, 32, 192, 64, 3, 1), (2, 16, 16, 64, 64, 3, 2), (1, 64, 64, 128, 128, 3, 2), (2, 128, 128, 64, 64, 3, 1),
    (4, 8, 8, 512, 512, 3, 1), (2, 16, 16, 1024, 512, 1, 1)])
def test_conv_matches_fp32(B, H, W, Cin, Cout, k, s):
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(B + H * 3 + Cin * 5 + Cout * 7 + k + s)
    x = torch.randn(B, Cin, H, W, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, k, k, generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, generator=g)
    y, stats = _native.test_conv(x.permute(0, 2, 3, 1).contiguous().cuda(), w.cuda(), bias.cuda(), k, s, want_stats=True)
    y = y.cpu().permute(0, 3, 1, 2)
    ref = F.conv2d(x.float(), w.bfloat16().float(), bias, stride=s, padding=k // 2)
    assert y.shape == ref.shape
    assert rel(y, ref) < 2e-5, rel(y, ref)
    # GroupNorm partial sums accumulated by the epilogue
    st = stats.cpu()
    assert st.dtype == torch.float64
    assert torch.allclose(st[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=1e-3)
    assert torch.allclose(st[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("nz,Lt,HW,C", [(3, 256, 256, 512), (2, 128, 64, 512), (2, 256, 256, 128), (1, 128, 128, 256), (2, 256, 64, 256)])
def test_fused_attention_matches_fp32(nz, Lt, HW, C):
    """attn_kernel (S = q k^T / sqrt(C), softmax over the keys of the same image, O = P v; reference unet.py:129-139) against fp64 on the
    same bf16 operands, rounding P and O where the kernel does (tests/_attention_ref.py); the plain fp32 softmax and a reference without
    one key per segment must both miss the bound."""
    from _attention_ref import check_fused
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(nz * 1000 + Lt + HW + C)
    q = torch.randn(nz, Lt, C, generator=g)
    k = torch.randn(nz, Lt, C, generator=g)
    v = torch.randn(nz, Lt, C, generator=g)
    q = q * 2.0                                  # logits with a spread of a few units after the 1/sqrt(C) scaling
    qk = torch.cat([q, k], dim=2).bfloat16()
    vb = v.bfloat16()
    vT = vb.transpose(1, 2).contiguous()         # [nz, C, Lt]
    out = _native.test_attention(qk.reshape(nz * Lt, 2 * C).cuda(), vT.reshape(nz * C, Lt).cuda(), nz, Lt, HW, C).float().cpu().reshape(nz, Lt, C)
    check_fused(out, qk, vb, Lt, HW, C)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 8, 1024, 512), (2, 16, 16, 512, 512), (16, 8, 8, 512, 512)])
def test_split_k_conv_is_deterministic(B, H, W, Cin, Cout):
    """Few-tile / long-K convs run split-K: the partial tiles are summed in a fixed split order (no atomics on the output), so two
    launches on the same inputs must agree bit for bit -- and with the fp32 reference."""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(B * 11 + H + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (1.0 / (Cin * 9) ** 0.5)
    bias = torch.randn(Cout, generator=g)
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    y1, _ = _native.test_conv(xd, w.cuda(), bias.cuda(), 3, 1, want_stats=True)
    y2, _ = _native.test_conv(xd, w.cuda(), bias.cuda(), 3, 1, want_stats=True)
    assert torch.equal(y1, y2)
    ref = F.conv2d(x.float(), w.bfloat16().float(), bias, stride=1, padding=1)
    assert rel(y1.cpu().permute(0, 3, 1, 2), ref) < 2e-5


def dgrad_weights(w):
    """Weights W' such that conv3x3(dY, W', pad 1) = dL/dX of y = conv3x3(X, W, pad 1): W'[ci, co, r, s] = W[co, ci, 2-r, 2-s]."""
    return w.flip(2, 3).transpose(0, 1).contiguous()


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 64, 128), (1, 32, 32, 128, 64), (2, 8, 8, 512, 512)])
def test_conv_dgrad_is_the_forward_kernel_on_mirrored_weights(B, H, W, Cin, Cout):
    """Training row, data gradient of a stride-1 conv3x3: the same implicit-GEMM tile kernel run on dY with mirrored taps and
    Cin <-> Cout swapped (DESIGN.md 6.1), against torch autograd (fp32 on the same bf16-rounded operands)."""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(B * 3 + H + Cin * 7 + Cout)
    x = torch.randn(B, Cin, H, W, generator=g, requires_grad=True)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (1.0 / (Cin * 9) ** 0.5)).bfloat16().float()
    dy = torch.randn(B, Cout, H, W, generator=g).bfloat16()
    y = F.conv2d(x, w, None, padding=1)
    (dx_ref,) = torch.autograd.grad(y, x, dy.float())
    zero_bias = torch.zeros(Cin)
    dx, _ = _native.test_conv(dy.permute(0, 2, 3, 1).contiguous().cuda(), dgrad_weights(w).cuda(), zero_bias.cuda(), 3, 1, want_stats=True)
    assert rel(dx.cpu().permute(0, 3, 1, 2), dx_ref) < 2e-5


@pytest.mark.parametrize("B,H,W,Cin,Cout,groups,ratio", [(2, 32, 32, 64, 128, 32, 30.0), (2, 16, 16, 128, 64, 16, 30.0), (1, 64, 64, 64, 64, 32, 100.0),
                                                         (4, 8, 8, 64, 256, 32, 0.0)])
def test_groupnorm_is_cancellation_safe(B, H, W, Cin, Cout, groups, ratio):
    """GroupNorm statistics (reference nn.GroupNorm(groups, dim), eps 1e-5, unet.py:84,119) for activations whose |mean| / std is ~30-100
    and with non-trivial affine weights: the conv epilogue accumulates shifted sums, the totals are fp64 -- a one-pass fp32
    E[x^2] - mean^2 would lose the variance here.  Checked against fp32 torch GroupNorm of the same conv output."""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(B * 5 + H + Cout + int(ratio))
    x = torch.randn(B, Cin, H, W, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (1.0 / (Cin * 9) ** 0.5)          # conv output std ~ 1
    bias = ratio * (1.0 + 0.1 * torch.randn(Cout, generator=g)) * (torch.randint(0, 2, (Cout,), generator=g) * 2 - 1).float()
    gamma = 0.5 + torch.rand(Cout, generator=g)
    beta = torch.randn(Cout, generator=g)
    y, a = _native.test_conv_groupnorm(x.permute(0, 2, 3, 1).contiguous().cuda(), w.cuda(), bias.cuda(), gamma.cuda(), beta.cuda(), groups, True, 3)
    yr = F.conv2d(x.float(), w.bfloat16().float(), bias, padding=1)
    assert rel(y.cpu().permute(0, 3, 1, 2), yr) < 2e-5
    ref = F.silu(F.group_norm(yr.double(), groups, gamma.double(), beta.double(), eps=1e-5)).float()
    got = a.float().cpu().permute(0, 3, 1, 2)
    # bf16 output rounding alone is ~1.7e-3 relative L2; a lost variance shows up as percent-level errors
    assert rel(got, ref) < 3e-3, rel(got, ref)
    # and against an fp64 GroupNorm of OUR fp32 conv output the only error left is that rounding
    ref2 = F.silu(F.group_norm(y.cpu().permute(0, 3, 1, 2).double(), groups, gamma.double(), beta.double(), eps=1e-5)).float()
    assert rel(got, ref2) < 2.5e-3, rel(got, ref2)


def test_groupnorm_statistics_are_bit_reproducible():
    """fp64 atomics on contributions rounded to a multiple of 2^-20: every addition is exact, so the sums -- and everything computed
    from them -- do not depend on the order in which the CTAs arrive."""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(3)
    x = torch.randn(4, 64, 64, 64, generator=g).bfloat16().permute(0, 2, 3, 1).contiguous().cuda()
    w = (torch.randn(128, 64, 3, 3, generator=g) * 0.05).cuda()
    bias = torch.randn(128, generator=g).cuda()
    runs = [_native.test_conv(x, w, bias, 3, 1, want_stats=True) for _ in range(4)]
    for y, st in runs[1:]:
        assert torch.equal(y, runs[0][0]) and torch.equal(st, runs[0][1])

"""The weight-gradient kernel of the training path (wgrad_kernel + wgrad_reduce_kernel, train_kernels.cuh) against fp64 references on the
CPU, called through sr3_test_wgrad with the launch shape the training plan builds (wgrad_shape / wgrad_params in engine.cu).

dW[co][ci][r][s] = gscale * sum over images and output pixels of dY[co] X[ci] at the tap's input pixel.  Products of bf16 operands are
exact, each slice accumulates in fp32 over at most B*OH*OW <= 2048 pixels and the slices are summed in fp32: relative L2 below 2e-5 and
element-wise within 1e-4 (|ref| + rms(ref)) against torch.nn.grad.conv2d_weight in fp64 on the same bf16-rounded operands.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def check(got, ref, what):
    r = rel(got.double(), ref)
    assert r < 2e-5, f"{what}: relative L2 {r:.3e}"
    bad = ((got.double() - ref).abs() > 1e-4 * (ref.abs() + ref.pow(2).mean().sqrt())).nonzero()
    if bad.numel():
        idx = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} elements out of bound, first at {idx}: got {got[idx].item():.7g}, want {ref[idx].item():.7g}")


def operands(B, OH, OW, CY, Cin, stride, seed):
    g = torch.Generator().manual_seed(seed)
    dy = torch.randn(B, OH, OW, CY, generator=g).bfloat16()
    x = torch.randn(B, OH * stride, OW * stride, Cin, generator=g).bfloat16()
    return dy, x


def wgrad_ref(dy, x, k, stride, cout_valid, cin_valid, gscale):
    xd = x.double().permute(0, 3, 1, 2)[:, :cin_valid]
    dyd = dy.double().permute(0, 3, 1, 2)[:, :cout_valid]
    return gscale * torch.nn.grad.conv2d_weight(xd, (cout_valid, cin_valid, k, k), dyd, stride=stride, padding=k // 2)


CASES = [
    # B, OH, OW, CY, Cin, k, stride, cout_valid, cin_valid, slices, gscale
    (2, 8, 8, 128, 128, 3, 1, None, None, 0, 1.0),
    (2, 16, 16, 128, 64, 3, 1, None, None, 0, 0.37),
    (2, 32, 32, 64, 128, 3, 1, None, None, 0, 1.0),
    (2, 8, 8, 128, 128, 3, 2, None, None, 0, 1.0),             # Downsample: taps through the stride-2 parity view
    (2, 16, 16, 64, 64, 3, 2, None, None, 0, 2.0 ** -10),
    (2, 16, 16, 256, 128, 1, 1, None, None, 0, 1.0),           # 1x1 (res_conv, attention projections)
    (2, 16, 16, 64, 128, 3, 1, None, None, 0, 1.0),            # Cout 64: co_pad 128 > cout_valid
    (2, 16, 16, 64, 64, 3, 1, 3, None, 0, 1.0),                # final conv: 3 of 64 rows
    (2, 32, 32, 64, 64, 3, 1, None, 6, 0, 1.0),                # first conv: 6 of 64 input channels
    (3, 16, 16, 128, 64, 3, 1, None, None, 0, 1.0),            # odd batch
    (3, 16, 16, 128, 64, 3, 1, None, None, 1, 1.0),            # one slice
    (3, 16, 16, 128, 64, 3, 1, None, None, 5, 0.37),           # 12 patches / 5 slices: uneven, straddling images
    (3, 16, 16, 128, 64, 3, 1, None, None, 6, 1.0),            # two patches per slice, inside one image
    (3, 16, 16, 128, 64, 3, 1, None, None, 12, 1.0),           # one patch per slice
    (3, 8, 16, 64, 128, 3, 2, None, None, 3, 1.0),             # stride 2, slices straddling images
]


@pytest.mark.parametrize("B,OH,OW,CY,Cin,k,stride,cout_valid,cin_valid,slices,gscale", CASES)
def test_wgrad_matches_fp64(B, OH, OW, CY, Cin, k, stride, cout_valid, cin_valid, slices, gscale):
    from sr3_b200 import _native
    dy, x = operands(B, OH, OW, CY, Cin, stride, seed=B * 1000 + OH * 10 + CY + Cin + k + stride + slices)
    cv = CY if cout_valid is None else cout_valid
    civ = Cin if cin_valid is None else cin_valid
    got, used = _native.test_wgrad(dy.cuda(), x.cuda(), k, stride, cout_valid=cv, cin_valid=civ, slices=slices, gscale=gscale)
    patches = B * (OH // 8) * (OW // 8)
    if slices:
        assert used == slices
    assert 1 <= used <= patches, used
    check(got.cpu(), wgrad_ref(dy, x, k, stride, cv, civ, gscale), f"wgrad k={k} s={stride} {CY}x{Cin} slices={used}")


@pytest.mark.parametrize("nb,Lt,C", [(2, 128, 128), (3, 256, 128), (2, 128, 256)])
def test_wgrad_batched_form_matches_einsum(nb, Lt, C):
    """The attention backward's dK = dS^T Q and dV = P^T dO: batch b alone is contracted over its Lt query rows (viewed as Lt/16 x 16
    pixels) into out[b][key][c], one slice per batch and no reduction."""
    from sr3_b200 import _native
    g = torch.Generator().manual_seed(nb * 7 + Lt + C)
    dy = torch.randn(nb, Lt // 16, 16, Lt, generator=g).bfloat16()
    x = torch.randn(nb, Lt // 16, 16, C, generator=g).bfloat16()
    got, used = _native.test_wgrad(dy.cuda(), x.cuda(), 1, raw=True)
    assert used == nb
    ref = torch.einsum("bqk,bqc->bkc", dy.double().reshape(nb, Lt, Lt), x.double().reshape(nb, Lt, C))
    check(got.cpu(), ref, "batched wgrad")


def test_wgrad_is_bit_reproducible():
    """The slices are summed in a fixed order (DESIGN.md 3.6): two launches on the same inputs agree bit for bit."""
    from sr3_b200 import _native
    dy, x = operands(3, 16, 16, 128, 128, 1, seed=11)
    dy, x = dy.cuda(), x.cuda()
    a, used = _native.test_wgrad(dy, x, 3, 1, slices=5)
    b, _ = _native.test_wgrad(dy, x, 3, 1, slices=5)
    c, _ = _native.test_wgrad(dy, x, 3, 1)
    d, _ = _native.test_wgrad(dy, x, 3, 1)
    assert used == 5 and torch.equal(a, b) and torch.equal(c, d)

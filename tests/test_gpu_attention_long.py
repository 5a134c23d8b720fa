"""The streaming-softmax attention kernel (attn_long_wgmma.cuh, attn_long_kernel): self-attention over more than 256 tokens in one launch.

Kernel level, through sr3_test_attention on bf16 operands: against an fp64 reference that walks the key blocks and rounds where the kernel
rounds (tests/_attention_long_ref.py), against plain fp64 softmax attention with a bound derived from the two bf16 roundings alone, on rows
built to stress the running maximum, against the device's own three-launch path, and for bit reproducibility and batch independence.
Plan level: a bf16 inference engine runs every attention layer as one launch and allocates no token x token buffer; precise mode and the
training plan keep the three launches; the sized golden cases that attend over more than 256 tokens still match the reference."""
import math
import os

import pytest
import torch

import _attention_long_ref as lr
import _sizes_inputs as si
from _attention_ref import FUSED_TOL, rel

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
# (nz, Lt, C): 512 / 1024 tokens at the channel counts of the small and the 16->128 configs, the 32x32 mid block of 64->512 (C = 1024),
# the 16->128 config at 512x512 (4096 tokens), and 16 key blocks at one channel slice
SHAPES = [(2, 512, 128), (1, 512, 512), (3, 1024, 256), (1, 1024, 1024), (1, 4096, 512), (1, 2048, 128)]


def random_inputs(nz, Lt, C, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(nz, Lt, C, generator=g) for _ in range(3))
    return 2.0 * q, k, v                    # logits with a spread of a few units after the 1/sqrt(C) scaling


def run_fused(qk, vb):
    from sr3_b200 import _native
    nz, Lt, C = vb.shape
    out = _native.test_attention(qk.reshape(nz * Lt, 2 * C).cuda(), vb.transpose(1, 2).contiguous().reshape(nz * C, Lt).cuda(), nz, Lt, Lt, C)
    return out.float().cpu().reshape(nz, Lt, C)


def first_bad(ok):
    bad = (~ok).nonzero()
    if bad.numel() == 0:
        return ""
    z, r, c = bad[0].tolist()
    return f"{int((~ok).sum())} elements out of bounds, first at batch {z} row {r} channel {c}"


def check_against_streaming(out, qk, vb, C, what):
    """Relative L2 at the short kernel's bound, and element by element: one bf16 ulp of the output (the fp32 value and the fp64 one may
    round to neighbours) plus one bf16 ulp of every P~ (an fp32 exponential next to a rounding boundary goes the other way; one such
    key that holds much of a row's weight moves the row by most of 2^-8 p |v|)."""
    ref = lr.streaming_reference(qk, vb, C)
    p = torch.softmax(qk[..., :C].double() @ qk[..., C:].double().transpose(1, 2) / math.sqrt(C), -1)
    tol = 2.0 ** -7 * ref.abs() + 2.0 ** -8 * (p @ vb.double().abs())
    e = rel(out, ref)
    ok = (out.double() - ref).abs() <= tol
    print(f"{what}: rel L2 {e:.2e} (bound {FUSED_TOL:.0e}), max |d|/tol {((out.double() - ref).abs() / tol).max():.2e}")
    assert torch.isfinite(out).all()
    assert e < FUSED_TOL, e
    assert ok.all(), first_bad(ok)


@pytest.mark.parametrize("nz,Lt,C", SHAPES)
def test_long_attention_matches_streaming_reference(nz, Lt, C):
    qk, vb = lr.operands(*random_inputs(nz, Lt, C, nz * 1000 + Lt + C))
    check_against_streaming(run_fused(qk, vb), qk, vb, C, f"long attention nz={nz} Lt={Lt} C={C}")


@pytest.mark.parametrize("nz,Lt,C", SHAPES)
def test_long_attention_matches_plain_softmax(nz, Lt, C):
    """Plain fp64 softmax attention, nothing of the kernel's order in the reference.  P~ and the output are rounded to bf16 (2^-9 relative
    each), S carries the fp32 accumulation over C products (an absolute error d in S is a relative error <= 2 d in P), O the one over Lt."""
    qk, vb = lr.operands(*random_inputs(nz, Lt, C, nz * 1000 + Lt + C + 1))
    out = run_fused(qk, vb).double()
    q, k, v = qk[..., :C].double(), qk[..., C:].double(), vb.double()
    ref = lr.plain_reference(qk, vb, C)
    p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(C), -1)
    d_s = ((C + 2) * U32 * (q.abs() @ k.abs().transpose(1, 2)) / math.sqrt(C)).max().item()
    bound = ((2.0 ** -9 + 2 * d_s + (Lt + 2) * U32) * (p @ v.abs()).norm() / ref.norm() + 2.0 ** -9).item()
    e = rel(out, ref)
    print(f"long attention vs plain softmax nz={nz} Lt={Lt} C={C}: rel L2 {e:.2e} (derived bound {bound:.2e})")
    assert e < bound, (e, bound)


@pytest.mark.parametrize("kind", lr.ADVERSARIAL)
@pytest.mark.parametrize("Lt,C", [(512, 128), (1024, 256)])
def test_running_maximum_on_adversarial_rows(kind, Lt, C):
    qk, vb = lr.operands(*lr.adversarial(kind, Lt, C, seed=Lt + C))
    check_against_streaming(run_fused(qk, vb), qk, vb, C, f"long attention on {kind} logits Lt={Lt} C={C}")


@pytest.mark.parametrize("nz,Lt,C", [(1, 512, 512), (3, 1024, 256), (1, 1024, 1024), (1, 4096, 512)])
def test_long_attention_matches_three_launches(nz, Lt, C):
    from sr3_b200 import _native
    qk, vb = lr.operands(*random_inputs(nz, Lt, C, 77 + nz + Lt + C))
    out = run_fused(qk, vb)
    _, _, O = _native.test_attention_unfused(qk.reshape(nz * Lt, 2 * C).cuda(), vb.transpose(1, 2).contiguous().reshape(nz * C, Lt).cuda(),
                                             nz, Lt, Lt, C)
    # the three launches round the normalised P to bf16, the fused kernel the unnormalised P~: two independent roundings of 2^-9 each
    # (measured 2.9e-3 on an H100 at every shape of tools/gpu_attention_bench.py)
    e = rel(out, O.float().cpu().reshape(nz, Lt, C))
    print(f"long attention vs three launches nz={nz} Lt={Lt} C={C}: rel L2 {e:.2e} (bound 5e-3)")
    assert e < 5e-3, e


@pytest.mark.parametrize("nz,Lt,C", [(3, 512, 256), (5, 1024, 128)])
def test_repeat_launches_and_batches_are_independent(nz, Lt, C):
    q, k, v = random_inputs(nz, Lt, C, 5 + nz)
    qk, vb = lr.operands(q, k, v)
    a, b = run_fused(qk, vb), run_fused(qk, vb)
    assert torch.equal(a, b)
    k2, v2 = k.clone(), v.clone()
    k2[1], v2[1] = -3.0 * k[1], v[1] + 1.0
    qk2, vb2 = lr.operands(q, k2, v2)
    c = run_fused(qk2, vb2)
    assert not torch.equal(c[1], a[1])
    for z in range(nz):
        if z != 1:
            assert torch.equal(c[z], a[z]), z


# ---------------------------------------------------------------------------------------------------------------- plan / UNet level
def make_opt(unet, image_size, sched):
    return {"phase": "val", "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}


def build(unet, image_size, seed, sched=si.SCHED, precision="bf16"):
    import sr3_b200
    torch.manual_seed(seed)
    net = sr3_b200.define_G(make_opt(dict(unet, precision=precision), image_size, sched)).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


@pytest.fixture(scope="module")
def sizes():
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sr3_sizes_golden.pt"), map_location="cpu",
                      weights_only=False)


def kinds_of(eng):
    return [k for k, _, _, _ in eng.profile_step(5, reps=1)]


@pytest.mark.parametrize("h,w", [(32, 64), (64, 64)])
def test_plan_runs_long_attention_as_one_launch(h, w):
    """512 (32x64) and 1024 (64x64) tokens on the small config: the bf16 inference plan has one fused launch per attention layer and no
    softmax launch; precise mode and the training plan keep S / softmax / P v."""
    B = 2
    engines = {}
    for precision in ("bf16", "fp32"):
        engines[precision] = build(si.TINY, 32, 0, precision=precision).denoise_fn.engine(B, height=h, width=w)
    net = build(si.TINY, 32, 0)
    train = net.denoise_fn.engine(B, train_dropout=0.0, height=h, width=w)
    g = torch.Generator().manual_seed(1)
    hr, sr, noise = (torch.randn(B, 3, h, w, generator=g).cuda() for _ in range(3))
    train.train_forward(hr, sr, torch.tensor([0.7, 0.4]), noise, "l1", 1, want_loss=False)
    kinds = {name: kinds_of(e) for name, e in (("bf16", engines["bf16"]), ("fp32", engines["fp32"]), ("train", train))}
    layers = kinds["fp32"].count(3)
    assert layers > 0 and kinds["fp32"].count(5) == 0
    assert kinds["bf16"].count(5) == layers and kinds["bf16"].count(3) == 0
    assert kinds["train"].count(3) == layers and kinds["train"].count(5) == 0
    assert len(kinds["bf16"]) == len(kinds["fp32"]) - 2 * layers
    for e in engines.values():
        assert e.ops_per_step() == e.launches_per_step()


def test_workspace_holds_no_token_matrix():
    """The small config at 256x256: 128x128 = 16384 tokens per image on its attention level.  S (fp32) and P (bf16) would take
    6 nz Lt^2 bytes, several times everything else the plan holds, so a plan that allocates neither is smaller than they alone would
    be.  The forward over 128 key blocks is finite and repeats bit for bit."""
    B, h, w = 1, 256, 256
    Lt, nz = (h // 2) * (w // 2), 2                      # image slots are padded to a multiple of two
    net = build(si.TINY, 32, 0)
    eng = net.denoise_fn.engine(B, height=h, width=w)
    print(f"workspace at {h}x{w}, batch {B}: {eng.workspace_bytes()} bytes; S + P would be {6 * nz * Lt * Lt}")
    assert eng.workspace_bytes() < 6 * nz * Lt * Lt
    g = torch.Generator().manual_seed(2)
    x, nl = torch.randn(B, 6, h, w, generator=g).cuda(), torch.tensor([[0.5]]).cuda()
    a, b = net.denoise_fn(x, nl), net.denoise_fn(x, nl)
    assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["tiny_32x64", "tiny_64x32", "tiny_64x64", "sr16_64_128x128", "full_128x256"])
def test_sized_golden_cases_over_256_tokens(sizes, name):
    """eps and the attention layers' outputs of every sized golden case that attends over more than 256 tokens, at the bounds of
    tests/test_gpu_sizes.py."""
    unet, image_size, seed, b, h, w = si.CASES[name][:6]
    g, inp = sizes[name], si.inputs(name)
    net = build(unet, image_size, g["seed"])
    eps = net.denoise_fn(inp["x"].cuda(), inp["noise_level"].cuda())
    eng = net.denoise_fn.engine(b, height=h, width=w)
    deep = len(unet["channel_multiplier"]) == 5
    errs = {layer: rel(si.tap_crop(name, layer, eng.read_activation(layer)).cpu(), ref) for layer, ref in g["taps"].items()}
    e_eps = rel(si.eps_crop(name, eps).cpu(), g["eps"])
    kinds = kinds_of(eng)                              # (an eager step of its own: after the activations were read)
    assert 5 in kinds and 3 not in kinds
    print(f"{name} rel err: eps {e_eps:.2e},", {k: f"{v:.2e}" for k, v in errs.items()})
    assert torch.isfinite(eps).all() and e_eps < 1e-2, e_eps
    for layer, e in errs.items():
        assert e < (2e-2 if deep else 1e-2), (layer, e)


@pytest.mark.timeout(900)
def test_128x256_is_bit_reproducible(sizes):
    """unet_forward and the 10-step loop with injected noise on the 16->128 config at 128x256 (512 tokens at C = 512): same bits twice."""
    name = si.LOOP_CASE
    unet, image_size = si.CASES[name][:2]
    inp, d = si.inputs(name), si.loop_inputs()
    net = build(unet, image_size, sizes[name]["seed"])
    x, nl = inp["x"].cuda(), inp["noise_level"].cuda()
    assert torch.equal(net.denoise_fn(x, nl), net.denoise_fn(x, nl))
    net.set_new_noise_schedule(si.SCHED10, "cuda")
    runs = [net.super_resolution(inp["cond"].cuda(), continous=True, x_T=d["x_T"].cuda(), noises=d["noises"].cuda()).cpu() for _ in range(2)]
    assert torch.isfinite(runs[0]).all() and torch.equal(runs[0], runs[1])

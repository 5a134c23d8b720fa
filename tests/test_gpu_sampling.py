"""The sampling step's own kernels against exact references: the posterior update of the final conv's epilogue (bit for bit), the Gaussian
noise it draws with Philox4x32-10 + Box-Muller (tests/_philox.py restates the stream; tests/test_sampling_noise.py checks the restatement's
statistics), the hand-off of x_{t-1} into the next step's input, and the noise-level embedding + FiLM projections at every batch size."""
import math

import numpy as np
import pytest
import torch

import _philox
import _sizes_inputs as si
from oracle import sr3_oracle as orc

pytestmark = pytest.mark.gpu

KNOBS = ("SR3_TALL_BN", "SR3_TALL_MH", "SR3_BLOCK_N", "SR3_KSPLIT", "SR3_STAGES", "SR3_PINGPONG", "SR3_MAX_CTAS")
SEED = 2 ** 62 + 0x1234_5678_9ABC          # both key words set
FIRST = 2 ** 32 - 2                        # batch 3: sample indices 2^32 - 2, 2^32 - 1, 2^32 (the high word of the index changes)
B = 3
SIZES = [(32, 32), (32, 64), (64, 32), (64, 64)]
MODES = ["graph"]
PRECISIONS = ["bf16", "fp32"]


def make_opt(unet, image_size, sched):
    return {"phase": "val", "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": True}}}


def build(monkeypatch, precision, sched, unet=si.TINY, image_size=32, seed=0):
    import sr3_b200
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    torch.manual_seed(seed)
    net = sr3_b200.define_G(make_opt(dict(unet, precision=precision), image_size, sched)).cuda()
    net.set_new_noise_schedule(sched, "cuda")
    net.eval()
    return net


def data(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, h, w, generator=g) * 2 - 1, torch.randn(B, 3, h, w, generator=g)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("h,w", SIZES)
def test_posterior_mean_bit_for_bit(monkeypatch, h, w, precision, mode):
    """predict_start_from_noise, clamp and q_posterior in torch-CPU fp32 on the eps unet_forward returns at the step's noise level equal the
    device's p_mean_variance mean bit for bit: the epilogue rounds every product and sum separately, as torch does."""
    net = build(monkeypatch, precision, si.SCHED)
    sch = orc.make_schedule(si.SCHED)
    T = sch.num_timesteps
    cond, x_t = data(h, w, h + w)
    eng = net._engine(B, h, w)
    for t in (T - 1, T // 2, 1, 0):
        eps = eng.unet_forward(torch.cat([cond, x_t], 1), orc.noise_level_for_t(sch, t, B)).cpu()
        for clip in (True, False):
            mean, lv = eng.p_mean_variance(x_t, t, clip, cond)
            x0 = orc.predict_start_from_noise(sch, x_t, t, eps)
            if clip:
                x0 = x0.clamp(-1.0, 1.0)
            ref, ref_lv = orc.q_posterior(sch, x0, x_t, t)
            diff = (mean.cpu() != ref).sum().item()
            assert diff == 0, f"t={t} clip={clip}: {diff} of {ref.numel()} means differ, max |d| {(mean.cpu() - ref).abs().max().item():.3e}"
            assert lv == float(ref_lv)


def _noise_bound(mean, z, sigma):
    """|x - (mean + z sigma)| with x = fl(mean + fl(z' sigma')): z' carries the errors of logf (1 ulp), sqrtf (0.5), sincospif (1) and two
    fp32 products, sigma' those of expf (2 ulp) and the product (0.5), and the sum rounds once more (0.5 ulp of |x| <= 2^-24 (|mean| +
    |z sigma|)): about 6 ulp of |z sigma| and one of |mean|, bounded by 1e-6 (16.8 fp32 ulp) of each."""
    return 1e-6 * (np.abs(mean) + sigma * np.abs(z)) + 1e-30


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("h,w", SIZES)
def test_seeded_noise_is_the_documented_stream(monkeypatch, h, w, precision, mode):
    """p_sample(seed, first_index) = mean + sampling_noise(...) exp(0.5 logvar) within the ulp bound of the device's logf / sincospif / expf,
    with a seed >= 2^62 and a batch that crosses the sample index's high-word boundary.  The bound is tight: the restatement with any
    counter word off by one, or with the seed's words swapped, misses it by orders of magnitude.  At t = 0 x is the mean, bit for bit."""
    net = build(monkeypatch, precision, si.SCHED)
    sch = orc.make_schedule(si.SCHED)
    T = sch.num_timesteps
    cond, x_t = data(h, w, 7 * h + w)
    eng = net._engine(B, h, w)
    idx = FIRST + np.arange(B, dtype=np.uint64)
    wrong = {f"counter word {i} + 1": (lambda i: lambda *w: tuple(x + np.uint64(1) if j == i else x for j, x in enumerate(w)))(i)
             for i in range(4)}
    wrong["seed words swapped"] = lambda c0, c1, c2, c3, k0, k1: (c0, c1, c2, c3, k1, k0)
    for t in (T - 1, T // 2, 1):
        x = eng.p_sample(x_t, t, cond, None, SEED, FIRST).cpu().double().numpy()
        mean = eng.p_mean_variance(x_t, t, True, cond)[0].cpu().double().numpy()
        sigma = math.exp(0.5 * float(sch.buffers["posterior_log_variance_clipped"][t]))
        z = _philox.sampling_noise(SEED, idx, t, h, w)
        ratio = np.abs(x - (mean + z * sigma)) / _noise_bound(mean, z, sigma)
        print(f"{h}x{w} {precision} {mode} t={t}: max |x - ref| / bound = {ratio.max():.3f}")
        assert ratio.max() <= 1.0, (t, ratio.max())
        for name, fn in wrong.items():
            zw = _philox.sampling_noise(SEED, idx, t, h, w, words=fn)
            rw = np.median(np.abs(x - (mean + zw * sigma)) / _noise_bound(mean, zw, sigma))
            assert rw > 1e3, (t, name, rw)
    x0 = eng.p_sample(x_t, 0, cond, None, SEED, FIRST)
    assert torch.equal(x0, eng.p_mean_variance(x_t, 0, True, cond)[0])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("h,w", SIZES)
def test_loop_is_its_steps(monkeypatch, h, w, precision, mode):
    """p_sample_loop(seed, first_index) over a 10-step schedule equals p_sample(seed, first_index) chained from x_T, bit for bit at every
    snapshot: the loop hands x_{t-1} (and in precise mode its low half) to the next step's input exactly as a fresh load does, and keys
    the noise with the step's own t."""
    net = build(monkeypatch, precision, si.SCHED10)
    cond, x_T = data(h, w, 11 * h + w)
    eng = net._engine(B, h, w)
    final, snaps = eng.p_sample_loop(cond, x_T, None, SEED, FIRST, want_snapshots=True)
    assert snaps.shape[0] == 10
    x = x_T.cuda()
    for t in range(9, -1, -1):
        x = eng.p_sample(x, t, cond, None, SEED, FIRST)
        assert torch.equal(snaps[9 - t], x), f"step t={t}: {(snaps[9 - t] != x).sum().item()} values differ"
    assert torch.equal(final, x)


# ------------------------------------------------------------------------------------------------ noise-level embedding + FiLM
def film_params(inner, F, seed):
    g = torch.Generator().manual_seed(seed)
    hid = 4 * inner
    return {"noise_level_mlp.1.weight": torch.randn(hid, inner, generator=g) / math.sqrt(inner),
            "noise_level_mlp.1.bias": torch.randn(hid, generator=g) * 0.1,
            "noise_level_mlp.3.weight": torch.randn(inner, hid, generator=g) / math.sqrt(hid),
            "noise_level_mlp.3.bias": torch.randn(inner, generator=g) * 0.1,
            "wf": torch.randn(F, inner, generator=g) / math.sqrt(inner), "bf": torch.randn(F, generator=g) * 0.1,
            "cb": torch.randn(F, generator=g) * 0.1}


LEVELS = {"0": 0.0, "1e-4": 1e-4, "0.5": 0.5, "1": 1.0}


@pytest.mark.parametrize("inner", [32, 64, 128])
@pytest.mark.parametrize("batch", [1, 3, 31, 32, 127, 128, 129, 300])
def test_embedding_and_film_forward_match_fp64(batch, inner):
    """embed_kernel + film_kernel as the plan launches them against fp64 oracle.positional_encoding / noise_level_mlp and the FiLM linear
    plus the folded block1 conv bias, element-wise within 1e-5 of the sum of |terms| (the scale of fp32 accumulation error) -- at batches on
    both sides of film_kernel's staging chunk (31 images at inner 128, 127 at inner 64) and far beyond it."""
    from sr3_b200 import _native
    F = 448 + 24                            # not a multiple of film_kernel's 64 outputs per block
    p = film_params(inner, F, batch * 7 + inner)
    dev = {k: v.cuda() for k, v in p.items()}
    g = torch.Generator().manual_seed(batch)
    cases = {name: torch.full((batch,), v) for name, v in LEVELS.items()}
    cases["per image"] = torch.rand(batch, generator=g)
    sd = {k: v.double() for k, v in p.items()}
    for name, nl in cases.items():
        tau, film = _native.test_film_embed_fwd(nl.cuda(), dev["noise_level_mlp.1.weight"], dev["noise_level_mlp.1.bias"],
                                                dev["noise_level_mlp.3.weight"], dev["noise_level_mlp.3.bias"], dev["wf"], dev["bf"], dev["cb"])
        nl64 = nl.double().view(-1, 1)
        pe = orc.positional_encoding(nl64, inner).view(batch, inner)
        h = orc.swish(pe @ sd["noise_level_mlp.1.weight"].t() + sd["noise_level_mlp.1.bias"])
        tau_ref = orc.noise_level_mlp(sd, nl64, inner).view(batch, inner)
        tau_abs = h.abs() @ sd["noise_level_mlp.3.weight"].abs().t() + sd["noise_level_mlp.3.bias"].abs()
        film_ref = tau_ref @ sd["wf"].t() + sd["bf"] + sd["cb"]
        film_abs = tau_ref.abs() @ sd["wf"].abs().t() + sd["bf"].abs() + sd["cb"].abs()
        et = ((tau.cpu().double() - tau_ref).abs() / tau_abs).max().item()
        ef = ((film.cpu().double() - film_ref).abs() / film_abs).max().item()
        print(f"B={batch} inner={inner} nl={name}: max |d tau| / sum|terms| {et:.2e}, max |d film| / sum|terms| {ef:.2e} (bound 1e-5)")
        assert et < 1e-5 and ef < 1e-5, (name, et, ef)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("inner,batch", [(128, 32), (64, 128)])
def test_film_at_large_batch(monkeypatch, inner, batch):
    """A batch whose embeddings do not fit film_kernel's shared memory at once (inner_channel 128 at 32 images, 64 at 128) runs: eps
    matches the same images through a batch-2 engine within the bf16 tolerance."""
    unet = dict(in_channel=6, out_channel=3, inner_channel=inner, channel_multiplier=[1, 2], attn_res=[8], res_blocks=1, dropout=0.0)
    g = torch.Generator().manual_seed(inner + batch)
    x = torch.randn(batch, 6, 16, 16, generator=g)
    nl = torch.rand(batch, 1, generator=g)
    net = build(monkeypatch, "bf16", si.SCHED10, unet=unet, image_size=16)
    eps = net.denoise_fn(x.cuda(), nl.cuda()).cpu()
    pairs = torch.cat([net.denoise_fn(x[i:i + 2].cuda(), nl[i:i + 2].cuda()).cpu() for i in range(0, batch, 2)])
    e = ((eps - pairs).norm() / pairs.norm()).item()
    print(f"inner {inner} batch {batch}: eps vs batch-2 engines rel L2 {e:.2e} (bound 1e-2)")
    assert torch.isfinite(eps).all()
    assert e < 1e-2, e


def test_per_layer_path_runs_a_batch_of_448(monkeypatch):
    """At inner_channel 128 a batch of 448, far beyond one chunk of film_kernel's tau staging (31 images), builds and runs: eps is finite."""
    unet = dict(in_channel=6, out_channel=3, inner_channel=128, channel_multiplier=[1, 2], attn_res=[8], res_blocks=1, dropout=0.0)
    x, nl = torch.zeros(448, 6, 16, 16).cuda(), torch.full((448, 1), 0.5).cuda()
    net = build(monkeypatch, "bf16", si.SCHED10, unet=unet, image_size=16)
    assert torch.isfinite(net.denoise_fn(x, nl)).all()

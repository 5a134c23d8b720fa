"""Drop-in check at the boundary SURVEY.md 8b names: the UNMODIFIED reference wrapper (model/model.py `DDPM`, created through
`model.create_model(opt)`) is run with `model.networks.define_G` replaced by `sr3_b200.define_G` -- the one-line change INTEGRATION.md
describes.  Everything the wrapper does with netG short of GPU compute is exercised here on CPU: construction, set_device, set_loss,
set_new_noise_schedule (both phases), print_network, the Adam optimizer over our parameters, save_network / load_network with the
reference's file naming and strict key matching, and a checkpoint written by the reference's own netG.

Needs the reference sources: /root/reference in the build container, or the verbatim copy oracle/build_ref.py puts into the
git-ignored oracle/_ref (that copy travels to the GPU box, so the `gpu` test below -- the unmodified `DDPM.test()` / `DDPM.sample()`
of model/model.py:60-78 driving our native sampler on an H100 -- runs there)."""
import os
import sys

import pytest
import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("SR3_REFERENCE", "/root/reference")
if not os.path.isdir(os.path.join(REF, "model")):
    REF = os.path.join(_ROOT, "oracle", "_ref")
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "model")), reason="reference sources not present")

SCHED = {"schedule": "linear", "n_timestep": 20, "linear_start": 1e-6, "linear_end": 1e-2}
TINY = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2], attn_res=[16], res_blocks=1, dropout=0.0)


def make_opt(phase, ckpt_dir, resume=None):
    return {"phase": phase, "gpu_ids": None, "distributed": False,
            "path": {"checkpoint": ckpt_dir, "resume_state": resume},
            "train": {"optimizer": {"type": "adam", "lr": 1e-4}},
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(TINY),
                      "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                      "diffusion": {"image_size": 32, "channels": 3, "conditional": True}}}


@pytest.fixture()
def ref_model_pkg(monkeypatch):
    """The reference's `model` package with define_G swapped for ours (and restored afterwards)."""
    sys.dont_write_bytecode = True
    monkeypatch.syspath_prepend(REF)
    for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
        monkeypatch.delitem(sys.modules, k)
    import model as ref_model                      # /root/reference/model/__init__.py
    import model.networks as ref_networks
    import sr3_b200
    orig = ref_networks.define_G
    monkeypatch.setattr(ref_networks, "define_G", sr3_b200.define_G)
    yield ref_model, ref_networks, orig
    for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
        sys.modules.pop(k, None)


def test_reference_ddpm_wrapper_runs_on_our_define_g(ref_model_pkg, tmp_path):
    ref_model, ref_networks, orig_define_G = ref_model_pkg
    import sr3_b200
    torch.manual_seed(0)
    m = ref_model.create_model(make_opt("train", str(tmp_path)))
    assert type(m.netG).__name__ == "GaussianDiffusion" and isinstance(m.netG, sr3_b200.GaussianDiffusion)
    s, n = m.get_network_description(m.netG)
    assert n == sum(p.numel() for p in m.netG.parameters()) and "GaussianDiffusion" in s
    assert len(m.optG.param_groups[0]["params"]) == len(list(m.netG.parameters()))
    # phase switch as sr.py does (sr.py:110-111,146-147)
    m.set_new_noise_schedule(make_opt("val", "")["model"]["beta_schedule"]["val"], schedule_phase="val")
    assert m.netG.num_timesteps == SCHED["n_timestep"] and m.netG.betas.device.type == "cpu"
    # checkpoint round trip with the reference's naming (model.py:124-166)
    m.save_network(epoch=3, iter_step=70)
    gen, optp = tmp_path / "I70_E3_gen.pth", tmp_path / "I70_E3_opt.pth"
    assert gen.exists() and optp.exists()
    torch.manual_seed(1)                                          # different init, then resume
    m2 = ref_model.create_model(make_opt("train", str(tmp_path), resume=str(tmp_path / "I70_E3")))
    assert m2.begin_step == 70 and m2.begin_epoch == 3
    for (k1, v1), (k2, v2) in zip(m.netG.state_dict().items(), m2.netG.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2), k1
    # a checkpoint written by the reference's OWN network loads strictly into ours, and the other way round
    torch.manual_seed(2)
    ref_net = orig_define_G(make_opt("val", ""))
    ref_net.set_new_noise_schedule(SCHED, "cpu")                  # as DDPM.__init__ does before any save (model.py:21-22)
    torch.save(ref_net.state_dict(), tmp_path / "I1_E1_gen.pth")
    m3 = ref_model.create_model(make_opt("val", str(tmp_path), resume=str(tmp_path / "I1_E1")))
    for k, v in ref_net.state_dict().items():
        assert torch.equal(m3.netG.state_dict()[k], v), k
    ref_net.load_state_dict(m.netG.state_dict(), strict=True)


@pytest.mark.gpu
def test_reference_ddpm_wrapper_samples_on_the_gpu(ref_model_pkg, tmp_path):
    """model/model.py:60-78,98-110 unmodified: feed_data -> test(continous) -> get_current_visuals, and sample(), with netG = our define_G
    on cuda:0; then the reference's own tensor2img (core/metrics.py:8-34) on the visuals."""
    ref_model, ref_networks, _ = ref_model_pkg
    import numpy as np
    opt = make_opt("val", str(tmp_path))
    opt["gpu_ids"] = [0]
    torch.manual_seed(0)
    m = ref_model.create_model(opt)
    assert m.device.type == "cuda" and next(m.netG.parameters()).is_cuda
    m.set_new_noise_schedule(opt["model"]["beta_schedule"]["val"], schedule_phase="val")
    g = torch.Generator().manual_seed(3)
    data = {"HR": torch.rand(2, 3, 32, 32, generator=g) * 2 - 1, "SR": torch.rand(2, 3, 32, 32, generator=g) * 2 - 1, "Index": torch.arange(2)}
    m.feed_data(data)
    m.test(continous=True)
    vis = m.get_current_visuals()
    n_snap = len([i for i in range(SCHED["n_timestep"]) if i % (1 | (SCHED["n_timestep"] // 10)) == 0])
    assert vis["SR"].shape == (2 * (1 + n_snap), 3, 32, 32) and vis["SR"].device.type == "cpu" and torch.isfinite(vis["SR"]).all()
    # (feed_data moved the entries of `data` to the GPU in place: base_model.py:29-40)
    assert torch.equal(vis["SR"][:2], data["SR"].cpu()) and torch.equal(vis["INF"], data["SR"].cpu()) and torch.equal(vis["HR"], data["HR"].cpu())
    m.test(continous=False)
    last = m.get_current_visuals()["SR"]
    assert last.shape == (3, 32, 32) and torch.isfinite(last).all()       # the reference returns ret_img[-1]: the last image only (diffusion.py:198-200)
    # tensor2img of the reference (core/metrics.py:8-34: clamp to [-1,1] -> [0,255] uint8 HWC), restated here because core/metrics.py
    # imports cv2, which this image does not have
    img = ((last.clamp(-1, 1) + 1) / 2 * 255.0).round().permute(1, 2, 0).numpy().astype(np.uint8)
    assert img.shape == (32, 32, 3) and img.dtype == np.uint8


@pytest.mark.gpu
def test_reference_optimize_parameters_trains_on_the_gpu(ref_model_pkg, tmp_path):
    """model/model.py:48-58 UNMODIFIED (zero_grad -> netG(data) -> sum / (b c h w) -> backward -> torch.optim.Adam.step) over
    sr3_b200.define_G: the loss carries our native backward as its grad_fn, every parameter receives a gradient, the parameters move and the
    loss of a fixed batch goes down over a few iterations."""
    ref_model, ref_networks, _ = ref_model_pkg
    import numpy as np
    opt = make_opt("train", str(tmp_path))
    opt["gpu_ids"] = [0]
    opt["model"]["unet"]["dropout"] = 0.2
    torch.manual_seed(0)
    np.random.seed(0)
    m = ref_model.create_model(opt)
    assert m.device.type == "cuda" and m.netG.training
    before = {k: v.detach().clone() for k, v in m.netG.state_dict().items() if k.startswith("denoise_fn.")}
    g = torch.Generator().manual_seed(3)
    losses = []
    for it in range(6):
        data = {"HR": torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(3)) * 2 - 1,
                "SR": torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(4)) * 2 - 1, "Index": torch.arange(2)}
        m.feed_data(data)
        np.random.seed(1)                          # the same (t, gamma) draw every iteration: the loss of this batch must go down
        torch.manual_seed(1)
        m.optimize_parameters()
        losses.append(m.get_current_log()["l_pix"])
        if it == 0:
            missing = [k for k, p in m.netG.named_parameters() if p.grad is None or not torch.isfinite(p.grad).all() or p.grad.abs().sum() == 0]
            assert not missing, missing[:5]
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < losses[0], losses
    moved = sum(int(not torch.equal(before[k], v)) for k, v in m.netG.state_dict().items() if k in before)
    assert moved == len(before)

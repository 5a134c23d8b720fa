"""Shared by tests/test_gpu_train.py and tools/gpu_train_check.py: one training forward / backward of sr3_b200 on the GPU next to the oracle's
autograd on the CPU, per-parameter relative errors in backward order."""
import numpy as np
import torch

from oracle import sr3_oracle as orc

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}


def make_opt(unet, image_size, conditional=True, phase="train", sched=SCHED):
    return {"phase": phase, "gpu_ids": [0], "distributed": False,
            "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(unet),
                      "beta_schedule": {"train": dict(sched), "val": dict(sched)},
                      "diffusion": {"image_size": image_size, "channels": 3, "conditional": conditional}}}


def build_train_net(unet, image_size, seed, loss_type="l1", sched=SCHED, conditional=True):
    import sr3_b200
    torch.manual_seed(seed)
    net = sr3_b200.define_G(make_opt(unet, image_size, conditional, "train", sched)).cuda()      # phase 'train': orthogonal init (networks.py:110-112)
    net.loss_type = loss_type
    net.set_loss("cuda")
    net.set_new_noise_schedule(sched, "cuda")
    return net


def oracle_cfg(unet, image_size):
    return orc.UNetConfig(in_channel=unet["in_channel"], out_channel=unet["out_channel"], inner_channel=unet["inner_channel"],
                          norm_groups=unet.get("norm_groups", 32),
                          channel_mults=tuple(unet["channel_multiplier"]), attn_res=tuple(unet["attn_res"]), res_blocks=unet["res_blocks"],
                          dropout=unet["dropout"], image_size=image_size)


def batch(B, R, seed):
    gen = torch.Generator().manual_seed(seed)
    hr = torch.rand(B, 3, R, R, generator=gen) * 2 - 1
    sr = torch.rand(B, 3, R, R, generator=gen) * 2 - 1
    noise = torch.randn(B, 3, R, R, generator=gen)
    return hr, sr, noise


def rel(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cosine(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-30)).item()


def ours_loss_and_grads(net, hr, sr, gamma, noise, train_mode=False, dropout_seed=0):
    """One reference-style iteration head (model.py:48-53): l = netG(data).sum() / (b c h w); l.backward().  Returns (summed loss, grads)."""
    net.train(train_mode)
    for p in net.parameters():
        p.grad = None
    b, c, h, w = hr.shape
    x_in = {"HR": hr.cuda(), "SR": sr.cuda()} if net.conditional else {"HR": hr.cuda()}
    l = net.p_losses(x_in, noise=noise.cuda(), gamma=gamma, dropout_seed=dropout_seed)
    (l.sum() / int(b * c * h * w)).backward()
    grads = {k[len("denoise_fn."):]: p.grad.detach().clone() for k, p in net.named_parameters()}
    return float(l.item()), grads


def oracle_loss_and_grads(net, unet, image_size, hr, sr, gamma, noise, loss_type, dropout_masks=None):
    cfg = oracle_cfg(unet, image_size)
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in net.denoise_fn.state_dict().items()}
    sch = orc.make_schedule(SCHED)
    loss = orc.train_loss(sd, cfg, sch, hr, sr if net.conditional else None, gamma, noise, loss_type, dropout_masks)
    loss.backward()
    b, c, h, w = hr.shape
    return float(loss.item()) * b * c * h * w, {k: v.grad for k, v in sd.items()}


def compare(ours, ref):
    """[(name, rel err, cosine, |ref|)] in state_dict order."""
    rows = []
    for k in ref:
        rows.append((k, rel(ours[k], ref[k]), cosine(ours[k], ref[k]), float(ref[k].norm())))
    return rows


def draw_gamma(B, seed):
    sch = orc.make_schedule(SCHED)
    _, g = orc.draw_gamma(sch, B, np.random.RandomState(seed))
    return g

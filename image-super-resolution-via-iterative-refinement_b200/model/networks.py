"""Drop-in for the reference's model/networks.py:83-116 `define_G(opt)`: same `opt` schema in, an nn.Module with the
reference's methods, attributes and state_dict layout out."""
import logging
import os

import torch
from torch import nn

logger = logging.getLogger("base")


def init_weights(net, init_type="orthogonal", scale=1, std=0.02):
    """Only the initialiser define_G actually uses (networks.py:110-112) is provided."""
    logger.info("Initialization method [{:s}]".format(init_type))
    if init_type != "orthogonal":
        raise NotImplementedError("initialization method [{:s}] not implemented".format(init_type))
    net.denoise_fn.init_orthogonal()


def define_G(opt):
    model_opt = opt["model"]
    if model_opt["which_model_G"] != "sr3":
        raise NotImplementedError("sr3_b200 covers which_model_G == 'sr3' (the path BASELINE.json names); got %r" % (model_opt["which_model_G"],))
    from .sr3_modules import diffusion, unet
    if ("norm_groups" not in model_opt["unet"]) or model_opt["unet"]["norm_groups"] is None:
        model_opt["unet"]["norm_groups"] = 32
    model = unet.UNet(
        in_channel=model_opt["unet"]["in_channel"], out_channel=model_opt["unet"]["out_channel"],
        norm_groups=model_opt["unet"]["norm_groups"], inner_channel=model_opt["unet"]["inner_channel"],
        channel_mults=model_opt["unet"]["channel_multiplier"], attn_res=model_opt["unet"]["attn_res"],
        res_blocks=model_opt["unet"]["res_blocks"], dropout=model_opt["unet"]["dropout"],
        image_size=model_opt["diffusion"]["image_size"],
        # not part of the reference's schema: optional opt['model']['unet']['precision'] in {"bf16", "fp32"} (or env SR3_PRECISION)
        precision=(model_opt["unet"].get("precision") if hasattr(model_opt["unet"], "get") else None) or os.environ.get("SR3_PRECISION", "bf16"))
    netG = diffusion.GaussianDiffusion(
        model, image_size=model_opt["diffusion"]["image_size"], channels=model_opt["diffusion"]["channels"], loss_type="l1",
        conditional=model_opt["diffusion"]["conditional"], schedule_opt=model_opt["beta_schedule"]["train"])
    if opt["phase"] == "train":
        init_weights(netG, init_type="orthogonal")
    if opt["gpu_ids"] and opt["distributed"]:
        # The reference wraps the net in nn.DataParallel here (networks.py:113-115).  DataParallel replicates nn.Modules per forward
        # call; a module that owns native engines (packed weights, TMA descriptors, a captured step graph) cannot be replicated that
        # way.  The multi-GPU path of this implementation is one process per GPU: sr3_b200.parallel (batch-sharded sampling over NCCL).
        raise NotImplementedError(
            "sr3_b200.define_G: opt['distributed']=True (nn.DataParallel) is not supported; run one process per GPU "
            "(torchrun) and use sr3_b200.parallel.sharded_super_resolution -- see INTEGRATION.md, 'Multi-GPU'")
    return netG

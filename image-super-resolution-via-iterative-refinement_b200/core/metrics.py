"""Device-side mirror of the pieces of the reference's core/metrics.py that sit on the sampling path's exit (sr.py / infer.py call them
on every snapshot and every evaluated image): `tensor2img` (core/metrics.py:8-34), `calculate_psnr` (:42-50), `ssim` and `calculate_ssim`
(:52-93).  Same signatures and results; the conversion to uint8 and the SSIM filtering happen on the GPU, so a quarter of the bytes cross
PCIe and the host never touches fp32 images.  `psnr_ssim` scores a whole sampled batch in one native call."""
import ctypes
import math

import numpy as np
import torch

from .. import _native


def tensor2img(tensor, out_type=np.uint8, min_max=(-1, 1)):
    """4D (B,C,H,W), 3D (C,H,W) or 2D (H,W) CUDA tensor -> numpy HWC (or HW) uint8 image, RGB order; 4-D input is tiled like
    torchvision.utils.make_grid(nrow=int(sqrt(B))), exactly as the reference does."""
    if out_type != np.uint8:
        raise NotImplementedError("sr3_b200.core.metrics.tensor2img produces uint8 images only")
    if not tensor.is_cuda:
        raise _native.NativeLibraryError("tensor2img expects a CUDA tensor (there is no CPU path)")
    t = tensor.squeeze().float().contiguous()
    n_dim = t.dim()
    if n_dim == 4:
        n, C, H, W = t.shape
        nrow = int(math.sqrt(n))
    elif n_dim == 3:
        n, (C, H, W), nrow = 1, t.shape, 1
    elif n_dim == 2:
        n, C, (H, W), nrow = 1, 1, t.shape, 1
    else:
        raise TypeError('Only support 4D, 3D and 2D tensor. But received with dimension: {:d}'.format(n_dim))
    if n > 1:
        ncol = min(nrow, n)
        rows = (n + ncol - 1) // ncol
        GH, GW = rows * (H + 2) + 2, ncol * (W + 2) + 2
        if C == 1:                                   # make_grid turns single-channel images into 3 channels
            t = t.expand(n, 3, H, W).contiguous()
            C = 3
    else:
        GH, GW = H, W
    out = torch.empty(GH, GW, C, dtype=torch.uint8, device=t.device)
    with torch.cuda.device(t.device):
        _native._check(_native.lib().sr3_tensor2img(_native._ptr(t), _native._ptr(out), n, C, H, W, max(nrow, 1), float(min_max[0]), float(min_max[1]),
                                                    _native._stream()))
    img = out.cpu().numpy()
    return img[:, :, 0] if n_dim == 2 else img


def calculate_psnr(img1, img2):
    """uint8 images (numpy arrays or CUDA uint8 tensors of the same shape) -> PSNR in dB, float64 arithmetic as the reference."""
    a = torch.as_tensor(img1).to("cuda", torch.uint8).contiguous() if not (torch.is_tensor(img1) and img1.is_cuda) else img1.contiguous()
    b = torch.as_tensor(img2).to(a.device, torch.uint8).contiguous() if not (torch.is_tensor(img2) and img2.is_cuda) else img2.contiguous()
    assert a.shape == b.shape and a.dtype == torch.uint8 and b.dtype == torch.uint8
    ssd = ctypes.c_uint64()
    with torch.cuda.device(a.device):
        _native._check(_native.lib().sr3_ssd_u8(_native._ptr(a), _native._ptr(b), a.numel(), ctypes.byref(ssd), _native._stream()))
    return _psnr(ssd.value, a.numel())


def _psnr(ssd, numel):
    mse = ssd / float(numel)
    if mse == 0:
        return float('inf')
    return 20 * math.log10(255.0 / math.sqrt(mse))


def _device_image(img, device=None):
    """numpy array or tensor -> contiguous CUDA tensor: uint8 stays uint8, every other dtype is cast to float64 on the device."""
    t = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img))
    if not t.is_cuda:
        t = t.to(device if device is not None else "cuda")
    if t.dtype != torch.uint8:
        t = t.to(torch.float64)
    return t.contiguous()


def ssim(img1, img2):
    """core/metrics.py:52-72 on the device: SSIM of two HW or HWC images in [0, 255] (numpy arrays or CUDA tensors), float64 arithmetic,
    11x11 Gaussian window (sigma 1.5) over the valid pixels, every channel filtered on its own; nan when H or W is below 11."""
    a = _device_image(img1)
    b = _device_image(img2, a.device)
    if a.shape != b.shape:
        raise ValueError('Input images must have the same dimensions.')
    if a.dim() == 2:
        (H, W), C = a.shape, 1
    elif a.dim() == 3:
        H, W, C = a.shape
    else:
        raise ValueError('Wrong input image dimensions.')
    if a.dtype != b.dtype:                      # one uint8 and one other image: both go through float64
        a, b = a.to(torch.float64), b.to(torch.float64)
    out = ctypes.c_double()
    with torch.cuda.device(a.device):
        _native._check(_native.lib().sr3_ssim(_native._ptr(a), _native._ptr(b), 0 if a.dtype == torch.uint8 else 1, 1, H, W, C,
                                              ctypes.byref(out), _native._stream()))
    return np.float64(out.value)


def _mean3(s):
    """calculate_ssim of an RGB image averages three identical ssim calls (core/metrics.py:85-89); the mean of three equal floats is not
    always that float, so it is formed the same way."""
    return np.array([s, s, s]).mean()


def calculate_ssim(img1, img2):
    """core/metrics.py:75-93: same dispatch, return values (None for an HWC image with neither 1 nor 3 channels) and errors."""
    if not img1.shape == img2.shape:
        raise ValueError('Input images must have the same dimensions.')
    if img1.ndim == 2:
        return ssim(img1, img2)
    elif img1.ndim == 3:
        if img1.shape[2] == 3:
            return _mean3(ssim(img1, img2))
        elif img1.shape[2] == 1:
            return ssim(img1.squeeze(), img2.squeeze())
    else:
        raise ValueError('Wrong input image dimensions.')


def psnr_ssim(sr, hr, min_max=(-1, 1), return_images=False):
    """The evaluation of a sampled batch in one native call: for every i, calculate_psnr and calculate_ssim of tensor2img(sr[i]) and
    tensor2img(hr[i]) (sr.py:216-217).  sr, hr: fp32 CUDA tensors [B, C, H, W], C in {1, 3}.  Returns float64 numpy arrays psnr[B] and
    ssim[B]; return_images=True also returns the uint8 images of sr and hr ([B, H, W, C], or [B, H, W] when C == 1: element i is
    tensor2img(sr[i]))."""
    if not (torch.is_tensor(sr) and torch.is_tensor(hr) and sr.is_cuda and hr.is_cuda):
        raise _native.NativeLibraryError("psnr_ssim expects CUDA tensors (there is no CPU path)")
    if sr.shape != hr.shape or sr.dim() != 4 or sr.shape[1] not in (1, 3):
        raise ValueError('psnr_ssim expects two [B, C, H, W] tensors of the same shape with C in {1, 3}, got %s and %s'
                         % (tuple(sr.shape), tuple(hr.shape)))
    B, C, H, W = sr.shape
    s = sr.detach().float().contiguous()
    h = hr.detach().to(s.device, torch.float32).contiguous()
    imgs = torch.empty(2, B, H, W, C, dtype=torch.uint8, device=s.device) if return_images else None
    ssd, ss = (ctypes.c_uint64 * B)(), (ctypes.c_double * B)()
    with torch.cuda.device(s.device):
        _native._check(_native.lib().sr3_image_metrics(_native._ptr(s), _native._ptr(h), B, C, H, W, float(min_max[0]), float(min_max[1]),
                                                       _native._ptr(imgs[0] if return_images else None),
                                                       _native._ptr(imgs[1] if return_images else None), ssd, ss, _native._stream()))
    psnrs = np.array([_psnr(ssd[i], C * H * W) for i in range(B)], dtype=np.float64)
    ssims = np.array([_mean3(ss[i]) if C == 3 else ss[i] for i in range(B)], dtype=np.float64)
    if not return_images:
        return psnrs, ssims
    u8 = imgs.cpu().numpy()
    if C == 1:
        u8 = u8[..., 0]
    return psnrs, ssims, u8[0], u8[1]

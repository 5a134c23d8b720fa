"""CPU oracle for the SSIM metric at the exit of the sampling path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy fp64 restatement of the reference's `ssim` / `calculate_ssim` (core/metrics.py:52-93) that needs no cv2: cv2.filter2D followed by
the [5:-5, 5:-5] crop is written out as the valid correlation.  tests/test_ssim.py pins it to what the unmodified reference computes
(tests/golden/sr3_ssim_golden.pt, written by tests/golden/make_ssim_golden.py) and checks the device metrics against it.  The rest of the
oracle (tensor2img, calculate_psnr, the UNet and diffusion) lives in oracle/sr3_oracle.py.
"""
import numpy as np


def _filter_valid(img: np.ndarray, window: np.ndarray) -> np.ndarray:
    """cv2.filter2D(img, -1, window)[5:-5, 5:-5] (core/metrics.py:61-68) for an 11x11 window: filter2D correlates (no kernel flip), each
    channel of an HWC image on its own, and the crop keeps exactly the pixels whose window lies inside the image, so the border mode
    never matters: the valid correlation, written out as 121 shifted, weighted sums."""
    k = window.shape[0]
    hv, wv = max(img.shape[0] - (k - 1), 0), max(img.shape[1] - (k - 1), 0)
    out = np.zeros((hv, wv) + img.shape[2:], dtype=np.float64)
    for i in range(k):
        for j in range(k):
            out += window[i, j] * img[i:i + hv, j:j + wv]
    return out


def ssim(img1: np.ndarray, img2: np.ndarray) -> float:
    """core/metrics.py:52-72."""
    C1 = (0.01 * 255) ** 2                                                         # :53
    C2 = (0.03 * 255) ** 2                                                         # :54
    img1 = img1.astype(np.float64)                                                 # :56
    img2 = img2.astype(np.float64)                                                 # :57
    x = np.arange(11, dtype=np.float64) - 5.0                                      # :58 cv2.getGaussianKernel(11, 1.5):
    kernel = np.exp(-0.5 / (1.5 * 1.5) * x * x)                                    #     exp(-(i - 5)^2 / (2 sigma^2)),
    kernel = (kernel * (1.0 / kernel.sum()))[:, None]                              #     normalised to sum 1, an 11x1 column
    window = np.outer(kernel, kernel.transpose())                                  # :59
    mu1 = _filter_valid(img1, window)                                              # :61
    mu2 = _filter_valid(img2, window)                                              # :62
    mu1_sq = mu1 ** 2                                                              # :63
    mu2_sq = mu2 ** 2                                                              # :64
    mu1_mu2 = mu1 * mu2                                                            # :65
    sigma1_sq = _filter_valid(img1 ** 2, window) - mu1_sq                          # :66
    sigma2_sq = _filter_valid(img2 ** 2, window) - mu2_sq                          # :67
    sigma12 = _filter_valid(img1 * img2, window) - mu1_mu2                         # :68
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))   # :70-71
    if ssim_map.size == 0:                                                         # :72 np.mean of an empty crop: nan (the reference
        return np.float64("nan")                                                   #     also warns)
    return ssim_map.mean()                                                         # :72


def calculate_ssim(img1: np.ndarray, img2: np.ndarray):
    """core/metrics.py:75-93 (an HWC image with neither 1 nor 3 channels falls off the end: None)."""
    if not img1.shape == img2.shape:                                               # :80-81
        raise ValueError("Input images must have the same dimensions.")
    if img1.ndim == 2:                                                             # :82-83
        return ssim(img1, img2)
    elif img1.ndim == 3:
        if img1.shape[2] == 3:                                                     # :85-89
            s = ssim(img1, img2)                                                   # three identical calls on the whole image:
            return np.array([s, s, s]).mean()                                      # computed once, averaged as the reference does
        elif img1.shape[2] == 1:                                                   # :90-91
            return ssim(np.squeeze(img1), np.squeeze(img2))
    else:                                                                          # :92-93
        raise ValueError("Wrong input image dimensions.")

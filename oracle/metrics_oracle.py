"""CPU oracle of the SSIM and PSNR evaluators (the reference's `lib/evaluator/eva_ssim.py` and `eva_psnr.py`).

SSIM is pytorch-ssim's: a Gaussian window (sigma 1.5, `window_size` taps normalised by their float32 sum), the outer
product of the taps as a 2-D window, depthwise `conv2d` with zero padding `window_size // 2` (an even window gives an
(H + 1) x (W + 1) map), the map ((2 mu1 mu2 + C1)(2 s12 + C2)) / ((mu1^2 + mu2^2 + C1)(s1^2 + s2^2 + C2)) with
s^2 = E[x^2] - mu^2, C1 = 0.01^2, C2 = 0.03^2, and its mean over everything (`size_average=True`) or per image.

PSNR is `psnr_evaluator.add_batch`'s per-image value: diff = (pred - gt) / rgb_range formed in float32; `None` keeps
the whole image, `"div2k"` shaves scale + 6 pixels from each side of H and W, `"benchmark"` first reduces the channels
to the gray difference sum_c diff_c * coef_c (coef = [65.738, 129.057, 25.064] / 256, float64) and shaves `scale`;
psnr = -10 log10(mean(valid^2)).

`fp32=False` is the float64 restatement: the reference's float32 taps cast to double, the window their exact outer
product, every sum and product in double.  `fp32=True` is the reference's own arithmetic (float32 tensors and a
float32 2-D window for SSIM, numpy on float32 arrays for PSNR); the difference of the two is the reference's error.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from .fid_oracle import make_images  # noqa: F401  (seeded structured images in [0, 1])
from .lpips_oracle import composed  # noqa: F401  (a hole-composited copy)

C1 = 0.01 ** 2
C2 = 0.03 ** 2
SIGMA = 1.5
GRAY_COEFFS = np.array([65.738, 129.057, 25.064]) / 256


def gaussian_taps(window_size: int) -> torch.Tensor:
    """The reference's 1-D taps, float32 [window_size]: exp(-(x - ws // 2)^2 / (2 sigma^2)) over their float32 sum."""
    gauss = torch.Tensor([np.exp(-(x - window_size // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(window_size)])
    return gauss / gauss.sum()


@torch.no_grad()
def ssim_map(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, fp32: bool = False) -> torch.Tensor:
    """The SSIM map [n, C, H', W'] (float64, or the reference's float32 with fp32=True) on the inputs' device."""
    g = gaussian_taps(window_size)
    if fp32:
        x, y = img1.float(), img2.float()
        w2 = g.unsqueeze(1).mm(g.unsqueeze(1).t()).float()
    else:
        x, y = img1.double(), img2.double()
        gd = g.double()
        w2 = gd.unsqueeze(1) * gd.unsqueeze(0)
    c = x.shape[1]
    window = w2.to(x).expand(c, 1, window_size, window_size).contiguous()
    p = window_size // 2

    def conv(t):
        return F.conv2d(t, window, padding=p, groups=c)

    mu1, mu2 = conv(x), conv(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(x * x) - mu1_sq
    sigma2_sq = conv(y * y) - mu2_sq
    sigma12 = conv(x * y) - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))


def ssim(img1, img2, window_size: int = 11, size_average: bool = True, fp32: bool = False) -> torch.Tensor:
    """compute_ssim: the mean of the map (0-dim), or per image [n] (the reference's mean(1).mean(1).mean(1))."""
    m = ssim_map(img1, img2, window_size, fp32)
    if size_average:
        return m.mean()
    return m.mean(1).mean(1).mean(1) if fp32 else m.mean((1, 2, 3))


def psnr(pred, gt, for_dataset="div2k", scale: int = 2, rgb_range=1, fp32: bool = False):
    """psnr_evaluator.add_batch's per-image PSNR of [n, C, H, W] float32 inputs (tensors or arrays): numpy [n], float32
    for None / "div2k" and float64 for "benchmark" with fp32=True, float64 throughout otherwise."""
    pred = np.asarray(pred.cpu() if isinstance(pred, torch.Tensor) else pred, dtype=np.float32)
    gt = np.asarray(gt.cpu() if isinstance(gt, torch.Tensor) else gt, dtype=np.float32)
    diff = (pred - gt) / rgb_range          # float32, as the reference forms it
    if not fp32:
        diff = diff.astype(np.float64)
    if for_dataset is None:
        valid = diff
    elif for_dataset == "benchmark":
        s = scale
        if diff.shape[1] > 1:
            diff = (diff * GRAY_COEFFS[None, :, None, None]).sum(1)
        valid = diff[:, s:-s, s:-s]
    elif for_dataset == "div2k":
        s = scale + 6
        valid = diff[:, :, s:-s, s:-s]
    else:
        raise NotImplementedError(for_dataset)
    axes = (1, 2) if valid.ndim == 3 else (1, 2, 3)
    with np.errstate(divide="ignore"):
        return -10 * np.log10((valid ** 2).mean(axis=axes))


def bright(n: int, c: int, h: int, w: int, seed: int = 0) -> torch.Tensor:
    """Seeded float32 images in [0.9, 1]: where s^2 = E[x^2] - mu^2 cancels worst."""
    return (0.9 + 0.1 * images(n, c, h, w, seed=seed)).float().contiguous()


def images(n: int, c: int, h: int, w: int, seed: int = 0) -> torch.Tensor:
    """make_images with any channel count (channels cycled from a 3-channel draw)."""
    x = make_images(n, h, w, seed=seed)
    return x[:, [k % 3 for k in range(c)]].contiguous() if c != 3 else x

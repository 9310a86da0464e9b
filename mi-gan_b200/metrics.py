"""SSIM and PSNR on the GPU: the reference's `eva_ssim` (pytorch-ssim) and `eva_psnr` arithmetic.

    from migan_b200 import metrics
    s = metrics.compute_ssim(real, composed)                              # CUDA float32, 0-dim
    s_img = metrics.compute_ssim(real, composed, size_average=False)      # CUDA float32 [n]
    p = metrics.compute_psnr(real, composed, for_dataset=None)            # CUDA float32 [n] (float64 for "benchmark")

The window sums, the SSIM map and every mean run in double in the C-ABI library (`include/metrics_b200.h`), two
launches per call.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np
import torch

from . import _abi

MAX_WINDOW = 31
SIGMA = 1.5

SYMBOLS = [
    ("metrics_ssim_workspace_bytes", ctypes.c_size_t, [ctypes.c_int] * 5),
    ("metrics_ssim", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 +
     [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    ("metrics_psnr_workspace_bytes", ctypes.c_size_t, [ctypes.c_int] * 4),
    ("metrics_psnr", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 6 +
     [ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
]


def lib(handle=None):
    """The product library with this module's symbols bound (`handle`: another build of the same sources)."""
    return _abi.library(SYMBOLS, handle)


def gaussian_taps(window_size: int) -> torch.Tensor:
    """pytorch-ssim's 1-D taps, float32 [window_size] on the CPU, by the reference's own expression (same bytes)."""
    gauss = torch.Tensor([np.exp(-(x - window_size // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(window_size)])
    return gauss / gauss.sum()


def map_size(H: int, W: int, window_size: int):
    """The SSIM map's H' x W' (conv2d with zero padding window_size // 2: an even window adds a row and a column)."""
    p = window_size // 2
    return H + 2 * p - window_size + 1, W + 2 * p - window_size + 1


def _check_window(window_size) -> int:
    if isinstance(window_size, bool) or int(window_size) != window_size or not 1 <= window_size <= MAX_WINDOW:
        raise ValueError("window_size must be an integer in 1..%d; got %r" % (MAX_WINDOW, window_size))
    return int(window_size)


def _pair(a, b, who):
    for t in (a, b):
        if not isinstance(t, torch.Tensor) or t.dim() != 4:
            raise RuntimeError("%s: expected two tensors of shape [n, C, H, W]" % who)
    if a.shape != b.shape:
        raise RuntimeError("%s: the inputs differ in shape: %s and %s" % (who, tuple(a.shape), tuple(b.shape)))
    if not (a.is_cuda and b.is_cuda):
        raise RuntimeError("migan_b200.metrics.%s runs on H100 (sm_90a) only; got %s and %s tensors. There is no CPU "
                           "path." % (who, a.device, b.device))
    if a.device != b.device:
        raise RuntimeError("%s: the inputs are on different devices: %s and %s" % (who, a.device, b.device))
    return a.to(torch.float32).contiguous(), b.to(torch.float32).contiguous()


def _workspace(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device=device)


@torch.no_grad()
def compute_ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True,
                 taps: Optional[torch.Tensor] = None) -> torch.Tensor:
    """pytorch-ssim's compute_ssim on CUDA [n, C, H, W] inputs: float32, 0-dim (the mean of the whole SSIM map) or [n]
    (each image's mean) with size_average=False.  `taps`: the 1-D window (default: the reference's Gaussian)."""
    ws = _check_window(window_size)
    a, b = _pair(img1, img2, "compute_ssim")
    n, C, H, W = a.shape
    dev = a.device
    g = (gaussian_taps(ws) if taps is None else taps).detach().to("cpu", torch.float32).contiguous()
    if g.numel() != ws:
        raise ValueError("taps: %d values for a window of %d" % (g.numel(), ws))
    per = torch.empty(n, dtype=torch.float32, device=dev)
    mean = torch.full((), float("nan"), dtype=torch.float32, device=dev)   # torch's mean of nothing
    if C == 0 or H == 0 or W == 0:
        raise ValueError("compute_ssim: empty images %s" % (tuple(a.shape),))
    if n == 0:
        return mean if size_average else per
    L = lib()
    with torch.cuda.device(dev):
        ws_t = _workspace(L.metrics_ssim_workspace_bytes(n, C, H, W, ws), dev)
        _abi.check(L.metrics_ssim(a.data_ptr(), b.data_ptr(), n, C, H, W, g.data_ptr(), ws,
                                  None if size_average else per.data_ptr(), mean.data_ptr() if size_average else None,
                                  ws_t.data_ptr(), ws_t.numel(), torch.cuda.current_stream(dev).cuda_stream), L)
    return mean if size_average else per


class SSIM(torch.nn.Module):
    """pytorch-ssim's SSIM module: forward(img1, img2) is compute_ssim(img1, img2, window_size, size_average)."""

    def __init__(self, window_size: int = 11, size_average: bool = True):
        super().__init__()
        self.window_size = _check_window(window_size)
        self.size_average = size_average
        self.taps = gaussian_taps(self.window_size)

    def forward(self, img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
        return compute_ssim(img1, img2, self.window_size, self.size_average, taps=self.taps)


_MODES = (None, "div2k", "benchmark")


@torch.no_grad()
def compute_psnr(pred: torch.Tensor, gt: torch.Tensor, for_dataset="div2k", scale: int = 2, rgb_range=1) -> torch.Tensor:
    """The per-image PSNR of psnr_evaluator(for_dataset, scale, rgb_range).add_batch(pred, gt) on CUDA [n, 3, H, W]
    inputs: a CUDA tensor [n], float32 for None and "div2k", float64 for "benchmark" (the reference's dtypes).
    None: the whole image; "div2k": scale + 6 pixels shaved from each side; "benchmark": the gray difference, `scale`
    shaved.  Identical images give inf."""
    if for_dataset not in _MODES:
        raise NotImplementedError("for_dataset must be None, 'div2k' or 'benchmark'; got %r" % (for_dataset,))
    if isinstance(scale, bool) or int(scale) != scale or scale < 0:
        raise ValueError("scale must be an integer >= 0; got %r" % (scale,))
    rgb = float(np.float32(rgb_range))
    if not rgb > 0:
        raise ValueError("rgb_range must be > 0; got %r" % (rgb_range,))
    a, b = _pair(pred, gt, "compute_psnr")
    n, C, H, W = a.shape
    if C != 3:
        raise ValueError("compute_psnr takes 3-channel images, as the evaluator does; got C=%d" % C)
    shave = {None: 0, "div2k": int(scale) + 6, "benchmark": int(scale)}[for_dataset]
    if for_dataset is not None and (shave == 0 or H - 2 * shave < 1 or W - 2 * shave < 1):
        raise ValueError("for_dataset=%r, scale=%r shaves %d pixels from each side of %d x %d: nothing is left, where the "
                         "reference returns NaN" % (for_dataset, scale, shave, H, W))
    if H == 0 or W == 0:
        raise ValueError("empty %d x %d images: the reference returns NaN" % (H, W))
    dev = a.device
    out = torch.empty(n, dtype=torch.float64, device=dev)
    if n > 0:
        L = lib()
        with torch.cuda.device(dev):
            ws_t = _workspace(L.metrics_psnr_workspace_bytes(n, H, W, shave), dev)
            _abi.check(L.metrics_psnr(a.data_ptr(), b.data_ptr(), n, C, H, W, int(for_dataset == "benchmark"), shave,
                                      rgb, out.data_ptr(), ws_t.data_ptr(), ws_t.numel(),
                                      torch.cuda.current_stream(dev).cuda_stream), L)
    return out if for_dataset == "benchmark" else out.to(torch.float32)

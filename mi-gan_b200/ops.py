"""sm_90a drop-ins for the reference's `torch_utils/ops` used around the generator path:
`upfirdn2d` (+ `setup_filter`, `filter2d`, `upsample2d`, `downsample2d`), `bias_act` and the 1x1
branches of `conv2d_resample`.  Same function names, argument meaning and error behaviour as the
reference (torch_utils/ops/upfirdn2d.py:72-384, bias_act.py:55-89, conv2d_resample.py:59-154);
forward only (inference), float32 NCHW CUDA tensors, no `impl='ref'` / CPU fallback -- the CPU
oracles live in oracle/ for the tests.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _abi

# name -> (cuda_idx, def_alpha, def_gain)   torch_utils/ops/bias_act.py:22-32
ACTIVATIONS = {
    "linear": (1, 0.0, 1.0), "relu": (2, 0.0, float(np.sqrt(2))), "lrelu": (3, 0.2, float(np.sqrt(2))),
    "tanh": (4, 0.0, 1.0), "sigmoid": (5, 0.0, 1.0), "elu": (6, 0.0, 1.0), "selu": (7, 0.0, 1.0),
    "softplus": (8, 0.0, 1.0), "swish": (9, 0.0, float(np.sqrt(2))),
}


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def _guard(device: torch.device):
    return torch.cuda.device(device)


def _require_cuda_f32(x: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(x, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % what)
    if not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: migan_b200.ops has no CPU path" % what)
    if x.dtype != torch.float32:
        raise RuntimeError("%s must be float32, got %s" % (what, x.dtype))
    return x.contiguous()


def _parse_scaling(scaling):
    if isinstance(scaling, int):
        scaling = [scaling, scaling]
    assert isinstance(scaling, (list, tuple)) and all(isinstance(v, int) for v in scaling)
    sx, sy = scaling
    assert sx >= 1 and sy >= 1
    return sx, sy


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(v, int) for v in padding)
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    padx0, padx1, pady0, pady1 = padding
    return padx0, padx1, pady0, pady1


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    return int(f.shape[-1]), int(f.shape[0])


def setup_filter(f, device=torch.device("cpu"), normalize=True, flip_filter=False, gain=1, separable=None):
    """FIR prototype -> filter tensor (torch_utils/ops/upfirdn2d.py:72-116)."""
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in [0, 1, 2] and f.numel() > 0
    if f.ndim == 0:
        f = f[None]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = torch.outer(f, f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def _upfirdn2d_pass(x, f2d, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain):
    lib = _abi.load()
    n, c, h, w = x.shape
    fh, fw = f2d.shape
    ow = (w * upx + padx0 + padx1 - fw + downx) // downx   # upfirdn2d.cpp:32-33
    oh = (h * upy + pady0 + pady1 - fh + downy) // downy
    if ow < 1 or oh < 1:
        raise RuntimeError("upfirdn2d: output size must be >= 1, got %dx%d" % (oh, ow))
    y = torch.empty((n, c, oh, ow), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _abi.check(lib.b200_upfirdn2d(x.data_ptr(), f2d.data_ptr(), y.data_ptr(), n, c, h, w, fh, fw, upx, upy, downx, downy,
                                      padx0, padx1, pady0, pady1, int(bool(flip)), float(gain), _stream(x)))
    return y


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl="cuda"):
    """Pad, zero-insert up-sample, FIR filter, decimate (torch_utils/ops/upfirdn2d.py:120-164)."""
    assert impl == "cuda", "migan_b200.ops has no reference/CPU implementation (see oracle/)"
    x = _require_cuda_f32(x, "x")
    if x.ndim != 4:
        raise RuntimeError("x must be rank 4 [N,C,H,W]")
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2] and f.dtype == torch.float32
    f = f.to(x.device).contiguous()
    if f.ndim == 2:
        return _upfirdn2d_pass(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain)
    # separable: two 1-D passes, sqrt(gain) each (upfirdn2d.py:238-240)
    y = _upfirdn2d_pass(x, f.unsqueeze(0).contiguous(), upx, 1, downx, 1, padx0, padx1, 0, 0, flip_filter, np.sqrt(gain))
    return _upfirdn2d_pass(y, f.unsqueeze(1).contiguous(), 1, upy, 1, downy, 0, 0, pady0, pady1, flip_filter, np.sqrt(gain))


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl="cuda"):
    """upfirdn2d.py:272-304."""
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + fw // 2, padx1 + (fw - 1) // 2, pady0 + fh // 2, pady1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl="cuda"):
    """upfirdn2d.py:308-343."""
    upx, upy = _parse_scaling(up)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw + upx - 1) // 2, padx1 + (fw - upx) // 2, pady0 + (fh + upy - 1) // 2, pady1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy, impl=impl)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl="cuda"):
    """upfirdn2d.py:347-382."""
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw - downx + 1) // 2, padx1 + (fw - downx) // 2, pady0 + (fh - downy + 1) // 2, pady1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def bias_act(x, b=None, dim=1, act="linear", alpha=None, gain=None, clamp=None, impl="cuda"):
    """Fused bias + activation + gain + clamp, forward only (torch_utils/ops/bias_act.py:55-89)."""
    assert impl == "cuda", "migan_b200.ops has no reference/CPU implementation (see oracle/)"
    x = _require_cuda_f32(x, "x")
    if act not in ACTIVATIONS:
        raise KeyError(act)
    idx, def_alpha, def_gain = ACTIVATIONS[act]
    alpha = float(def_alpha if alpha is None else alpha)
    gain = float(def_gain if gain is None else gain)
    assert clamp is None or clamp >= 0
    clamp = float(-1 if clamp is None else clamp)
    step_b, size_b, bptr = 1, 1, None
    if b is not None:
        b = _require_cuda_f32(b, "b")
        assert b.ndim == 1 and 0 <= dim < x.ndim and b.shape[0] == x.shape[dim]
        step_b = int(np.prod(x.shape[dim + 1:])) if dim + 1 < x.ndim else 1
        size_b = int(b.shape[0])
        bptr = b.data_ptr()
    y = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _abi.check(_abi.load().b200_bias_act(x.data_ptr(), bptr, y.data_ptr(), x.numel(), step_b, size_b, idx, alpha, gain, clamp,
                                             _stream(x)))
    return y


def _conv1x1(x, w):
    """y[n,o,h,w] = sum_i w[o,i] x[n,i,h,w] on the CUDA-core GEMM (NHWC inside; the layout change is torch plumbing)."""
    n, ci, h, wd = x.shape
    co = w.shape[0]
    xa = x.permute(0, 2, 3, 1).contiguous()
    wt = w.reshape(co, ci).t().contiguous()
    y = torch.empty((n, h, wd, co), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _abi.check(_abi.load().b200_conv1x1_nhwc(xa.data_ptr(), wt.data_ptr(), y.data_ptr(), n * h * wd, ci, co, _stream(x)))
    return y.permute(0, 3, 1, 2).contiguous()


def _conv2d_resample_general(x, w, f, up, down, padding, groups, flip_weight, flip_filter):
    """All six branches through the C ABI (`b200_conv2d_resample`, include/comodgan_b200.h): NHWC im2col + fp32 GEMM,
    transposed convolution as GEMM + col2im, NHWC upfirdn2d.  `padding` is the caller's (un-adjusted) padding."""
    lib = _abi.load()
    n, cin, h, wd = x.shape
    cout, _, kh, kw = w.shape
    if f is None:
        f2d, fh, fw = None, 0, 0
    else:
        f = f.to(device=x.device, dtype=torch.float32)
        f2d = (torch.outer(f, f) if f.ndim == 1 else f).contiguous()       # separable == outer product (upfirdn2d.py:239-240)
        fh, fw = f2d.shape
    px0, px1, py0, py1 = padding
    args = [n, cin, h, wd, cout, kh, kw, fh, fw, up, down, px0, px1, py0, py1, groups, int(bool(flip_weight)), int(bool(flip_filter))]
    need, oh, ow = ctypes.c_size_t(), ctypes.c_int(), ctypes.c_int()
    _abi.check(lib.b200_conv2d_resample(None, None, None, None, *args, None, 0, ctypes.byref(need), ctypes.byref(oh),
                                        ctypes.byref(ow), None))
    y = torch.empty((n, cout, oh.value, ow.value), dtype=torch.float32, device=x.device)
    raw = torch.empty(need.value + 1024, dtype=torch.uint8, device=x.device)
    off = (-raw.data_ptr()) % 1024
    with _guard(x.device):
        _abi.check(lib.b200_conv2d_resample(x.data_ptr(), w.data_ptr(), f2d.data_ptr() if f2d is not None else None,
                                            y.data_ptr(), *args, raw.data_ptr() + off, need.value, None, None, None,
                                            _stream(x)))
    return y


def conv2d_resample(x, w, f=None, up=1, down=1, padding=0, groups=1, flip_weight=True, flip_filter=False):
    """2-D convolution with optional up/down-sampling (torch_utils/ops/conv2d_resample.py:59-154), every branch:
    1x1 + down (:106-109), 1x1 + up (:112-115), k x k down (:118-121), up via transposed convolution (:124-142),
    plain (:145-147) and the generic fallback (:150-154); `groups` included."""
    x = _require_cuda_f32(x, "x")
    w = _require_cuda_f32(w, "w")
    assert x.ndim == 4 and w.ndim == 4
    assert isinstance(up, int) and up >= 1 and isinstance(down, int) and down >= 1 and groups >= 1
    assert f is None or (isinstance(f, torch.Tensor) and f.ndim in [1, 2] and f.dtype == torch.float32)
    out_channels, in_channels_per_group, kh, kw = w.shape
    assert x.shape[1] == in_channels_per_group * groups and out_channels % groups == 0
    pad = list(_parse_padding(padding))
    fast_1x1 = (kh == 1 and kw == 1 and groups == 1 and x.shape[1] % 16 == 0 and out_channels % 64 == 0)
    if not fast_1x1:
        return _conv2d_resample_general(x, w, f, up, down, pad, groups, flip_weight, flip_filter)
    # MI-GAN's 1x1 branches: channels-last GEMM straight on the tensor (no im2col)
    fw, fh = _get_filter_size(f)
    px0, px1, py0, py1 = pad
    if up > 1:   # conv2d_resample.py:94-98
        px0 += (fw + up - 1) // 2; px1 += (fw - up) // 2; py0 += (fh + up - 1) // 2; py1 += (fh - up) // 2
    if down > 1:  # :101-104
        px0 += (fw - down + 1) // 2; px1 += (fw - down) // 2; py0 += (fh - down + 1) // 2; py1 += (fh - down) // 2
    if down > 1 and up == 1:    # :106-110  FIR-down, then conv
        x = upfirdn2d(x, f, down=down, padding=[px0, px1, py0, py1], flip_filter=flip_filter)
        return _conv1x1(x, w)
    if up > 1 and down == 1:    # :113-116  conv, then FIR-up with gain up^2
        x = _conv1x1(x, w)
        return upfirdn2d(x, f, up=up, padding=[px0, px1, py0, py1], gain=up ** 2, flip_filter=flip_filter)
    if up == 1 and down == 1 and [px0, px1, py0, py1] == [0, 0, 0, 0]:   # :145-147
        return _conv1x1(x, w)
    return _conv2d_resample_general(x, w, f, up, down, pad, groups, flip_weight, flip_filter)


def preprocess_u8(img_u8: torch.Tensor, mask_u8: torch.Tensor) -> torch.Tensor:
    """x[N,4,R,R] = cat([mask-0.5, img*mask]) from uint8 CUDA tensors img [N,R,R,3], mask [N,R,R] (255 = known):
    scripts/demo.py:56-66, bit-exact with the torch expression there."""
    if not (img_u8.is_cuda and mask_u8.is_cuda) or img_u8.dtype != torch.uint8 or mask_u8.dtype != torch.uint8:
        raise RuntimeError("preprocess_u8 expects uint8 CUDA tensors: migan_b200.ops has no CPU path")
    n, r = img_u8.shape[0], img_u8.shape[1]
    if tuple(img_u8.shape) != (n, r, r, 3) or tuple(mask_u8.shape) != (n, r, r):
        raise RuntimeError("preprocess_u8 expects img [N,R,R,3] and mask [N,R,R]")
    img_u8, mask_u8 = img_u8.contiguous(), mask_u8.contiguous()
    x = torch.empty((n, 4, r, r), dtype=torch.float32, device=img_u8.device)
    with _guard(img_u8.device):
        _abi.check(_abi.load().b200_preprocess_u8(img_u8.data_ptr(), mask_u8.data_ptr(), x.data_ptr(), n, r, _stream(img_u8)))
    return x


def postprocess_u8(y: torch.Tensor, img_u8: torch.Tensor, mask_u8: torch.Tensor) -> torch.Tensor:
    """uint8 [N,R,R,3] composite of the generator output y [N,3,R,R] with the known pixels (scripts/demo.py:135-142)."""
    y = _require_cuda_f32(y, "y")
    n, r = y.shape[0], y.shape[2]
    if tuple(y.shape) != (n, 3, r, r) or tuple(img_u8.shape) != (n, r, r, 3) or tuple(mask_u8.shape) != (n, r, r):
        raise RuntimeError("postprocess_u8 expects y [N,3,R,R], img [N,R,R,3], mask [N,R,R]")
    if not (img_u8.is_cuda and mask_u8.is_cuda) or img_u8.dtype != torch.uint8 or mask_u8.dtype != torch.uint8:
        raise RuntimeError("postprocess_u8 expects uint8 CUDA tensors")
    img_u8, mask_u8 = img_u8.contiguous(), mask_u8.contiguous()
    out = torch.empty((n, r, r, 3), dtype=torch.uint8, device=y.device)
    with _guard(y.device):
        _abi.check(_abi.load().b200_postprocess_u8(y.data_ptr(), img_u8.data_ptr(), mask_u8.data_ptr(), out.data_ptr(), n, r,
                                                   _stream(y)))
    return out


def feather_kernel(kernel_size: int = 5, sigma: float = 1.0) -> torch.Tensor:
    """The smoothing kernel of the deployed pipeline's GaussianSmoothing (scripts/create_onnx_pipeline.py:66-88), built with the
    same torch expression so that it is bit-identical to the buffer the reference registers (5x5, sigma 1 at :127-128)."""
    import math
    grids = torch.meshgrid([torch.arange(kernel_size, dtype=torch.float32) for _ in range(2)], indexing="ij")
    kernel = 1
    mean = (kernel_size - 1) / 2
    for g in grids:
        kernel = kernel * (1 / (sigma * math.sqrt(2 * math.pi)) * torch.exp(-((g - mean) / (2 * sigma)) ** 2))
    return (kernel / torch.sum(kernel)).contiguous()


def feather_composite(y: torch.Tensor, image_u8: torch.Tensor, mask_u8: torch.Tensor, kernel: torch.Tensor = None) -> torch.Tensor:
    """uint8 [N,3,H,W] = the feathered blend of the deployed pipeline (scripts/create_onnx_pipeline.py:233-245) of the generator
    output y [N,3,H,W] (float32, CUDA) with image_u8 [N,3,H,W] under mask_u8 [N,1,H,W] (255 = known), all at the same size:
    the mask is dilated (3x3 max-pool), smoothed (5x5, reflect border) and used as the per-pixel weight."""
    y = _require_cuda_f32(y, "y")
    n, h, w = y.shape[0], y.shape[2], y.shape[3]
    if tuple(y.shape) != (n, 3, h, w) or tuple(image_u8.shape) != (n, 3, h, w) or tuple(mask_u8.shape) != (n, 1, h, w):
        raise RuntimeError("feather_composite expects y [N,3,H,W], image [N,3,H,W], mask [N,1,H,W]")
    if not (image_u8.is_cuda and mask_u8.is_cuda) or image_u8.dtype != torch.uint8 or mask_u8.dtype != torch.uint8:
        raise RuntimeError("feather_composite expects uint8 CUDA tensors: migan_b200.ops has no CPU path")
    k = (feather_kernel() if kernel is None else kernel).detach().to("cpu", torch.float32).contiguous()
    if k.numel() != 25:
        raise RuntimeError("feather_composite implements the pipeline's 5x5 smoothing kernel (25 taps)")
    image_u8, mask_u8 = image_u8.contiguous(), mask_u8.contiguous()
    out = torch.empty((n, 3, h, w), dtype=torch.uint8, device=y.device)
    with _guard(y.device):
        _abi.check(_abi.load().b200_feather_composite(y.data_ptr(), image_u8.data_ptr(), mask_u8.data_ptr(), out.data_ptr(), n, h, w,
                                                      k.data_ptr(), _stream(y)))
    return out

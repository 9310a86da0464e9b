"""LPIPS on the GPU: lpips 0.1's `LPIPS(net="alex")`, the distance evaluate_fid_lpips.py reports.

    compute_lpips = LPIPS(net="alex")                        # lpips.LPIPS(net="alex") drop-in
    compute_lpips.to("cuda")
    d = compute_lpips(imgs, composed_imgs, normalize=True)   # CUDA float32 [n, 1, 1, 1]

The network runs in the C-ABI library (`include/lpips_b200.h`): AlexNet's five convolutions on the tensor-core implicit
GEMM of the FID network (TF32 hi / lo operands in three passes, fp32-faithful), both inputs as one batch.  There is no
CPU path.
"""
from __future__ import annotations

import ctypes
import importlib.util
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import _abi, _convnet

LAYERS = 5
MIN_SIZE = 31
CHANNELS = (64, 192, 384, 256, 256)
ALEXNET_FILE = "alexnet-owt-7be5be79.pth"
# lpips' ScalingLayer constants
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
# lpips' AlexNet slices hold torchvision's features.{0, 3, 6, 8, 10}
TORCHVISION_KEYS = {"net.slice1.0": "features.0", "net.slice2.3": "features.3", "net.slice3.6": "features.6",
                    "net.slice4.8": "features.8", "net.slice5.10": "features.10"}
_DEFAULTS = {"net": "alex", "version": "0.1", "lpips": True, "spatial": False, "pnet_rand": False, "pnet_tune": False}

SYMBOLS = [
    ("lpips_create", ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    ("lpips_destroy", ctypes.c_int, [ctypes.c_void_p]),
    ("lpips_num_weights", ctypes.c_int, [ctypes.c_void_p]),
    ("lpips_weight_info", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_char_p),
                                         ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int64)]),
    ("lpips_set_weight", ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int64]),
    ("lpips_finalize_weights", ctypes.c_int, [ctypes.c_void_p]),
    ("lpips_workspace_bytes", ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    ("lpips_forward", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 +
     [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    ("lpips_last_launch_count", ctypes.c_int, [ctypes.c_void_p]),
    ("lpips_launch_plan", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p,
                                         ctypes.c_int]),
    ("lpips_input", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 +
     [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
]


def lib(handle=None):
    """The product library with this module's symbols bound (`handle`: another build of the same sources)."""
    return _abi.library(SYMBOLS, handle)


def weight_spec(handle=None) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every state_dict entry the library takes, in state_dict order (the `lins.*` aliases aside)."""
    return _convnet.weight_spec(lib(handle), "lpips")


def launch_plan(n: int, H: int, W: int, handle=None) -> List[str]:
    """The forward's launches for n pairs of H x W, one line each ("<kind> <name> key=value ...")."""
    return _convnet.launch_plan(lib(handle), "lpips", n, H, W)


def default_alexnet_path() -> str:
    """Where torchvision caches AlexNet's weights: <torch.hub.get_dir()>/checkpoints/alexnet-owt-7be5be79.pth."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", ALEXNET_FILE)


def default_lin_path() -> Optional[str]:
    """The installed lpips package's weights/v0.1/alex.pth, or None when lpips is not installed."""
    try:
        spec = importlib.util.find_spec("lpips")
    except (ImportError, ValueError):
        return None
    if spec is None or not spec.submodule_search_locations:
        return None
    return os.path.join(list(spec.submodule_search_locations)[0], "weights", "v0.1", "alex.pth")


def _load(path_or_dict) -> Dict[str, torch.Tensor]:
    if isinstance(path_or_dict, (str, os.PathLike)):
        path_or_dict = torch.load(path_or_dict, map_location="cpu", weights_only=True)
    return dict(path_or_dict)


def _default_weights(model_path) -> Dict[str, torch.Tensor]:
    """AlexNet from torchvision's cache and the linear layers from model_path or the lpips package: never downloads."""
    alex_path = default_alexnet_path()
    lin_path = model_path if model_path is not None else default_lin_path()
    missing = []
    if not os.path.isfile(alex_path):
        missing.append("AlexNet weights %s (the file torchvision caches; place it there)" % alex_path)
    if lin_path is None:
        missing.append("LPIPS linear layers weights/v0.1/alex.pth (the lpips package is not installed; pass "
                       "model_path=<path to alex.pth>)")
    elif not os.path.isfile(lin_path):
        missing.append("LPIPS linear layers %s (lpips' weights/v0.1/alex.pth; place it there or pass model_path=)" % lin_path)
    if missing:
        raise FileNotFoundError("LPIPS weights not found. This package never downloads; missing: " + "; ".join(missing)
                                + ". Or pass weights=<state_dict or path>.")
    alex = _load(alex_path)
    state = {"scaling_layer.shift": torch.tensor(SHIFT).view(1, 3, 1, 1),
             "scaling_layer.scale": torch.tensor(SCALE).view(1, 3, 1, 1)}
    for ours, tv in TORCHVISION_KEYS.items():
        for leaf in ("weight", "bias"):
            if tv + "." + leaf not in alex:
                raise KeyError("%s: no '%s.%s' (expected torchvision's AlexNet state_dict)" % (alex_path, tv, leaf))
            state[ours + "." + leaf] = alex[tv + "." + leaf]
    state.update(_load(lin_path))
    return state


def _canonical(state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Drops recent lpips versions' `lins.{k}.model.1.weight`, which must equal `lin{k}.model.1.weight`."""
    out = {k: v for k, v in state.items() if not k.startswith("lins.")}
    for k, v in state.items():
        if not k.startswith("lins."):
            continue
        parts = k.split(".")
        key = "lin%s.%s" % (parts[1], ".".join(parts[2:]))
        if key not in out:
            out[key] = v
        elif out[key].shape != v.shape or not torch.equal(out[key].detach().cpu(), v.detach().cpu()):
            raise ValueError("'%s' differs from '%s': the two names are one tensor in lpips" % (k, key))
    return out


class LPIPS(_convnet.Network):
    """lpips.LPIPS at the configuration evaluate_fid_lpips.py uses: net="alex", version "0.1", linear layers, not
    spatial, eval mode.  forward(in0, in1) returns CUDA float32 [n, 1, 1, 1]."""

    def __init__(self, pretrained=True, net="alex", version="0.1", lpips=True, spatial=False, pnet_rand=False,
                 pnet_tune=False, use_dropout=True, model_path=None, eval_mode=True, verbose=True, *, weights=None):
        super().__init__()
        got = {"net": net, "version": version, "lpips": lpips, "spatial": spatial, "pnet_rand": pnet_rand,
               "pnet_tune": pnet_tune}
        for k, v in got.items():
            if v != _DEFAULTS[k]:
                raise NotImplementedError(
                    "only LPIPS(net='alex', version='0.1', lpips=True, spatial=False, pnet_rand=False, pnet_tune=False) "
                    "is built; got %s=%r" % (k, v))
        if not pretrained and weights is None:
            raise NotImplementedError("pretrained=False (randomly initialised linear layers) is not built; pass weights=")
        self.pnet_type, self.version, self.spatial, self.L = "alex", "0.1", False, LAYERS
        state = _canonical(_default_weights(model_path) if weights is None else _load(weights))
        self._set_state(lib(), "lpips", {k: v.detach().to("cpu", torch.float32).contiguous() for k, v in state.items()})

    @torch.no_grad()
    def forward(self, in0: torch.Tensor, in1: torch.Tensor, retPerLayer=False, normalize=False):
        for t in (in0, in1):
            if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != 3:
                raise RuntimeError("expected in0, in1 of shape [N, 3, H, W]")
        if in0.shape != in1.shape:
            raise RuntimeError("in0 and in1 differ in shape: %s and %s" % (tuple(in0.shape), tuple(in1.shape)))
        if not (in0.is_cuda and in1.is_cuda):
            raise RuntimeError("migan_b200.lpips.LPIPS runs on H100 (sm_90a) only; got %s and %s tensors. There is no "
                               "CPU path." % (in0.device, in1.device))
        if in0.device != in1.device:
            raise RuntimeError("in0 and in1 are on different devices: %s and %s" % (in0.device, in1.device))
        n, _, H, W = in0.shape
        if H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError("LPIPS (AlexNet) needs H, W >= %d, the smallest size its second max pool has an output for; "
                             "got %d x %d" % (MIN_SIZE, H, W))
        dev = in0.device
        a = in0.to(torch.float32).contiguous()
        b = in1.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            eng = self._engine(dev)
            val = torch.empty(n, dtype=torch.float32, device=dev)
            per = torch.empty((LAYERS, n), dtype=torch.float32, device=dev) if retPerLayer else None
            if n > 0:
                ws = eng.workspace(n, H, W)
                _abi.check(eng.lib.lpips_forward(eng.handle, a.data_ptr(), b.data_ptr(), n, H, W, int(bool(normalize)),
                                                 val.data_ptr(), per.data_ptr() if per is not None else None,
                                                 ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream),
                           eng.lib)
        val = val.view(n, 1, 1, 1)
        if retPerLayer:
            return val, [per[k].view(n, 1, 1, 1) for k in range(LAYERS)]
        return val

    def launch_plan(self, n: int, H: int, W: int) -> List[str]:
        """The forward's launches for n pairs of H x W, one line each."""
        return launch_plan(n, H, W)


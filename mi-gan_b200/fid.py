"""FID on the GPU: pytorch_fid's InceptionV3 pool3 features, the feature statistics and the Frechet distance.

    model = InceptionV3()                                  # pytorch_fid.inception.InceptionV3([3]) drop-in
    stats = FeatureStatistics(device="cuda")
    for real in batches:
        stats.add(model(real)[0].squeeze(-1).squeeze(-1))
    mu, sigma = stats.mean_cov()                            # np.mean / np.cov(rowvar=False), float64
    fid = calculate_frechet_distance(mu, sigma, mu2, sigma2)

The network runs in the C-ABI library (`include/inception_b200.h`): 94 convolutions on the tensor-core implicit GEMM
with TF32 hi / lo operands in three passes (fp32-faithful), BatchNorm folded at load time.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List, Tuple, Union

import numpy as np
import torch
from scipy import linalg

from . import _abi

FEATURES = 2048
WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"
_DEFAULTS = {"output_blocks": [3], "resize_input": True, "normalize_input": True, "requires_grad": False,
             "use_fid_inception": True}

SYMBOLS = [
    ("inception_create", ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    ("inception_destroy", ctypes.c_int, [ctypes.c_void_p]),
    ("inception_num_weights", ctypes.c_int, [ctypes.c_void_p]),
    ("inception_weight_info", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_char_p),
                                             ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int64)]),
    ("inception_set_weight", ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int64]),
    ("inception_finalize_weights", ctypes.c_int, [ctypes.c_void_p]),
    ("inception_workspace_bytes", ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    ("inception_features", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    ("inception_last_launch_count", ctypes.c_int, [ctypes.c_void_p]),
    ("inception_launch_plan", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_char_p, ctypes.c_int]),
    ("inception_resize", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                        ctypes.c_void_p]),
    ("inception_pool", ctypes.c_int, [ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 4 +
     [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    ("inception_conv2d", ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_void_p] +
     [ctypes.c_int] * 6 + [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                           ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p]),
    ("fid_stats_update", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
]

_bound = set()


def lib(handle=None):
    """The product library with this module's symbols bound (`handle`: another build of the same sources)."""
    h = handle if handle is not None else _abi.load()
    if id(h) not in _bound:
        _abi.bind(h, SYMBOLS)
        _bound.add(id(h))
    return h


def weight_spec(handle=None) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every state_dict entry the library takes, in state_dict order (num_batches_tracked aside)."""
    L = lib(handle)
    h = ctypes.c_void_p()
    _abi.check(L.inception_create(-1, ctypes.byref(h)), L)
    try:
        out = []
        name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
        for i in range(L.inception_num_weights(h)):
            _abi.check(L.inception_weight_info(h, i, ctypes.byref(name), ctypes.byref(nd), shape), L)
            out.append((name.value.decode(), tuple(int(v) for v in shape[:nd.value])))
        return out
    finally:
        L.inception_destroy(h)


def default_weights_path() -> str:
    """Where pytorch_fid caches the FID Inception weights: <torch.hub.get_dir()>/checkpoints/<file>."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)


def _load_weights(weights) -> Dict[str, torch.Tensor]:
    if weights is None:
        path = default_weights_path()
        if not os.path.isfile(path):
            raise FileNotFoundError(
                "FID Inception weights not found at %s. This package never downloads; place %s there (the file "
                "pytorch_fid downloads on first use) or pass weights=<state_dict or path>." % (path, WEIGHTS_FILE))
        weights = path
    if isinstance(weights, (str, os.PathLike)):
        weights = torch.load(weights, map_location="cpu", weights_only=True)
    return dict(weights)


class InceptionV3(torch.nn.Module):
    """pytorch_fid.inception.InceptionV3 at the configuration evaluate_fid_lpips.py uses: block 3 (2048-d pool3),
    resize to 299 x 299, inputs in [0, 1] normalised to [-1, 1], the FID Inception blocks.  forward(x) returns
    [features [n, 2048, 1, 1]] as CUDA float32."""

    BLOCK_INDEX_BY_DIM = {2048: 3}
    DEFAULT_BLOCK_INDEX = 3

    def __init__(self, output_blocks=(3,), resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True, *, weights=None):
        super().__init__()
        got = {"output_blocks": list(output_blocks), "resize_input": resize_input, "normalize_input": normalize_input,
               "requires_grad": requires_grad, "use_fid_inception": use_fid_inception}
        for k, v in got.items():
            if v != _DEFAULTS[k]:
                raise NotImplementedError(
                    "only InceptionV3(output_blocks=[3], resize_input=True, normalize_input=True, requires_grad=False, "
                    "use_fid_inception=True) is built; got %s=%r" % (k, v))
        self.output_blocks = [3]
        self.last_needed_block = 3
        self._state = {k: v.detach().to("cpu", torch.float32).contiguous() for k, v in _load_weights(weights).items()
                       if not k.endswith("num_batches_tracked")}
        _Engine(None, self._state)   # checks the keys on the host now: missing, unknown or mis-shaped fail by name
        self._engines = {}

    def _engine(self, device):
        eng = self._engines.get(device)
        if eng is None:
            eng = _Engine(device, self._state)
            self._engines[device] = eng
        return eng

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError("expected x of shape [N, 3, H, W] in [0, 1]")
        if not x.is_cuda:
            raise RuntimeError("migan_b200.fid.InceptionV3 runs on H100 (sm_90a) only; got a %s tensor. There is no CPU "
                               "path." % x.device)
        n, _, H, W = x.shape
        x = x.to(torch.float32).contiguous()
        with torch.cuda.device(x.device):
            eng = self._engine(x.device)
            feats = torch.empty((n, FEATURES), dtype=torch.float32, device=x.device)
            if n > 0:
                ws = eng.workspace(n, H, W)
                _abi.check(eng.lib.inception_features(eng.handle, x.data_ptr(), n, H, W, feats.data_ptr(), ws.data_ptr(),
                                                      ws.numel(), torch.cuda.current_stream(x.device).cuda_stream))
        return [feats.view(n, FEATURES, 1, 1)]

    def last_launch_count(self) -> int:
        eng = next(iter(self._engines.values()))
        return int(eng.lib.inception_last_launch_count(eng.handle))

    def launch_plan(self, n: int, H: int, W: int) -> List[str]:
        """The forward's launches for n images of H x W, one line each."""
        return launch_plan(n, H, W)


def launch_plan(n: int, H: int, W: int, handle=None) -> List[str]:
    """The forward's launches for n images of H x W, one line each ("<kind> <name> key=value ...")."""
    L = lib(handle)
    h = ctypes.c_void_p()
    _abi.check(L.inception_create(-1, ctypes.byref(h)), L)
    try:
        size = L.inception_launch_plan(h, n, H, W, None, 0)
        if size < 0:
            _abi.check(-size, L)
        buf = ctypes.create_string_buffer(size + 1)
        L.inception_launch_plan(h, n, H, W, buf, size + 1)
        return buf.value.decode().splitlines()
    finally:
        L.inception_destroy(h)


class _Engine:
    """One library context: device None = description only (weights parsed, nothing uploaded)."""

    def __init__(self, device, state: Dict[str, torch.Tensor], handle=None):
        self.lib = lib(handle)
        self.handle = ctypes.c_void_p()
        index = -1 if device is None else (device.index if device.index is not None else torch.cuda.current_device())
        _abi.check(self.lib.inception_create(index, ctypes.byref(self.handle)), self.lib)
        self.workspaces: Dict[tuple, torch.Tensor] = {}
        self.device = device
        for k, t in state.items():
            t = t.detach().to("cpu", torch.float32).contiguous()
            _abi.check(self.lib.inception_set_weight(self.handle, k.encode(), t.data_ptr(), t.numel()), self.lib)
        if device is not None:
            _abi.check(self.lib.inception_finalize_weights(self.handle), self.lib)
        else:
            missing = self._first_missing(state)
            if missing:
                raise _abi.MiganError(_abi.ERR_INVALID, "missing key '%s' in the state_dict" % missing)

    def _first_missing(self, state):
        name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
        for i in range(self.lib.inception_num_weights(self.handle)):
            self.lib.inception_weight_info(self.handle, i, ctypes.byref(name), ctypes.byref(nd), shape)
            if name.value.decode() not in state:
                return name.value.decode()
        return None

    def workspace(self, n, H, W) -> torch.Tensor:
        ws = self.workspaces.get((n, H, W))
        if ws is None:
            nbytes = int(self.lib.inception_workspace_bytes(self.handle, n, H, W))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self.workspaces = {(n, H, W): ws}
        return ws

    def __del__(self):
        try:
            if self.handle:
                self.lib.inception_destroy(self.handle)
        except Exception:
            pass


class FeatureStatistics:
    """Streaming np.mean / np.cov(rowvar=False) of feature rows, accumulated in float64 on the device.  The sums are
    taken about a fixed shift (the first batch's mean), so a large common offset does not cancel."""

    def __init__(self, dim: int = FEATURES, device: Union[str, torch.device] = "cuda"):
        self.dim = int(dim)
        self.device = torch.device(device)
        self.shift = torch.zeros(self.dim, dtype=torch.float64, device=self.device)
        self.sum = torch.zeros(self.dim, dtype=torch.float64, device=self.device)
        self.sumsq = torch.zeros((self.dim, self.dim), dtype=torch.float64, device=self.device)
        self.count = 0

    @torch.no_grad()
    def add(self, feats: torch.Tensor) -> None:
        """feats: [n, dim] (or [n, dim, 1, 1]) CUDA tensor."""
        f = feats.reshape(feats.shape[0], -1)
        if f.shape[1] != self.dim:
            raise ValueError("expected features of dimension %d, got %d" % (self.dim, f.shape[1]))
        if not f.is_cuda:
            raise RuntimeError("FeatureStatistics.add takes CUDA features")
        if f.shape[0] == 0:
            return
        f = f.to(device=self.device, dtype=torch.float32).contiguous()
        with torch.cuda.device(self.device):
            _abi.check(lib().fid_stats_update(f.data_ptr(), f.shape[0], self.dim, self.shift.data_ptr(),
                                              self.sum.data_ptr(), self.sumsq.data_ptr(), int(self.count == 0),
                                              torch.cuda.current_stream(self.device).cuda_stream))
        self.count += int(f.shape[0])

    def mean_cov(self) -> Tuple[np.ndarray, np.ndarray]:
        """(mu, sigma) as float64 numpy arrays: np.mean(axis=0) and np.cov(rowvar=False) (ddof 1) of every row added."""
        if self.count < 2:
            raise ValueError("FeatureStatistics needs at least 2 feature rows, has %d" % self.count)
        s1 = self.sum.cpu().numpy()
        s2 = self.sumsq.cpu().numpy()
        n = float(self.count)
        mu = self.shift.cpu().numpy() + s1 / n
        sigma = (s2 - np.outer(s1, s1) / n) / (n - 1)
        return mu, sigma


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps: float = 1e-6) -> float:
    """||mu1 - mu2||^2 + tr(sigma1) + tr(sigma2) - 2 tr(sqrt(sigma1 sigma2)), with scipy's sqrtm on the host.  A singular
    product is retried with eps on both diagonals; a significant imaginary part raises ValueError."""
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    if mu1.shape != mu2.shape:
        raise ValueError("training and test mean vectors have different lengths")
    if sigma1.shape != sigma2.shape:
        raise ValueError("training and test covariances have different dimensions")
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))

"""FID on the GPU: pytorch_fid's InceptionV3 pool3 features, the feature statistics and the Frechet distance.

    model = InceptionV3()                                  # pytorch_fid.inception.InceptionV3([3]) drop-in
    stats = FeatureStatistics(device="cuda")
    for real in batches:
        stats.add(model(real)[0].squeeze(-1).squeeze(-1))
    mu, sigma = stats.mean_cov()                            # np.mean / np.cov(rowvar=False), float64
    fid = calculate_frechet_distance(mu, sigma, mu2, sigma2)   # pytorch_fid's scipy route, on the host
    fid = stats.frechet_distance(stats_fake)                # or all on the device (float64 eigensolver)
    fid = frechet_distance(mu, sigma, mu2, sigma2)          # the same from numpy arrays or CUDA tensors

The network runs in the C-ABI library (`include/inception_b200.h`): 94 convolutions on the tensor-core implicit GEMM
with TF32 hi / lo operands in three passes (fp32-faithful), BatchNorm folded at load time.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from scipy import linalg

from . import _abi, _convnet

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
    ("inception_workspace_bytes_u8", ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int]),
    ("inception_features_u8", ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int] + [ctypes.c_void_p] * 2 +
     [ctypes.c_size_t, ctypes.c_void_p]),
    ("inception_input_u8", ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] + [ctypes.c_void_p] * 2),
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
    ("fid_stats_update_binned", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 3 +
     [ctypes.c_void_p] * 5),
]
MAX_BINS = 32                                  # include/inception_b200.h FID_STATS_MAX_BINS; 32 MiB per bin at d = 2048
# csrc/frechet.cu: the device mean / covariance and the Fréchet distance
FRECHET_SYMBOLS = [
    ("fid_stats_mean_cov", ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 3),
    ("fid_frechet_workspace_bytes", ctypes.c_size_t, [ctypes.c_int]),
    ("fid_frechet_distance", ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                                            ctypes.POINTER(ctypes.c_int), ctypes.c_void_p, ctypes.c_size_t,
                                            ctypes.c_void_p]),
]


def lib(handle=None):
    """The product library with this module's symbols bound (`handle`: another build of the same sources)."""
    return _abi.library(SYMBOLS, handle)


def frechet_lib(handle=None):
    """The product library (or `handle`, another build of csrc/frechet.cu) with the Fréchet symbols bound."""
    return _abi.library(FRECHET_SYMBOLS, lib(handle))


def weight_spec(handle=None) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every state_dict entry the library takes, in state_dict order (num_batches_tracked aside)."""
    return _convnet.weight_spec(lib(handle), "inception")


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


class InceptionV3(_convnet.Network):
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
        state = {k: v.detach().to("cpu", torch.float32).contiguous() for k, v in _load_weights(weights).items()
                 if not k.endswith("num_batches_tracked")}
        self._set_state(lib(), "inception", state)
        self._staged: Dict[torch.device, Tuple[torch.Tensor, torch.cuda.Event]] = {}   # features_u8's pinned buffers

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

    @torch.no_grad()
    def features_u8(self, photos: Sequence[np.ndarray], device=None) -> torch.Tensor:
        """Features [n, 2048] (CUDA float32, on `device` or the current CUDA device) of decoded photos: host uint8
        [H, W, 3] arrays of any sizes, such as `np.array(Image.open(p).convert("RGB"))`.  Row i equals
        `self(ToTensor(photos[i])[None])[0]` bit for bit, for any batch and any mix of sizes in it.

        The photos are packed into a pinned staging buffer and reach the device in one copy on the current stream; the
        buffer is kept for the next call (it grows to the largest call's bytes) and is refilled only once that copy is
        done."""
        arrays = [np.ascontiguousarray(p) for p in photos]
        for i, a in enumerate(arrays):
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
                raise ValueError("features_u8: photo %d is %s %s; expected uint8 [H, W, 3] with H, W >= 1"
                                 % (i, a.dtype, a.shape))
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("migan_b200.fid.InceptionV3 runs on H100 (sm_90a) only; got device %s. There is no CPU "
                               "path." % device)
        n = len(arrays)
        feats = torch.empty((n, FEATURES), dtype=torch.float32, device=device)
        if n == 0:
            return feats
        sizes = np.array([a.nbytes for a in arrays], dtype=np.int64)
        off = np.zeros(n, dtype=np.int64)
        np.cumsum(sizes[:-1], out=off[1:])
        h = np.array([a.shape[0] for a in arrays], dtype=np.int32)
        w = np.array([a.shape[1] for a in arrays], dtype=np.int32)
        total = int(sizes.sum())
        with torch.cuda.device(device):
            eng = self._engine(device)
            stream = torch.cuda.current_stream(device)
            host, copied = self._staging(device, total)
            flat = host.numpy()
            for a, o in zip(arrays, off):
                flat[o:o + a.nbytes] = a.reshape(-1)
            photos_d = torch.empty(total, dtype=torch.uint8, device=device)
            photos_d.copy_(host[:total], non_blocking=True)
            copied.record(stream)
            ws = eng._workspace.get(("u8", n), lambda: eng.lib.inception_workspace_bytes_u8(eng.handle, n), device)
            _abi.check(eng.lib.inception_features_u8(eng.handle, photos_d.data_ptr(), off.ctypes.data, h.ctypes.data,
                                                     w.ctypes.data, n, feats.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     stream.cuda_stream))
        return feats

    def _staging(self, device, nbytes: int) -> Tuple[torch.Tensor, torch.cuda.Event]:
        """The pinned staging buffer of `device`, at least nbytes long, once the copy that last read it is done, and the
        event to record after the copy that reads it next."""
        buf, done = self._staged.get(device, (None, None))
        if done is not None:
            done.synchronize()
        if buf is None or buf.numel() < nbytes:
            buf = None
            buf = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        self._staged[device] = (buf, torch.cuda.Event())
        return self._staged[device]

    def launch_plan(self, n: int, H: int, W: int) -> List[str]:
        """The forward's launches for n images of H x W, one line each."""
        return launch_plan(n, H, W)


def launch_plan(n: int, H: int, W: int, handle=None) -> List[str]:
    """The forward's launches for n images of H x W, one line each ("<kind> <name> key=value ...")."""
    return _convnet.launch_plan(lib(handle), "inception", n, H, W)


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

    def mean_cov_device(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """mean_cov() computed on the device, as float64 CUDA tensors: the same bits, and no host copy of a matrix."""
        if self.count < 2:
            raise ValueError("FeatureStatistics needs at least 2 feature rows, has %d" % self.count)
        mu = torch.empty(self.dim, dtype=torch.float64, device=self.device)
        sigma = torch.empty((self.dim, self.dim), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _abi.check(frechet_lib().fid_stats_mean_cov(self.shift.data_ptr(), self.sum.data_ptr(), self.sumsq.data_ptr(),
                                                self.count, self.dim, mu.data_ptr(), sigma.data_ptr(),
                                                torch.cuda.current_stream(self.device).cuda_stream))
        return mu, sigma

    def frechet_distance(self, other: "FeatureStatistics") -> float:
        """The FID between these statistics and `other`'s, computed on the device from both objects' sums."""
        if not isinstance(other, FeatureStatistics):
            raise TypeError("frechet_distance takes another FeatureStatistics")
        if other.dim != self.dim:
            raise ValueError("training and test covariances have different dimensions")
        if other.device != self.device:
            raise ValueError("both statistics must be on one device, got %s and %s" % (self.device, other.device))
        mu1, sigma1 = self.mean_cov_device()
        mu2, sigma2 = other.mean_cov_device()
        return _frechet(mu1, sigma1, mu2, sigma2).fid


class BinnedFeatureStatistics:
    """`nbins` FeatureStatistics at once: `add(feats, bins)` gives row i to bin bins[i] (-1: to none), on the device and
    with no host synchronisation.  Bin b holds, bit for bit, what a FeatureStatistics holds after add(feats[bins == b])
    for every call in turn (calls with no row in b skipped)."""

    def __init__(self, nbins: int, dim: int = FEATURES, device: Union[str, torch.device] = "cuda"):
        self.nbins, self.dim = int(nbins), int(dim)
        if not 1 <= self.nbins <= MAX_BINS:
            raise ValueError("BinnedFeatureStatistics: %d bins (1 to %d)" % (self.nbins, MAX_BINS))
        self.device = torch.device(device)
        self.shift = torch.zeros((self.nbins, self.dim), dtype=torch.float64, device=self.device)
        self.sum = torch.zeros((self.nbins, self.dim), dtype=torch.float64, device=self.device)
        self.sumsq = torch.zeros((self.nbins, self.dim, self.dim), dtype=torch.float64, device=self.device)
        self.count = torch.zeros(self.nbins, dtype=torch.int64, device=self.device)

    @torch.no_grad()
    def add(self, feats: torch.Tensor, bins: torch.Tensor) -> None:
        """feats: [n, dim] (or [n, dim, 1, 1]) CUDA tensor; bins: [n] CUDA integer tensor, -1 for a row in no bin."""
        f = feats.reshape(feats.shape[0], -1)
        if f.shape[1] != self.dim:
            raise ValueError("expected features of dimension %d, got %d" % (self.dim, f.shape[1]))
        if not f.is_cuda or not bins.is_cuda:
            raise RuntimeError("BinnedFeatureStatistics.add takes CUDA features and bins")
        if tuple(bins.shape) != (f.shape[0],) or bins.dtype not in (torch.int32, torch.int64):
            raise ValueError("bins must be an integer tensor of shape [%d], got %s %s" % (f.shape[0], bins.dtype,
                                                                                        tuple(bins.shape)))
        if f.shape[0] == 0:
            return
        f = f.to(device=self.device, dtype=torch.float32).contiguous()
        b = bins.to(device=self.device, dtype=torch.int32).contiguous()
        with torch.cuda.device(self.device):
            _abi.check(lib().fid_stats_update_binned(f.data_ptr(), b.data_ptr(), f.shape[0], self.dim, self.nbins,
                                                     self.shift.data_ptr(), self.sum.data_ptr(), self.sumsq.data_ptr(),
                                                     self.count.data_ptr(),
                                                     torch.cuda.current_stream(self.device).cuda_stream))

    def counts(self) -> np.ndarray:
        """The rows each bin has received: int64 [nbins] (one device-to-host copy)."""
        return self.count.cpu().numpy()

    def mean_cov_device(self, b: int, count: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Bin b's FeatureStatistics.mean_cov_device(): float64 CUDA tensors.  `count` (the bin's entry of counts())
        saves the copy of the counts."""
        n = int(self.counts()[b]) if count is None else int(count)
        if n < 2:
            raise ValueError("BinnedFeatureStatistics: bin %d needs at least 2 feature rows, has %d" % (b, n))
        mu = torch.empty(self.dim, dtype=torch.float64, device=self.device)
        sigma = torch.empty((self.dim, self.dim), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _abi.check(frechet_lib().fid_stats_mean_cov(self.shift[b].data_ptr(), self.sum[b].data_ptr(),
                                                        self.sumsq[b].data_ptr(), n, self.dim, mu.data_ptr(),
                                                        sigma.data_ptr(),
                                                        torch.cuda.current_stream(self.device).cuda_stream))
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


class FrechetTerms(NamedTuple):
    """The Fréchet distance and its terms: fid = mean_term + trace1 + trace2 - 2 * trace_sqrt.  `sweeps`: the Jacobi
    sweeps of the two eigensolves (sigma1's, then the one behind tr sqrt(sigma1 sigma2))."""
    fid: float
    mean_term: float
    trace1: float
    trace2: float
    trace_sqrt: float
    sweeps: Tuple[int, int]


MAX_DIM = 4096
_workspace = _abi.Workspace()


def _check_covariance(name, x, xp) -> None:
    """Finite, and symmetric to 1e-9 of the largest entry (xp: numpy or torch)."""
    if not bool(xp.isfinite(x).all()):
        raise ValueError("%s has non-finite values" % name)
    if name.startswith("sigma") and float(xp.abs(x - x.T).max()) > 1e-9 * float(xp.abs(x).max()):
        raise ValueError("%s is not symmetric to 1e-9 of its largest entry, so it is not a covariance" % name)


def frechet_distance(mu1, sigma1, mu2, sigma2) -> float:
    """||mu1 - mu2||^2 + tr(sigma1) + tr(sigma2) - 2 tr(sqrt(sigma1 sigma2)) in float64 on the GPU.

    Takes float64 numpy arrays (for example np.load of a pytorch_fid .npz with `mu` and `sigma`) or CUDA tensors; host
    arrays are uploaded once.  sigma1 and sigma2 must be covariances: finite and symmetric to 1e-9 of their largest
    entry.  tr sqrt comes from two float64 block-Jacobi eigensolves (no matrix square root of the non-symmetric
    product): the square roots of eigenvalues that rounding left slightly negative count as 0."""
    return frechet_terms(mu1, sigma1, mu2, sigma2).fid


def frechet_terms(mu1, sigma1, mu2, sigma2) -> FrechetTerms:
    """frechet_distance() with its terms and the eigensolver's sweeps."""
    names = ("mu1", "sigma1", "mu2", "sigma2")
    args = [x.detach() if isinstance(x, torch.Tensor) and x.is_cuda else np.asarray(x, dtype=np.float64)
            for x in (mu1, sigma1, mu2, sigma2)]
    shapes = [tuple(x.shape) for x in args]
    if len(shapes[0]) != 1 or len(shapes[2]) != 1 or len(shapes[1]) != 2 or len(shapes[3]) != 2:
        raise ValueError("expected mu of shape [d] and sigma of shape [d, d]")
    if shapes[0] != shapes[2]:
        raise ValueError("training and test mean vectors have different lengths")
    if shapes[1] != shapes[3]:
        raise ValueError("training and test covariances have different dimensions")
    if shapes[1] != (shapes[0][0], shapes[0][0]):
        raise ValueError("sigma of shape %s does not match mu of length %d" % (shapes[1], shapes[0][0]))
    if not 1 <= shapes[0][0] <= MAX_DIM:
        raise ValueError("feature dimension %d outside 1..%d" % (shapes[0][0], MAX_DIM))
    for name, x in zip(names, args):
        if isinstance(x, np.ndarray):
            _check_covariance(name, x, np)
    cuda = [x for x in args if isinstance(x, torch.Tensor)]
    device = cuda[0].device if cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        t = []
        for name, x in zip(names, args):
            if isinstance(x, torch.Tensor):
                x = x.to(device=device, dtype=torch.float64).contiguous()
                _check_covariance(name, x, torch)
            else:
                x = torch.from_numpy(np.ascontiguousarray(x)).to(device)
            t.append(x)
        return _frechet(*t)


def _frechet(mu1, sigma1, mu2, sigma2, handle=None) -> FrechetTerms:
    """The library call on float64 contiguous CUDA tensors of one device."""
    L = frechet_lib(handle)
    d = int(mu1.shape[0])
    if d < 1 or d > MAX_DIM:
        raise ValueError("feature dimension %d outside 1..%d" % (d, MAX_DIM))
    device = mu1.device
    ws = _workspace.get((device, d), lambda: L.fid_frechet_workspace_bytes(d), device)
    out = (ctypes.c_double * 4)()
    sweeps = (ctypes.c_int * 2)()
    with torch.cuda.device(device):
        _abi.check(L.fid_frechet_distance(mu1.data_ptr(), sigma1.data_ptr(), mu2.data_ptr(), sigma2.data_ptr(), d, out,
                                          sweeps, ws.data_ptr(), ws.numel(),
                                          torch.cuda.current_stream(device).cuda_stream), L)
    fid = out[0] + out[1] + out[2] - 2 * out[3]
    return FrechetTerms(float(fid), out[0], out[1], out[2], out[3], (sweeps[0], sweeps[1]))

"""Precision, recall, density and coverage on the GPU: the k-nearest-neighbour manifold metrics of Kynkaanniemi et al.
2019 (StyleGAN2-ADA's `pr50k3`) and Naeem et al. 2020.

    res = precision_recall_density_coverage(real_feats, fake_feats)    # [N, d] and [M, d]
    res.precision, res.recall, res.density, res.coverage

FID and KID fold two failures into one number: composites that do not look real, and composites that look real but
cover only part of the real distribution.  Precision (and density, less sensitive to outliers) measures the first,
recall (and coverage) the second.  With r_i the (k + 1)-th smallest squared distance from real row i to the real rows
(itself included, so duplicate rows count as neighbours) and s_j the same within the fake rows:

    precision = #{j : exists i, |X_j - Y_i|^2 <= r_i} / M          recall   = #{i : exists j, |Y_i - X_j|^2 <= s_j} / N
    density   = sum_j #{i : |X_j - Y_i|^2 <= r_i} / (k M)          coverage = #{i : min_j |Y_i - X_j|^2 <= r_i} / N

The comparison is `<=`, as StyleGAN2-ADA's `compute_pr`; the prdc package uses `<`, which differs only at exact ties.
The library (`include/inception_b200.h`, `prdc_counts`) computes the four integer counts on fp64 tensor-core tiles,
every distance in float64; the ratios are finished here in float64.  The evaluation commands take pytorch_fid's
InceptionV3 pool3 features, whereas `pr50k3` uses a VGG16 detector: the formula is the same, the numbers are not.
There is no CPU path.

`RealRadii(real, k, max_fake)` computes the real side once, for scoring several fake sets against one real set.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Union

import numpy as np
import torch

from . import _abi, ids

MAX_DIM, MAX_K, DEFAULT_K = 4096, 32, 3

SYMBOLS = [
    ("prdc_workspace_bytes", ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    ("prdc_counts", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                   ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                   ctypes.c_void_p]),
    ("prdc_real_radii", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    ("prdc_counts_with_real_radii", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                   ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
]


def prdc_lib(handle=None):
    """The product library (or `handle`, another build of csrc/prdc.cu) with the PRDC symbols bound."""
    return _abi.library(SYMBOLS, handle)


class PRDCResult(NamedTuple):
    """The four metrics, the neighbourhood size k and the two set sizes."""
    precision: float
    recall: float
    density: float
    coverage: float
    k: int
    n_real: int
    n_fake: int


_workspace = _abi.Workspace()


def finish(counts, k: int, n_real: int, n_fake: int) -> PRDCResult:
    """The ratios of the four counts (precision, recall, density, coverage), each one correctly rounded division."""
    p, r, d, c = (int(v) for v in counts)
    return PRDCResult(p / n_fake, r / n_real, d / (k * n_fake), c / n_real, int(k), int(n_real), int(n_fake))


def _check_k(k, n_real: int, n_fake: int = None) -> int:
    k = int(k)
    if not 1 <= k <= MAX_K:
        raise ValueError("k must be in 1..%d, got %d" % (MAX_K, k))
    for name, n in (("real", n_real), ("fake", n_fake)):
        if n is not None and k + 1 > n:
            raise ValueError("k = %d needs at least k + 1 = %d %s rows, got %d" % (k, k + 1, name, n))
    return k


def _rows(name, x, d=None):
    """x as a contiguous 2-D CUDA float32 / float64 tensor, checked (width, finite) before any device work."""
    x = ids._prepare(name, x)
    if d is not None and int(x.shape[1]) != d:
        raise ValueError("real and fake features differ in width: %d and %d" % (d, int(x.shape[1])))
    if not 1 <= int(x.shape[1]) <= MAX_DIM:
        raise ValueError("feature dimension %d outside 1..%d" % (int(x.shape[1]), MAX_DIM))
    finite = bool(torch.isfinite(x).all()) if isinstance(x, torch.Tensor) else bool(np.isfinite(x).all())
    if not finite:
        raise ValueError("%s has non-finite values" % name)
    return x


def _to_device(x, device, dtype) -> torch.Tensor:
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(x))
    return x.to(device=device, dtype=dtype).contiguous()


def _dtype_code(x: torch.Tensor) -> int:
    return ids.FLOAT64 if x.dtype == torch.float64 else ids.FLOAT32


class RealRadii:
    """The real side of the metrics, computed once: the real rows on the device and a workspace holding their squared
    norms and radii r_i, for any number of fake sets of at most `max_fake` rows (default: as many as the real rows).
    Calls with it must be ordered on one stream: they share the workspace."""

    def __init__(self, real, k: int = DEFAULT_K, max_fake: int = None, handle=None):
        real = _rows("real", real)
        self.n_real, self.dim = (int(v) for v in real.shape)
        self.max_fake = self.n_real if max_fake is None else int(max_fake)
        self.k = _check_k(k, self.n_real, self.max_fake)
        self.device = (real.device if isinstance(real, torch.Tensor)
                       else torch.device("cuda", torch.cuda.current_device()))
        self.rows = _to_device(real, self.device, torch.float64 if real.dtype in (np.float64, torch.float64)
                               else torch.float32)
        self.handle = handle
        L = prdc_lib(handle)
        with torch.cuda.device(self.device):
            nbytes = L.prdc_workspace_bytes(self.n_real, self.max_fake, self.dim, self.k)
            self.workspace = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
            stream = torch.cuda.current_stream(self.device)
            _abi.check(L.prdc_real_radii(self.rows.data_ptr(), self.n_real, self.dim, _dtype_code(self.rows), self.k,
                                         self.workspace.data_ptr(), self.workspace.numel(), stream.cuda_stream), L)

    def counts(self, fake) -> torch.Tensor:
        """int64 [4] on the device: the counts of `fake` (a contiguous CUDA tensor, checked) against the real rows."""
        n_fake = int(fake.shape[0])
        if n_fake > self.max_fake:
            raise ValueError("%d fake rows, the real radii were prepared for at most %d" % (n_fake, self.max_fake))
        real = self.rows
        if fake.dtype == torch.float64 and real.dtype == torch.float32:
            real = real.double()          # the same values: the stored norms and radii still hold
        fake = fake.to(real.dtype).contiguous()
        L = prdc_lib(self.handle)
        out = torch.empty(4, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            _abi.check(L.prdc_counts_with_real_radii(real.data_ptr(), self.n_real, fake.data_ptr(), n_fake, self.dim,
                                                     _dtype_code(real), self.k, out.data_ptr(),
                                                     self.workspace.data_ptr(), self.workspace.numel(),
                                                     stream.cuda_stream), L)
        return out


def precision_recall_density_coverage(real: Union[torch.Tensor, np.ndarray, RealRadii], fake,
                                      k: int = DEFAULT_K) -> PRDCResult:
    """The four metrics of real [N, d] and fake [M, d] features: CUDA float32 / float64 tensors, or numpy arrays, which
    are uploaded once; both sides are read at the wider of their two dtypes.  `real` may be a `RealRadii` (its k then
    applies).  ValueError for k outside 1..32, k + 1 above N or M, mismatched or out-of-range widths and non-finite
    values, before any device work."""
    if isinstance(real, RealRadii):
        fake = _rows("fake", fake, real.dim)
        _check_k(real.k, real.n_real, int(fake.shape[0]))
        fake = _to_device(fake, real.device, torch.float64 if fake.dtype in (np.float64, torch.float64)
                          else torch.float32)
        counts = real.counts(fake).cpu().numpy()
        return finish(counts, real.k, real.n_real, int(fake.shape[0]))
    real = _rows("real", real)
    fake = _rows("fake", fake, int(real.shape[1]))
    n_real, n_fake = int(real.shape[0]), int(fake.shape[0])
    k = _check_k(k, n_real, n_fake)
    wide = any(x.dtype in (np.float64, torch.float64) for x in (real, fake))
    cuda = [x for x in (real, fake) if isinstance(x, torch.Tensor)]
    device = cuda[0].device if cuda else torch.device("cuda", torch.cuda.current_device())
    dtype = torch.float64 if wide else torch.float32
    with torch.cuda.device(device):
        counts = prdc_counts(_to_device(real, device, dtype), _to_device(fake, device, dtype), k).cpu().numpy()
    return finish(counts, k, n_real, n_fake)


def prdc_counts(real: torch.Tensor, fake: torch.Tensor, k: int = DEFAULT_K, handle=None) -> torch.Tensor:
    """The library call on contiguous CUDA tensors of one device and one dtype: int64 [4] (precision, recall, density,
    coverage counts) on the device, enqueued on the current stream.  The module's workspace is shared, so calls on
    different streams must be ordered by the caller."""
    L = prdc_lib(handle)
    device = real.device
    n_real, n_fake, d = int(real.shape[0]), int(fake.shape[0]), int(real.shape[1])
    ws = _workspace.get((device, n_real, n_fake, d, k), lambda: L.prdc_workspace_bytes(n_real, n_fake, d, k), device)
    out = torch.empty(4, dtype=torch.int64, device=device)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        _abi.check(L.prdc_counts(real.data_ptr(), n_real, fake.data_ptr(), n_fake, d, _dtype_code(real), k,
                                 out.data_ptr(), ws.data_ptr(), ws.numel(), stream.cuda_stream), L)
    return out

"""KID on the GPU: the kernel Inception distance of Binkowski et al. 2018, as StyleGAN2-ADA reports it (`kid50k_full`).

    res = kernel_inception_distance(real_feats, fake_feats)    # [n_r, d] and [n_f, d]
    res.kid, res.std

KID is the unbiased estimate of the squared MMD between the real and the fake features under the cubic polynomial
kernel k(u, v) = (u.v / d + 1)^3, averaged over `num_subsets` random subsets of m = min(n_r, n_f, max_subset_size)
rows of each side.  Unlike FID it has no bias in the number of images, so values over sets of different sizes compare.

The subsets are drawn on the host by `np.random.RandomState(seed)`: per subset, first the fake rows
`rng.choice(n_f, m, replace=False)`, then the real rows `rng.choice(n_r, m, replace=False)`, StyleGAN2-ADA's order.
The library (`include/inception_b200.h`, `kid_subset_terms`) computes each subset's sums Sxx, Syy, Sxy in float64 on
fp64 tensor-core tiles; the mean is then taken here in StyleGAN2-ADA's expression and order, in float64 where
StyleGAN2-ADA uses float32.  `std` is `np.std` of the per-subset estimates, the figure torch-fidelity reports next to
the mean.  The evaluation commands take pytorch_fid's InceptionV3 features, the ones behind their FID, whereas
StyleGAN2-ADA uses its own TorchScript Inception with a different resize: the formula is the same, the numbers are not.
There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Tuple

import numpy as np
import torch

from . import _abi, ids

MAX_DIM = 4096
NUM_SUBSETS, MAX_SUBSET_SIZE = 100, 1000

SYMBOLS = [
    ("kid_workspace_bytes", ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    ("kid_subset_terms", ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
]


def kid_lib(handle=None):
    """The product library (or `handle`, another build of csrc/kid.cu) with the KID symbols bound."""
    return _abi.library(SYMBOLS, handle)


class KIDResult(NamedTuple):
    """`kid`: the mean of the per-subset estimates; `std`: their standard deviation (ddof 0); `subsets` and
    `subset_size`: S and m."""
    kid: float
    std: float
    subsets: int
    subset_size: int


_workspace = _abi.Workspace()


def draw_subsets(n_real: int, n_fake: int, num_subsets: int, m: int, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """(fake_idx, real_idx): int32 [S, m] each, drawn by RandomState(seed) fake first, then real, subset by subset."""
    rng = np.random.RandomState(seed)
    fake_idx = np.empty((num_subsets, m), dtype=np.int32)
    real_idx = np.empty((num_subsets, m), dtype=np.int32)
    for s in range(num_subsets):
        fake_idx[s] = rng.choice(n_fake, m, replace=False)
        real_idx[s] = rng.choice(n_real, m, replace=False)
    return fake_idx, real_idx


def finish(terms: np.ndarray, m: int) -> Tuple[float, float]:
    """(KID, std) from the per-subset sums [S, 3] = (Sxx, Syy, Sxy): StyleGAN2-ADA's accumulation in float64."""
    t = 0.0
    e = []
    for sxx, syy, sxy in terms.tolist():
        a = (sxx + syy) / (m - 1) - 2 * sxy / m
        t += a
        e.append(a / m)
    return t / len(e) / m, float(np.std(np.array(e, dtype=np.float64)))


def kernel_inception_distance(real, fake, num_subsets: int = NUM_SUBSETS, max_subset_size: int = MAX_SUBSET_SIZE,
                              seed: int = 0) -> KIDResult:
    """KID of real [n_r, d] and fake [n_f, d] features: CUDA float32 / float64 tensors, or numpy arrays, which are
    uploaded once.  Both sides are read at the wider of their two dtypes.  ValueError for m < 2, mismatched or
    out-of-range shapes, S < 1 and non-finite values, before any device work."""
    real, fake = ids._prepare("real", real), ids._prepare("fake", fake)
    (n_r, d), (n_f, d_f) = (tuple(int(v) for v in x.shape) for x in (real, fake))
    if d != d_f:
        raise ValueError("real and fake features differ in width: %d and %d" % (d, d_f))
    if not 1 <= d <= MAX_DIM:
        raise ValueError("feature dimension %d outside 1..%d" % (d, MAX_DIM))
    num_subsets, max_subset_size = int(num_subsets), int(max_subset_size)
    if num_subsets < 1:
        raise ValueError("num_subsets must be >= 1, got %d" % num_subsets)
    m = min(n_r, n_f, max_subset_size)
    if m < 2:
        raise ValueError("KID needs subsets of at least 2 rows: min(%d real, %d fake, max_subset_size %d) = %d"
                         % (n_r, n_f, max_subset_size, m))
    for name, x in (("real", real), ("fake", fake)):
        finite = bool(torch.isfinite(x).all()) if isinstance(x, torch.Tensor) else bool(np.isfinite(x).all())
        if not finite:
            raise ValueError("%s has non-finite values" % name)
    fake_idx, real_idx = draw_subsets(n_r, n_f, num_subsets, m, seed)
    wide = any(x.dtype in (np.float64, torch.float64) for x in (real, fake))
    cuda = [x for x in (real, fake) if isinstance(x, torch.Tensor)]
    device = cuda[0].device if cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        t = []
        for x in (real, fake):
            if not isinstance(x, torch.Tensor):
                x = torch.from_numpy(np.ascontiguousarray(x))
            t.append(x.to(device=device, dtype=torch.float64 if wide else torch.float32).contiguous())
        terms = subset_terms(t[0], t[1], real_idx, fake_idx).cpu().numpy()
    kid, std = finish(terms, m)
    return KIDResult(kid, std, num_subsets, m)


def subset_terms(real, fake, real_idx: np.ndarray, fake_idx: np.ndarray, handle=None) -> torch.Tensor:
    """The library call on contiguous CUDA tensors of one device and one dtype: float64 [S, 3] (Sxx, Syy, Sxy) on the
    device, enqueued on the current stream.  The module's workspace holds the index tables until the kernels have read
    them, so calls on different streams must be ordered by the caller."""
    real_idx = np.ascontiguousarray(real_idx, dtype=np.int32)
    fake_idx = np.ascontiguousarray(fake_idx, dtype=np.int32)
    if real_idx.ndim != 2 or real_idx.shape != fake_idx.shape:
        raise ValueError("index tables of shapes %s and %s: both [S, m]" % (real_idx.shape, fake_idx.shape))
    L = kid_lib(handle)
    S, m = fake_idx.shape
    device = real.device
    ws = _workspace.get((device, S, m), lambda: L.kid_workspace_bytes(S, m), device)
    terms = torch.empty((S, 3), dtype=torch.float64, device=device)
    dtype = ids.FLOAT64 if real.dtype == torch.float64 else ids.FLOAT32
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        _abi.check(L.kid_subset_terms(real.data_ptr(), real.shape[0], fake.data_ptr(), fake.shape[0], real.shape[1],
                                      dtype, real_idx.ctypes.data, fake_idx.ctypes.data, S, m, terms.data_ptr(),
                                      ws.data_ptr(), ws.numel(), stream.cuda_stream), L)
    return terms

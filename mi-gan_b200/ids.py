"""P-IDS and U-IDS on the GPU: the paired and unpaired Inception discriminative scores of Co-Mod-GAN.

    res = inception_discriminative_scores(real_feats, fake_feats)   # [N, d] each; row i of both is the same photo
    res.p_ids, res.u_ids

The scores come from the linear SVM Co-Mod-GAN's authors fit with scikit-learn, `LinearSVC(dual=False)` (C = 1,
squared hinge, L2, the intercept regularised as a weight on a constant feature), on the real rows (label 1) and the
fake rows (label 0):

    U-IDS = the SVM's misclassification rate over the 2N rows (a decision value of exactly 0 counts as fake)
    P-IDS = the fraction of pairs whose fake decision value is above the real one

The library (`include/inception_b200.h`, `ids_scores`) finds the SVM's minimiser to float64 rounding by the finite Newton
method on the device, not sklearn's stopping point at tol=1e-4, so its objective is no worse than sklearn's and the
scores agree with sklearn's up to the rows sklearn leaves within its tolerance of the boundary.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import numpy as np
import torch

from . import _abi, fid

MAX_DIM = 4096
FLOAT32, FLOAT64 = 0, 1
STOP_RULES = {1: "active set", 2: "gradient"}

SYMBOLS = [
    ("ids_workspace_bytes", ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    ("ids_scores", ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                  ctypes.c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int),
                                  ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
]


def ids_lib(handle=None):
    """The product library (or `handle`, another build of csrc/ids.cu) with the IDS symbols bound."""
    return _abi.library(SYMBOLS, fid.lib(handle))


class IDSResult(NamedTuple):
    """The scores and the SVM behind them: coef [d] and intercept are its weights, objective its f(b*), residual
    |grad f(b*)| / |grad f(0)|, iterations the Newton iterations, stop_rule "active set" or "gradient"."""
    p_ids: float
    u_ids: float
    coef: np.ndarray
    intercept: float
    objective: float
    residual: float
    iterations: int
    stop_rule: str = "active set"


_workspace = _abi.Workspace()


def _prepare(name, x):
    """x as a 2-D float32 / float64 array or CUDA tensor; ValueError naming `name` when it is not one."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            x = x.detach().cpu().numpy()
        else:
            x = x.detach()
            if x.dtype not in (torch.float32, torch.float64):
                x = x.to(torch.float64)
    if not isinstance(x, torch.Tensor):
        x = np.asarray(x)
        if x.dtype not in (np.float32, np.float64):
            x = x.astype(np.float64)
    if x.ndim != 2:
        raise ValueError("%s must be an [N, d] feature array, got shape %s" % (name, tuple(x.shape)))
    return x


def inception_discriminative_scores(real, fake) -> IDSResult:
    """P-IDS and U-IDS of paired features real[i] / fake[i] ([N, d] each): CUDA float32 / float64 tensors, or numpy
    arrays, which are uploaded once.  Both sides are read at the wider of their two dtypes."""
    real, fake = _prepare("real", real), _prepare("fake", fake)
    if tuple(real.shape) != tuple(fake.shape):
        raise ValueError("real and fake must have the same shape (paired rows), got %s and %s"
                         % (tuple(real.shape), tuple(fake.shape)))
    n, d = (int(v) for v in real.shape)
    if n < 1:
        raise ValueError("real and fake hold no rows")
    if not 1 <= d <= MAX_DIM:
        raise ValueError("feature dimension %d outside 1..%d" % (d, MAX_DIM))
    if n * 2 * (d + 1) >= 2 ** 31:
        raise ValueError("%d pairs of %d features: n x 2 x (d + 1) reaches 2^31" % (n, d))
    for name, x in (("real", real), ("fake", fake)):
        finite = bool(torch.isfinite(x).all()) if isinstance(x, torch.Tensor) else bool(np.isfinite(x).all())
        if not finite:
            raise ValueError("%s has non-finite values" % name)
    wide = any(x.dtype in (np.float64, torch.float64) for x in (real, fake))
    cuda = [x for x in (real, fake) if isinstance(x, torch.Tensor)]
    device = cuda[0].device if cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        t = []
        for x in (real, fake):
            if not isinstance(x, torch.Tensor):
                x = torch.from_numpy(np.ascontiguousarray(x))
            t.append(x.to(device=device, dtype=torch.float64 if wide else torch.float32).contiguous())
        return _scores(t[0], t[1])


def _scores(real, fake, handle=None) -> IDSResult:
    """The library call on contiguous CUDA tensors of one device and one dtype."""
    L = ids_lib(handle)
    n, d = (int(v) for v in real.shape)
    device = real.device
    ws = _workspace.get((device, n, d), lambda: L.ids_workspace_bytes(n, d), device)
    coef = torch.empty(d, dtype=torch.float64, device=device)
    out = (ctypes.c_double * 5)()
    its = (ctypes.c_int * 2)()
    dtype = FLOAT64 if real.dtype == torch.float64 else FLOAT32
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        _abi.check(L.ids_scores(real.data_ptr(), fake.data_ptr(), n, d, dtype, coef.data_ptr(), out, its,
                                ws.data_ptr(), ws.numel(), stream.cuda_stream), L)
        coef = coef.cpu().numpy()
    return IDSResult(out[0], out[1], coef, out[2], out[3], out[4], its[0], STOP_RULES[its[1]])

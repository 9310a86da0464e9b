"""Float64 numpy oracle of the kernel Inception distance (Binkowski et al. 2018), the library's contract.

Real features Y [n_r, d], fake (composed) features X [n_f, d]; S = num_subsets subsets of m = min(n_r, n_f,
max_subset_size) rows, drawn by `rng = np.random.RandomState(seed)`: for each subset in order, first the fake rows
`rng.choice(n_f, m, replace=False)`, then the real rows `rng.choice(n_r, m, replace=False)` (StyleGAN2-ADA's order).
With k(u, v) = t t t, t = (u.v) / d + 1:

    Sxx = sum_{i != j} k(x_i, x_j),  Syy = sum_{i != j} k(y_i, y_j),  Sxy = sum_{i, j} k(x_i, y_j)
    e_s = ((Sxx + Syy) / (m - 1) - 2 Sxy / m) / m                   (the unbiased MMD^2 estimate of subset s)
    t = 0;  t += (Sxx + Syy) / (m - 1) - 2 Sxy / m  in subset order;  KID = t / S / m;  std = np.std(e)

StyleGAN2-ADA's `compute_kid` is this expression and order in float32.
"""
from typing import NamedTuple, Tuple

import numpy as np


class KID(NamedTuple):
    kid: float
    std: float
    terms: np.ndarray          # float64 [S, 3]: Sxx, Syy, Sxy
    estimates: np.ndarray      # float64 [S]: e_s


def subset_size(n_real: int, n_fake: int, max_subset_size: int = 1000) -> int:
    return min(int(n_real), int(n_fake), int(max_subset_size))


def draw(n_real: int, n_fake: int, num_subsets: int, m: int, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """(fake_idx, real_idx), int64 [S, m] each, drawn in the contract's order."""
    rng = np.random.RandomState(seed)
    fake_idx, real_idx = [], []
    for _ in range(num_subsets):
        fake_idx.append(rng.choice(n_fake, m, replace=False))
        real_idx.append(rng.choice(n_real, m, replace=False))
    return np.stack(fake_idx), np.stack(real_idx)


def kernel(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    t = a @ b.T / a.shape[1] + 1.0
    return t * t * t


def terms(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """[Sxx, Syy, Sxy] of one subset, x and y float64 [m, d]."""
    off = ~np.eye(len(x), dtype=bool)
    return np.array([kernel(x, x)[off].sum(), kernel(y, y)[off].sum(), kernel(x, y).sum()])


def finish(T: np.ndarray, m: int) -> Tuple[float, float, np.ndarray]:
    """(KID, std, e) from the terms [S, 3], accumulated in subset order."""
    t = 0.0
    e = []
    for sxx, syy, sxy in T.tolist():
        a = (sxx + syy) / (m - 1) - 2 * sxy / m
        t += a
        e.append(a / m)
    e = np.array(e, dtype=np.float64)
    return t / len(T) / m, float(np.std(e)), e


def kid(real, fake, num_subsets: int = 100, max_subset_size: int = 1000, seed: int = 0) -> KID:
    real, fake = np.asarray(real, np.float64), np.asarray(fake, np.float64)
    m = subset_size(len(real), len(fake), max_subset_size)
    if m < 2:
        raise ValueError("KID needs subsets of at least 2 rows, got m = %d" % m)
    fi, ri = draw(len(real), len(fake), num_subsets, m, seed)
    T = np.stack([terms(fake[a], real[b]) for a, b in zip(fi, ri)])
    value, std, e = finish(T, m)
    return KID(value, std, T, e)


def stylegan2_ada_float32(real, fake, num_subsets: int = 100, max_subset_size: int = 1000, seed: int = 0) -> float:
    """StyleGAN2-ADA's `compute_kid` on float32 features, with the seeded draws in place of the global RNG."""
    real, fake = np.asarray(real, np.float32), np.asarray(fake, np.float32)
    n = real.shape[1]
    m = subset_size(len(real), len(fake), max_subset_size)
    rng = np.random.RandomState(seed)
    t = 0
    for _ in range(num_subsets):
        x = fake[rng.choice(fake.shape[0], m, replace=False)]
        y = real[rng.choice(real.shape[0], m, replace=False)]
        a = (x @ x.T / n + 1) ** 3 + (y @ y.T / n + 1) ** 3
        b = (x @ y.T / n + 1) ** 3
        t += (a.sum() - np.diag(a).sum()) / (m - 1) - b.sum() * 2 / m
    return float(t / num_subsets / m)


def features(n: int, d: int, seed: int, shift: float = 0.0) -> np.ndarray:
    """Seeded non-negative float32 rows shaped like pool3 features (means of ReLU outputs)."""
    rng = np.random.RandomState(seed)
    return (np.abs(rng.standard_normal((n, d))) * 0.4 + shift * rng.standard_normal(d) ** 2).astype(np.float32)

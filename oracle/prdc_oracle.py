"""Float64 oracle of precision, recall, density and coverage (Kynkaanniemi et al. 2019, Naeem et al. 2020), the
library's contract.

Real rows Y [N, d], fake (composed) rows X [M, d], promoted to float64; squared Euclidean distances D(a, b) =
sum_c (a_c - b_c)^2, summed directly (not through |a|^2 + |b|^2 - 2 a.b), a chunk of rows at a time.

    r_i = the (k + 1)-th smallest of {D(Y_i, Y_j) : j}, row i itself included;  s_j the same within X
    precision = #{j : exists i, D(X_j, Y_i) <= r_i} / M          recall   = #{i : exists j, D(Y_i, X_j) <= s_j} / N
    density   = sum_j #{i : D(X_j, Y_i) <= r_i} / (k M)          coverage = #{i : min_j D(Y_i, X_j) <= r_i} / N

`margin` is the smallest |D - threshold| over every comparison made: a library whose distances and radii are within
rounding of these must give the same counts whenever the margin is above that rounding.

The rows may also be float64 torch tensors: the distance expression is the same and runs where the tensors are (the
library's tests use that at 10,000 rows, where numpy would take hours); everything after it is numpy.
"""
from typing import Iterator, NamedTuple, Tuple

import numpy as np


class PRDC(NamedTuple):
    counts: np.ndarray         # int64 [4]: the precision, recall, density and coverage counts
    precision: float
    recall: float
    density: float
    coverage: float
    margin: float
    r_real: np.ndarray         # float64 [N]
    r_fake: np.ndarray         # float64 [M]


def _numpy(x) -> np.ndarray:
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def sq_dists(a, b, chunk: int = 64) -> Iterator[Tuple[int, np.ndarray]]:
    """(start, D[start:start + c, :]) for chunks of a's rows: float64 sum of squared differences against every row of b."""
    for s in range(0, len(a), chunk):
        yield s, _numpy(((a[s:s + chunk, None, :] - b[None, :, :]) ** 2).sum(-1))


def radii(rows, k: int, chunk: int = 64) -> np.ndarray:
    """The (k + 1)-th smallest distance of each row to the rows of its set, itself included."""
    out = np.empty(len(rows))
    for s, D in sq_dists(rows, rows, chunk):
        out[s:s + len(D)] = np.partition(D, k, axis=1)[:, k]
    return out


def prdc(real, fake, k: int = 3, chunk: int = 64) -> PRDC:
    """The four metrics of real [N, d] and fake [M, d] (numpy arrays, promoted to float64, or float64 tensors)."""
    if isinstance(real, np.ndarray):
        real, fake = real.astype(np.float64), fake.astype(np.float64)
    N, M = len(real), len(fake)
    r, s = radii(real, k, chunk), radii(fake, k, chunk)
    covered = np.zeros(N, dtype=bool)
    recalled = np.zeros(N, dtype=bool)
    precision = density = 0
    margin = np.inf
    for j0, D in sq_dists(fake, real, chunk):          # D[j, i] = D(X_j, Y_i)
        sj = s[j0:j0 + len(D), None]
        near = D <= r[None, :]
        count = near.sum(1)
        precision += int((count > 0).sum())
        density += int(count.sum())
        covered |= near.any(0)
        recalled |= (D <= sj).any(0)
        margin = min(margin, float(np.abs(D - r[None, :]).min()), float(np.abs(D - sj).min()))
    counts = np.array([precision, int(recalled.sum()), density, int(covered.sum())], dtype=np.int64)
    return PRDC(counts, counts[0] / M, counts[1] / N, counts[2] / (k * M), counts[3] / N, margin, r, s)


def rounding_bound(real, fake) -> float:
    """A bound on the rounding a comparison of the library's can carry: its distance and its threshold each
    |a|^2 + |b|^2 - 2 a.b summed over d products, so at most 4 (d + 2) 2^-53 max|row|^2 each; taken 4 times over."""
    sq = [float(_numpy(((x.astype(np.float64) if isinstance(x, np.ndarray) else x) ** 2).sum(-1)).max())
          for x in (real, fake)]
    return 32 * (real.shape[1] + 4) * 2.0 ** -53 * max(sq)


def features(n: int, d: int, seed: int, shift: float = 0.0) -> np.ndarray:
    """Seeded non-negative float32 rows shaped like pool3 features (means of ReLU outputs)."""
    rng = np.random.RandomState(seed)
    return (np.abs(rng.standard_normal((n, d))) * 0.4 + shift * rng.standard_normal(d) ** 2).astype(np.float32)


def integer_features(n: int, d: int, seed: int, high: int = 3, dup_of=None, dups: int = 0) -> np.ndarray:
    """Small integer-valued float32 rows, where every distance is exact and ties are everywhere; with `dup_of`, the
    first `dups` rows are copies of rows of `dup_of`, and a few rows repeat within the set too."""
    rng = np.random.RandomState(seed)
    x = rng.randint(0, high, (n, d)).astype(np.float32)
    x[n // 2:n // 2 + max(1, n // 10)] = x[:max(1, n // 10)]
    if dup_of is not None and dups:
        x[:dups] = dup_of[rng.choice(len(dup_of), dups, replace=False)]
    return x

"""Float64 numpy oracle of the Fréchet distance, by the symmetric eigenvalue route.

tr sqrt(S1 S2) = sum_i sqrt(max(lambda_i(M), 0)) with M = D^1/2 V^T S2 V D^1/2 and S1 = V D V^T (negative d clamped to
0): the eigenvalues of S1 S2 are those of M, and nothing forms the non-symmetric product.  Test inputs:

- commuting_pair(): S1 = Q diag(d1) Q^T and S2 = Q diag(d2) Q^T, whose trace is exactly sum sqrt(max(d1 d2, 0));
- feature_stats(): the mean and covariance of ReLU'd correlated Gaussian features, like Inception pool3 features.
"""
import numpy as np


def _cut(ev, cutoff):
    """ev with the values at or below the numerical-rank cutoff d 2^-52 max|ev| (numpy's matrix_rank) set to 0."""
    if not cutoff:
        return np.maximum(ev, 0.0)
    return np.where(ev > len(ev) * np.finfo(np.float64).eps * np.abs(ev).max(), ev, 0.0)


def trace_sqrt(sigma1, sigma2, cutoff=False):
    """sum sqrt(max(lambda, 0)) over the eigenvalues of sigma1 sigma2, by two numpy eigh calls.  With `cutoff`,
    sigma1's eigenvalues at or below the numerical-rank cutoff count as 0, as the library counts them."""
    s1, s2 = np.atleast_2d(np.asarray(sigma1, np.float64)), np.atleast_2d(np.asarray(sigma2, np.float64))
    s1, s2 = (s1 + s1.T) / 2, (s2 + s2.T) / 2
    d, v = np.linalg.eigh(s1)
    sd = np.sqrt(_cut(d, cutoff))
    m = (v.T @ s2 @ v) * sd[:, None] * sd[None, :]
    lam = np.linalg.eigvalsh((m + m.T) / 2)
    return float(np.sqrt(np.maximum(lam, 0.0)).sum())


def frechet_distance(mu1, sigma1, mu2, sigma2, cutoff=False):
    """(fid, tr sqrt(sigma1 sigma2)) by the eigh route, in pytorch_fid's order of the terms."""
    diff = np.asarray(mu1, np.float64) - np.asarray(mu2, np.float64)
    ts = trace_sqrt(sigma1, sigma2, cutoff)
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * ts), ts


def random_orthogonal(d, rng):
    q, r = np.linalg.qr(rng.standard_normal((d, d)))
    return q * np.sign(np.diag(r))[None, :]


def commuting_pair(d, d1, d2, seed=0):
    """(sigma1, sigma2, exact tr sqrt(sigma1 sigma2)) for eigenvalues d1, d2 (length d) on one seeded random basis."""
    rng = np.random.default_rng(seed)
    q = random_orthogonal(d, rng)
    d1, d2 = np.asarray(d1, np.float64), np.asarray(d2, np.float64)
    s1, s2 = (q * d1[None, :]) @ q.T, (q * d2[None, :]) @ q.T
    s1, s2 = (s1 + s1.T) / 2, (s2 + s2.T) / 2
    return s1, s2, float(np.sqrt(np.maximum(d1 * d2, 0.0)).sum())


def log_spectrum(d, lo, hi, rank=None, seed=0):
    """d eigenvalues log-spaced in [lo, hi] in a seeded order; with `rank`, all but `rank` of them are 0."""
    rng = np.random.default_rng(seed)
    ev = np.zeros(d)
    r = d if rank is None else rank
    ev[:r] = np.logspace(np.log10(lo), np.log10(hi), r)
    return ev[rng.permutation(d)]


def feature_stats(N, d, seed=0, rank=64):
    """(mu, sigma) of N rows of relu(z L + b): z standard normal in `rank` latent dimensions mixed into d features."""
    rng = np.random.default_rng(seed)
    mix = rng.standard_normal((rank, d)) / np.sqrt(rank)
    noise = 0.3 * rng.standard_normal((N, d))
    f = np.maximum(rng.standard_normal((N, rank)) @ mix + noise + 0.2 * rng.standard_normal(d)[None, :], 0.0)
    return f.mean(axis=0), np.atleast_2d(np.cov(f, rowvar=False))

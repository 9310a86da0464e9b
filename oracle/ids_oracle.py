"""Float64 numpy oracle of the Inception discriminative scores: the finite Newton solve of LinearSVC(dual=False).

Rows x~_i = [x_i, 1], labels y = +1 (real) / -1 (fake), and f(b) = 1/2 |b|^2 + C sum_i max(0, 1 - y_i b.x~_i)^2 with
C = 1 (liblinear regularises the intercept as an ordinary weight).  The solver and its stop rules are the library's:
Newton point b~ = (I + 2C X~_I^T X~_I)^-1 2C X~_I^T y_I on the active set I = {y o < 1}; stop when the active set at b~
is I, or when |grad f| <= 1e-12 |grad f(0)|; otherwise an exact line search along b~ - b.  Also seeded feature sets.
"""
from typing import NamedTuple

import numpy as np

C = 1.0
GRAD_TOL = 1e-12
MAX_ITER = 100


def augment(real, fake):
    """(X~ [2n, d + 1], y [2n]) in float64: the real rows, then the fake rows."""
    real, fake = np.asarray(real, np.float64), np.asarray(fake, np.float64)
    X = np.concatenate([real, fake])
    return np.concatenate([X, np.ones((X.shape[0], 1))], axis=1), np.concatenate([np.ones(len(real)), -np.ones(len(fake))])


def objective(beta, X, y):
    """f(b) = 1/2 |b|^2 + C sum max(0, 1 - y X~ b)^2 (beta includes the intercept as its last entry)."""
    m = np.maximum(0.0, 1.0 - y * (X @ beta))
    return 0.5 * float(beta @ beta) + C * float(m @ m)


def gradient(beta, X, y):
    """grad f(b) = b - 2C X~_I^T (y - o)_I, I = {y o < 1}."""
    o = X @ beta
    act = y * o < 1.0
    return beta - 2 * C * (X[act].T @ (y[act] - o[act]))


def scores(o_real, o_fake):
    """(P-IDS, U-IDS) from the decision values: U counts o = 0 as fake (sklearn's predict), P is strict."""
    n = len(o_real)
    return float(np.mean(o_fake > o_real)), float(((o_real <= 0).sum() + (o_fake > 0).sum()) / (2 * n))


def line_search(beta, delta, o, od, y):
    """argmin_{t >= 0} f(b + t d), with od = X~ d: bracket the root of the piecewise-linear phi', bisect until no row
    changes sides inside the bracket, then solve that segment."""
    a, e = 1.0 - y * o, y * od
    bd, dd = float(beta @ delta), float(delta @ delta)

    def pq(t):
        act = a - t * e > 0
        return bd - 2 * C * float(a[act] @ e[act]), dd + 2 * C * float(e[act] @ e[act])

    lo, hi = 0.0, 1.0
    for _ in range(64):
        P, Q = pq(hi)
        if P + hi * Q >= 0:
            break
        lo, hi = hi, 2 * hi
    for _ in range(256):
        mid = 0.5 * (lo + hi)
        if not np.any((a - lo * e > 0) != (a - hi * e > 0)):
            P, Q = pq(mid)
            return min(max(-P / Q if Q > 0 else lo, lo), hi)
        if not lo < mid < hi:
            return mid
        P, Q = pq(mid)
        if P + mid * Q < 0:
            lo = mid
        else:
            hi = mid
    return 0.5 * (lo + hi)


class Solution(NamedTuple):
    p_ids: float
    u_ids: float
    coef: np.ndarray
    intercept: float
    objective: float
    residual: float
    iterations: int
    stop_rule: str
    decision: np.ndarray          # o over the 2n rows, real then fake


def solve(real, fake):
    """The minimiser of f and the scores at it."""
    X, y = augment(real, fake)
    n = len(y) // 2
    beta = np.zeros(X.shape[1])
    o = np.zeros(len(y))
    g0 = None
    prev = None
    for k in range(MAX_ITER + 1):
        g = gradient(beta, X, y)
        gn = float(np.linalg.norm(g))
        g0 = gn if g0 is None else g0
        act = y * o < 1.0
        if k > 0 and np.array_equal(act, prev):
            rule = "active set"
            break
        if gn <= GRAD_TOL * g0:
            rule = "gradient"
            break
        if k == MAX_ITER:
            raise RuntimeError("no convergence in %d iterations" % MAX_ITER)
        XI = X[act]
        G = np.eye(X.shape[1]) + 2 * C * (XI.T @ XI)
        bbar = np.linalg.solve(G, 2 * C * (XI.T @ y[act]))
        ob = X @ bbar
        if np.array_equal(y * ob < 1.0, act):
            beta, o, prev = bbar, ob, act
            continue
        t = line_search(beta, bbar - beta, o, ob - o, y)
        beta = beta + t * (bbar - beta)
        o = X @ beta
        prev = None
    p, u = scores(o[:n], o[n:])
    return Solution(p, u, beta[:-1].copy(), float(beta[-1]), objective(beta, X, y), gn / g0 if g0 > 0 else 0.0, k,
                    rule, o)


def features(n, d, kind, seed=0):
    """Seeded (real, fake) [n, d] float32 features, gamma-distributed like Inception pool3 activations.
    kind "overlap": fake = real's distribution slightly shifted (the classes overlap); "separable": a larger shift."""
    rng = np.random.default_rng(seed)
    shift = {"overlap": 0.02, "separable": 0.3}[kind]
    real = rng.gamma(2.0, 0.25, (n, d))
    fake = rng.gamma(2.0, 0.25, (n, d)) * (1.0 + shift * rng.random(d))
    return real.astype(np.float32), fake.astype(np.float32)

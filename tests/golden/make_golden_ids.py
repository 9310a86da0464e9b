"""Writes tests/golden/ids.npz: sklearn's LinearSVC(dual=False) on paired feature sets, as Co-Mod-GAN's authors compute
P-IDS and U-IDS, for tests/test_ids_emul.py and tests/test_ids_gpu.py (which need no sklearn).

    python tests/golden/make_golden_ids.py

Features are stored as uint8 multiples of 1/64 (exact in float32).  Per case <c>: <c>_real / <c>_fake [n, d] uint8,
sklearn's <c>_coef, <c>_intercept, <c>_decision (real rows, then fake), <c>_n_iter, <c>_u_ids, <c>_p_ids and
<c>_objective (f at sklearn's coefficients, float64), and <c>_u_rows / <c>_p_rows: by how many rows the float64
finite-Newton oracle's counts differ from sklearn's (sklearn stops at tol=1e-4, short of the minimiser).
"""
import os
import sys

import numpy as np
import sklearn
from sklearn.svm import LinearSVC

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ids_oracle as O  # noqa: E402

# (name, n, d, varying columns, relative shift of the fake columns)
CASES = [("overlap2048", 400, 2048, 48, 0.1), ("separable2048", 100, 2048, 2048, 0.3),
         ("n197", 197, 256, 256, 0.02), ("d37", 300, 37, 37, 0.1)]


def quantised(rng, n, d, vary, shift):
    """uint8 real / fake: gamma features in the first `vary` columns (the fake ones scaled by up to 1 + shift), one
    constant per column in the rest, the same for both."""
    const = rng.gamma(2.0, 0.25, d)
    scale = 1.0 + shift * rng.random(vary)
    out = []
    for s in (np.ones(vary), scale):
        x = np.broadcast_to(const, (n, d)).copy()
        x[:, :vary] = rng.gamma(2.0, 0.25, (n, vary)) * s
        out.append(np.clip(np.rint(x * 64), 0, 255).astype(np.uint8))
    return out


def main():
    rng = np.random.default_rng(2024)
    out = {"sklearn_version": np.array(sklearn.__version__)}
    for name, n, d, vary, shift in CASES:
        qr, qf = quantised(rng, n, d, vary, shift)
        real, fake = qr / 64.0, qf / 64.0
        svm = LinearSVC(dual=False).fit(np.concatenate([real, fake]), [1] * n + [0] * n)
        dec = svm.decision_function(np.concatenate([real, fake]))
        u = 1 - svm.score(np.concatenate([real, fake]), [1] * n + [0] * n)
        p = float(np.mean(dec[n:] > dec[:n]))
        X, y = O.augment(real, fake)
        beta = np.concatenate([svm.coef_[0], svm.intercept_])
        sol = O.solve(real, fake)
        print("%s: sklearn %d iterations, U %.6f P %.6f f %.12g; oracle %d iterations (%s), U %.6f P %.6f f %.12g"
              % (name, svm.n_iter_, u, p, O.objective(beta, X, y), sol.iterations, sol.stop_rule, sol.u_ids, sol.p_ids,
                 sol.objective))
        out.update({name + "_real": qr, name + "_fake": qf, name + "_coef": svm.coef_[0], name + "_intercept":
                    np.float64(svm.intercept_[0]), name + "_decision": dec, name + "_n_iter": np.int64(svm.n_iter_),
                    name + "_u_ids": np.float64(u), name + "_p_ids": np.float64(p),
                    name + "_objective": np.float64(O.objective(beta, X, y)),
                    name + "_u_rows": np.int64(round(abs(sol.u_ids - u) * 2 * n)),
                    name + "_p_rows": np.int64(round(abs(sol.p_ids - p) * n))})
    path = os.path.join(HERE, "ids.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()

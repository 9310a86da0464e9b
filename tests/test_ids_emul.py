"""P-IDS and U-IDS without a GPU: the float64 finite-Newton oracle against sklearn's LinearSVC(dual=False) on the stored
fixture, the library's solver in the emulation build (the same phases, DMMA tile products as loops in their k order)
against the oracle, every refusal of the C ABI, and the evaluation command's `--ids` argument handling."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, ids  # noqa: E402
from oracle import ids_oracle as O  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ids.npz")
CASES = ["overlap2048", "separable2048", "n197", "d37"]
GUARD = -7.25
# Emulated coefficients against the oracle, max |coef - oracle| / max |oracle coef|: both reach the minimiser to
# float64 rounding by different sums; measured at most 8.1e-12 on these sets.
COEF_REL = 1e-10


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(build_emul.CSRC, s) for s in ("inception_abi.cu", "ids.cu", "abi_error.cu")]
    L = ids.ids_lib(ctypes.CDLL(build_emul._compile("ids_emul", srcs)))
    L.migan_last_error.restype = ctypes.c_char_p
    return L


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def case(g, name):
    return (g[name + "_real"] / np.float32(64)).astype(np.float32), (g[name + "_fake"] / np.float32(64)).astype(np.float32)


class Workspace:
    """256-byte aligned host memory with guard bytes after the `nbytes` the call may use."""

    def __init__(self, nbytes, guard=512):
        self.buf = (ctypes.c_uint8 * (nbytes + guard + 256))()
        self.base = (ctypes.addressof(self.buf) + 255) // 256 * 256
        self.nbytes, self.guard = nbytes, guard
        ctypes.memset(self.base + nbytes, 0xA5, guard)

    def guard_intact(self):
        return bytes((ctypes.c_uint8 * self.guard).from_address(self.base + self.nbytes)) == b"\xa5" * self.guard


def call(L, real, fake):
    """The emulated ids_scores: (out[5], coef, iterations[2]), with the workspace and output guards checked."""
    n, d = real.shape
    ws = Workspace(L.ids_workspace_bytes(n, d))
    coef = np.full(d + 2, GUARD)
    out = (ctypes.c_double * 7)(GUARD, 0, 0, 0, 0, 0, GUARD)
    its = (ctypes.c_int * 4)(-5, 0, 0, -5)
    dtype = ids.FLOAT64 if real.dtype == np.float64 else ids.FLOAT32
    rc = L.ids_scores(real.ctypes.data, fake.ctypes.data, n, d, dtype, coef[1:].ctypes.data,
                      ctypes.cast(ctypes.byref(out, 8), ctypes.POINTER(ctypes.c_double)),
                      ctypes.cast(ctypes.byref(its, 4), ctypes.POINTER(ctypes.c_int)), ws.base, ws.nbytes, None)
    _abi.check(rc, L)
    assert ws.guard_intact() and out[0] == GUARD and out[6] == GUARD and its[0] == -5 and its[3] == -5
    assert coef[0] == GUARD and coef[-1] == GUARD
    return np.array(out[1:6]), coef[1:-1], (its[1], its[2])


# -- the oracle against sklearn ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", CASES)
def test_oracle_against_sklearn(golden, name):
    real, fake = case(golden, name)
    n = len(real)
    sol = O.solve(real, fake)
    print("%s: oracle f %.15g (sklearn %.15g), residual %.2e, %d iterations (%s; sklearn %d, version %s)"
          % (name, sol.objective, golden[name + "_objective"], sol.residual, sol.iterations, sol.stop_rule,
             golden[name + "_n_iter"], golden["sklearn_version"]))
    assert sol.objective <= golden[name + "_objective"] * (1 + 1e-12)
    X, y = O.augment(real, fake)
    beta = np.concatenate([sol.coef, [sol.intercept]])
    g = np.linalg.norm(O.gradient(beta, X, y)) / np.linalg.norm(O.gradient(np.zeros_like(beta), X, y))
    assert g <= 1e-12 and sol.residual <= 1e-12
    assert abs(sol.u_ids - golden[name + "_u_ids"]) * 2 * n <= golden[name + "_u_rows"] + 1e-9
    assert abs(sol.p_ids - golden[name + "_p_ids"]) * n <= golden[name + "_p_rows"] + 1e-9
    # sklearn's own decision values give its stored scores (the contract's formulas; U-IDS was stored as 1 - score)
    dec = golden[name + "_decision"]
    p, u = O.scores(dec[:n], dec[n:])
    assert p == golden[name + "_p_ids"] and u == pytest.approx(float(golden[name + "_u_ids"]), abs=1e-12)


# -- the emulated runtime against the oracle ----------------------------------------------------------------------

def _check(out, coef, its, sol):
    scale = max(float(np.abs(sol.coef).max()), abs(sol.intercept), 1e-300)
    err = max(float(np.abs(coef - sol.coef).max()), abs(out[2] - sol.intercept)) / scale
    print("P %r U %r f %.15g (oracle %.15g), residual %.2e, %d iterations (rule %d; oracle %d, %s), coef err %.2e"
          % (out[0], out[1], out[3], sol.objective, out[4], its[0], its[1], sol.iterations, sol.stop_rule, err))
    assert (out[0], out[1]) == (sol.p_ids, sol.u_ids)
    assert err <= COEF_REL
    assert out[3] <= sol.objective * (1 + 1e-12)
    assert its[1] in (1, 2) and 0 <= its[0] <= 100


def test_emulation_at_2048_features(emul):
    real, fake = O.features(200, 2048, "overlap", seed=1)
    out, coef, its = call(emul, real, fake)
    _check(out, coef, its, O.solve(real, fake))
    again = call(emul, real, fake)
    assert out.tobytes() == again[0].tobytes() and coef.tobytes() == again[1].tobytes() and its == again[2]


@pytest.mark.parametrize("name", ["n197", "d37"])
def test_emulation_on_the_fixture(emul, golden, name):
    real, fake = case(golden, name)
    out, coef, its = call(emul, real, fake)
    _check(out, coef, its, O.solve(real, fake))
    assert out[3] <= golden[name + "_objective"] * (1 + 1e-12)
    wide = call(emul, real.astype(np.float64), fake.astype(np.float64))
    assert wide[0].tobytes() == out.tobytes() and wide[1].tobytes() == coef.tobytes()   # exact promotion


@pytest.mark.parametrize("n,d,kind", [(1, 5, "overlap"), (1, 64, "separable"), (2, 63, "overlap"),
                                      (150, 37, "separable"), (130, 128, "overlap")])
def test_emulation_edges(emul, n, d, kind):
    real, fake = O.features(n, d, kind, seed=n + d)
    out, coef, its = call(emul, real, fake)
    _check(out, coef, its, O.solve(real, fake))


def test_identical_sides_stop_at_zero(emul):
    real, _ = O.features(3, 10, "overlap", seed=2)
    out, coef, its = call(emul, real, real.copy())
    assert np.all(coef == 0) and out[2] == 0 and its == (0, 2)   # grad f(0) = 0: b* = 0
    assert out[0] == 0.0 and out[1] == 0.5                        # o = 0: every real row counts as fake


# -- refusals ----------------------------------------------------------------------------------------------------------

def test_workspace_bytes(emul):
    assert emul.ids_workspace_bytes(0, 2048) == 0
    assert emul.ids_workspace_bytes(10, 0) == 0
    assert emul.ids_workspace_bytes(10, 4097) == 0
    assert emul.ids_workspace_bytes(2 ** 30 // 2049 + 1, 2048) == 0
    assert emul.ids_workspace_bytes(2 ** 30 // 2049, 2048) > 0
    assert emul.ids_workspace_bytes(36500, 2048) < 100_000_000
    assert emul.ids_workspace_bytes(36500, 2048) > 2112 * 2112 * 8


def _refused(L, rc, text):
    assert rc == _abi.ERR_INVALID, (rc, L.migan_last_error())
    assert text in L.migan_last_error().decode()


def test_refusals(emul):
    L = emul
    n, d = 4, 7
    x = np.zeros((n, d), np.float32)
    ws = Workspace(L.ids_workspace_bytes(n, d))
    coef = np.zeros(d)
    out, its = (ctypes.c_double * 5)(), (ctypes.c_int * 2)()
    args = [x.ctypes.data, x.ctypes.data, n, d, ids.FLOAT32, coef.ctypes.data, out, its, ws.base, ws.nbytes, None]

    def with_(k, v):
        a = list(args)
        a[k] = v
        return L.ids_scores(*a)
    for k in (0, 1, 5, 6, 7):
        _refused(L, with_(k, None), "null")
    _refused(L, with_(8, None), "null workspace")
    _refused(L, with_(2, 0), "n 0 < 1")
    _refused(L, with_(3, 0), "dim 0 outside")
    _refused(L, with_(3, 4097), "dim 4097 outside")
    _refused(L, with_(2, 2 ** 31 // (2 * 8)), "2^31")
    _refused(L, with_(4, 7), "dtype 7")
    _refused(L, with_(9, ws.nbytes - 8), "needed")
    _refused(L, with_(8, ws.base + 8), "aligned")
    for bad in (np.nan, np.inf):
        y = x.copy()
        y[2, 3] = bad
        _refused(L, with_(1, y.ctypes.data), "non-finite")
    assert ws.guard_intact()


def test_python_checks_refuse_before_the_device():
    x = np.zeros((4, 8), np.float32)
    with pytest.raises(ValueError, match="same shape"):
        ids.inception_discriminative_scores(x, np.zeros((4, 9), np.float32))
    with pytest.raises(ValueError, match="no rows"):
        ids.inception_discriminative_scores(x[:0], x[:0])
    with pytest.raises(ValueError, match="outside 1..4096"):
        ids.inception_discriminative_scores(np.zeros((2, 4097)), np.zeros((2, 4097)))
    with pytest.raises(ValueError, match=r"real must be an \[N, d\]"):
        ids.inception_discriminative_scores(np.zeros(5), np.zeros(5))
    bad = x.copy()
    bad[0, 0] = np.inf
    with pytest.raises(ValueError, match="real has non-finite"):
        ids.inception_discriminative_scores(bad, x)
    with pytest.raises(ValueError, match="fake has non-finite"):
        ids.inception_discriminative_scores(x, bad)


# -- the evaluation command ---------------------------------------------------------------------------------------

def test_ids_flag_parses():
    from migan_b200 import evaluate_fid_lpips as E
    base = ["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", "r"]
    assert E.get_args(base).ids is False
    assert E.get_args(base + ["--ids"]).ids is True


def test_ids_with_real_stats_is_refused_before_any_work(tmp_path):
    from migan_b200 import evaluate_fid_lpips as E
    missing = tmp_path / "nothing_here"          # no images, no model: the refusal comes first
    with pytest.raises(ValueError, match="--real-stats"):
        E.evaluate("migan-256", missing / "m.pt", missing, real_stats=(np.zeros(2048), np.eye(2048)), ids=True)
    with pytest.raises(ValueError, match="--real-stats"):
        E.main(["--model-name", "migan-256", "--model-path", str(missing / "m.pt"), "--real-dir", str(missing),
                "--real-stats", str(missing / "s.npz"), "--ids", "--device", "cuda"])


def test_merge_without_real_features_cannot_keep_them():
    from migan_b200 import evaluate_fid_lpips as E
    with pytest.raises(ValueError, match="real features"):
        E.Merge(4, "cpu", real_features=False, keep_features=True)

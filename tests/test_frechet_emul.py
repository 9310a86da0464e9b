"""The Fréchet distance without a GPU: the library's eigensolver, M product and reductions in the emulation build (the
same pair and update phases, tile products as loops in the DMMA's k order) against exact answers of commuting pairs
and against the float64 eigh oracle, fid_stats_mean_cov against FeatureStatistics.mean_cov()'s arithmetic, and every
refusal of the C ABI."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, fid  # noqa: E402
from oracle import frechet_oracle as O  # noqa: E402

DIMS = [1, 2, 7, 64, 100, 257]
GUARD = -7.25


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(build_emul.CSRC, s) for s in ("inception_abi.cu", "frechet.cu", "abi_error.cu")]
    L = fid.frechet_lib(ctypes.CDLL(build_emul._compile("frechet_emul", srcs)))
    L.migan_last_error.restype = ctypes.c_char_p
    return L


class Workspace:
    """256-byte aligned host memory with guard bytes after the `nbytes` the call may use."""

    def __init__(self, nbytes, guard=512):
        self.buf = (ctypes.c_uint8 * (nbytes + guard + 256))()
        self.base = (ctypes.addressof(self.buf) + 255) // 256 * 256
        self.nbytes, self.guard = nbytes, guard
        ctypes.memset(self.base + nbytes, 0xA5, guard)

    def guard_intact(self):
        return bytes((ctypes.c_uint8 * self.guard).from_address(self.base + self.nbytes)) == b"\xa5" * self.guard


def call(L, mu1, s1, mu2, s2, ws=None):
    """(out[4], sweeps[2]) of the emulated fid_frechet_distance, with the workspace and output guards checked."""
    a = [np.ascontiguousarray(x, np.float64) for x in (mu1, s1, mu2, s2)]
    d = a[0].shape[0]
    ws = ws or Workspace(L.fid_frechet_workspace_bytes(d))
    out = (ctypes.c_double * 6)(GUARD, 0, 0, 0, 0, GUARD)
    sweeps = (ctypes.c_int * 4)(-5, 0, 0, -5)
    rc = L.fid_frechet_distance(*[x.ctypes.data for x in a], d, ctypes.cast(ctypes.byref(out, 8),
                                ctypes.POINTER(ctypes.c_double)), ctypes.cast(ctypes.byref(sweeps, 4),
                                ctypes.POINTER(ctypes.c_int)), ws.base, ws.nbytes, None)
    _abi.check(rc, L)
    assert ws.guard_intact() and out[0] == GUARD and out[5] == GUARD and sweeps[0] == -5 and sweeps[3] == -5
    return np.array(out[1:5]), (sweeps[1], sweeps[2])


def bound(T, oracle_err):
    """The accuracy rule: 1e-12 of tr S1 + tr S2, or twice the eigh oracle's own error on rank-deficient input."""
    return max(1e-12 * T, 2 * abs(oracle_err), 1e-14)


@pytest.mark.parametrize("d", DIMS)
def test_commuting_full_rank_is_exact(emul, d):
    ev1, ev2 = O.log_spectrum(d, 1e-6, 1e2, seed=1), O.log_spectrum(d, 1e-5, 1e1, seed=2)
    s1, s2, exact = O.commuting_pair(d, ev1, ev2, seed=3)
    mu1, mu2 = np.linspace(0, 1, d), np.linspace(1, 0, d)
    out, sweeps = call(emul, mu1, s1, mu2, s2)
    T = np.trace(s1) + np.trace(s2)
    assert abs(out[3] - exact) <= 1e-12 * T, (out[3], exact)
    diff = mu1 - mu2
    assert out[0] == pytest.approx(diff.dot(diff), rel=1e-14, abs=1e-300)
    assert out[1] == pytest.approx(np.trace(s1), rel=1e-14) and out[2] == pytest.approx(np.trace(s2), rel=1e-14)
    assert 0 <= sweeps[0] <= 40 and 0 <= sweeps[1] <= 40


@pytest.mark.parametrize("d", DIMS)
def test_features_against_oracle(emul, d):
    mu1, s1 = O.feature_stats(3 * d + 5, d, seed=5)
    mu2, s2 = O.feature_stats(2 * d + 9, d, seed=6)
    out, _ = call(emul, mu1, s1, mu2, s2)
    want, ts = O.frechet_distance(mu1, s1, mu2, s2)
    T = np.trace(s1) + np.trace(s2)
    assert abs(out[3] - ts) <= 1e-11 * T, (out[3], ts)
    assert abs((out[0] + out[1] + out[2] - 2 * out[3]) - want) <= 3e-11 * T


@pytest.mark.parametrize("d", [7, 100])
def test_rank_deficient(emul, d):
    r1, r2 = max(1, d // 4), max(1, d // 3)
    ev1, ev2 = O.log_spectrum(d, 1e-3, 1e1, rank=r1, seed=7), O.log_spectrum(d, 1e-3, 1e1, rank=r2, seed=8)
    s1, s2, exact = O.commuting_pair(d, ev1, ev2, seed=9)
    out, _ = call(emul, np.zeros(d), s1, np.zeros(d), s2)
    oracle_err = O.trace_sqrt(s1, s2) - exact
    assert abs(out[3] - exact) <= bound(np.trace(s1) + np.trace(s2), oracle_err), (out[3], exact, oracle_err)


def test_small_negative_eigenvalues_are_clamped(emul):
    d = 64
    ev1 = O.log_spectrum(d, 1e-2, 1e1, seed=11)
    ev1[:5] = -1e-13          # rounding-sized negative eigenvalues, as np.cov can leave
    ev2 = O.log_spectrum(d, 1e-2, 1e1, seed=12)
    s1, s2, _ = O.commuting_pair(d, ev1, ev2, seed=13)
    exact = float(np.sqrt(np.maximum(ev1, 0) * ev2).sum())
    out, _ = call(emul, np.zeros(d), s1, np.zeros(d), s2)
    assert np.isfinite(out).all()
    assert abs(out[3] - exact) <= 1e-11 * (np.trace(s1) + np.trace(s2))


def test_equal_and_scaled_covariances(emul):
    d = 100
    mu1, s1 = O.feature_stats(400, d, seed=21)
    mu2 = mu1 + 0.01 * np.arange(d)
    T = 2 * np.trace(s1)
    out, _ = call(emul, mu1, s1, mu2, s1)
    dm = (mu1 - mu2).dot(mu1 - mu2)
    assert abs(out[3] - np.trace(s1)) <= 1e-12 * T
    assert abs(out[0] + out[1] + out[2] - 2 * out[3] - dm) <= 1e-12 * T
    c = 1.7
    out, _ = call(emul, mu1, s1, mu1, c * c * s1)
    assert abs(out[3] - c * np.trace(s1)) <= 1e-12 * (1 + c * c) * np.trace(s1)


def test_repeat_calls_are_bitwise_equal(emul):
    d = 100
    mu1, s1 = O.feature_stats(150, d, seed=31)
    mu2, s2 = O.feature_stats(170, d, seed=32)
    a, sa = call(emul, mu1, s1, mu2, s2)
    b, sb = call(emul, mu1, s1, mu2, s2)
    assert a.tobytes() == b.tobytes() and sa == sb


def test_mean_cov_is_bitwise_the_host_arithmetic(emul):
    rng = np.random.default_rng(41)
    d, count = 33, 57
    shift, s1 = rng.standard_normal(d) * 100, rng.standard_normal(d) * 3
    f = rng.standard_normal((count, d))
    s2 = f.T @ f
    mu = np.full(d + 2, GUARD)
    sigma = np.full(d * d + 2, GUARD)
    _abi.check(emul.fid_stats_mean_cov(shift.ctypes.data, s1.ctypes.data, s2.ctypes.data, count, d, mu[1:].ctypes.data,
                                       sigma[1:].ctypes.data, None), emul)
    n = float(count)
    want_mu, want_sigma = shift + s1 / n, (s2 - np.outer(s1, s1) / n) / (n - 1)   # FeatureStatistics.mean_cov()
    assert mu[1:-1].tobytes() == want_mu.tobytes()
    assert sigma[1:-1].tobytes() == want_sigma.reshape(-1).tobytes()
    assert mu[0] == mu[-1] == sigma[0] == sigma[-1] == GUARD


def test_workspace_bytes(emul):
    assert emul.fid_frechet_workspace_bytes(0) == 0
    assert emul.fid_frechet_workspace_bytes(-3) == 0
    assert emul.fid_frechet_workspace_bytes(4097) == 0
    assert emul.fid_frechet_workspace_bytes(2048) >= 4 * 2048 * 2048 * 8
    assert emul.fid_frechet_workspace_bytes(2048) < 150_000_000
    assert emul.fid_frechet_workspace_bytes(1) == emul.fid_frechet_workspace_bytes(64)


def _refused(L, rc, code, text):
    assert rc == code, (rc, L.migan_last_error())
    assert text in L.migan_last_error().decode()


def test_refusals(emul):
    L = emul
    d = 7
    mu, s = np.zeros(d), np.eye(d)
    ws = Workspace(L.fid_frechet_workspace_bytes(d))
    out = (ctypes.c_double * 4)()
    p = mu.ctypes.data, s.ctypes.data, mu.ctypes.data, s.ctypes.data
    _refused(L, L.fid_frechet_distance(*p, 0, out, None, ws.base, ws.nbytes, None), _abi.ERR_INVALID, "dim 0")
    _refused(L, L.fid_frechet_distance(*p, 4097, out, None, ws.base, 1 << 40, None), _abi.ERR_INVALID, "dim 4097")
    for k in range(4):
        q = list(p)
        q[k] = None
        _refused(L, L.fid_frechet_distance(*q, d, out, None, ws.base, ws.nbytes, None), _abi.ERR_INVALID, "null")
    _refused(L, L.fid_frechet_distance(*p, d, None, None, ws.base, ws.nbytes, None), _abi.ERR_INVALID, "null")
    _refused(L, L.fid_frechet_distance(*p, d, out, None, None, ws.nbytes, None), _abi.ERR_INVALID, "null workspace")
    _refused(L, L.fid_frechet_distance(*p, d, out, None, ws.base, ws.nbytes - 8, None), _abi.ERR_WORKSPACE, "needed")
    _refused(L, L.fid_frechet_distance(*p, d, out, None, ws.base + 8, ws.nbytes, None), _abi.ERR_WORKSPACE, "aligned")
    bad = np.eye(d)
    bad[2, 3] = bad[3, 2] = np.nan
    _refused(L, L.fid_frechet_distance(mu.ctypes.data, bad.ctypes.data, mu.ctypes.data, s.ctypes.data, d, out, None,
                                       ws.base, ws.nbytes, None), _abi.ERR_INVALID, "not finite")
    assert ws.guard_intact()
    f = np.zeros(d)
    _refused(L, L.fid_stats_mean_cov(f.ctypes.data, f.ctypes.data, s.ctypes.data, 1, d, f.ctypes.data, s.ctypes.data,
                                     None), _abi.ERR_INVALID, "at least 2")
    _refused(L, L.fid_stats_mean_cov(None, f.ctypes.data, s.ctypes.data, 5, d, f.ctypes.data, s.ctypes.data, None),
             _abi.ERR_INVALID, "null")
    _refused(L, L.fid_stats_mean_cov(f.ctypes.data, f.ctypes.data, s.ctypes.data, 5, 0, f.ctypes.data, s.ctypes.data,
                                     None), _abi.ERR_INVALID, "dim 0")


def test_python_checks_refuse_before_the_device():
    d = 4
    mu, s = np.zeros(d), np.eye(d)
    with pytest.raises(ValueError, match="mean vectors have different lengths"):
        fid.frechet_distance(np.zeros(3), s, mu, s)
    with pytest.raises(ValueError, match="covariances have different dimensions"):
        fid.frechet_distance(mu, s, mu, np.eye(5))
    with pytest.raises(ValueError, match="non-finite"):
        fid.frechet_distance(mu, np.full((d, d), np.inf), mu, s)

"""The Fréchet distance on the H100 at d = 2048: commuting pairs against their exact trace, seeded feature statistics
against the float64 eigh oracle and scipy, the FeatureStatistics path on InceptionV3 features of EvalPipeline
outputs, bitwise repeatability across calls and streams, guard bands and refusals."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import migan_b200  # noqa: E402
from migan_b200 import _abi, fid  # noqa: E402
from oracle import fid_oracle as FO  # noqa: E402
from oracle import frechet_oracle as O  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 2048
# Errors of tr sqrt measured on one NVIDIA H100 80GB HBM3 at a 700 W power limit (the results are bitwise repeatable):
# commuting full rank 8.6e-12, commuting rank 500 / 700 1.2e-6, features N = 500 1.8e-6 (against the oracle, whose own
# distance from scipy is 3.9e-5), N = 5000 8.5e-12, the Inception statistics 7.8e-8 of a 2.9e7 FID.  Bounds: ~3x those,
# each also inside the rule max(1e-12 (tr S1 + tr S2), 2 x the eigh oracle's own error).
BOUND = {"full rank": 3e-11, "rank 500 / 700": 4e-6, "N=500": 6e-6, "N=5000": 3e-11, "inception": 2.5e-7}


def check(got, want, T, oracle_err, what):
    rule = max(1e-12 * T, 2 * abs(oracle_err))
    print("%s: error %.3e, oracle's own %.3e, rule %.3e, bound %.3e (T = %.4g)"
          % (what, got - want, oracle_err, rule, BOUND[what], T))
    assert abs(got - want) <= min(rule, BOUND[what])


def test_commuting_full_rank():
    ev1, ev2 = O.log_spectrum(D, 1e-6, 1e2, seed=1), O.log_spectrum(D, 1e-5, 1e1, seed=2)
    s1, s2, exact = O.commuting_pair(D, ev1, ev2, seed=3)
    r = fid.frechet_terms(np.zeros(D), s1, np.zeros(D), s2)
    print("sweeps", r.sweeps)
    check(r.trace_sqrt, exact, np.trace(s1) + np.trace(s2), 0.0, "full rank")
    assert all(0 < s <= 40 for s in r.sweeps[:1])


def test_commuting_rank_deficient():
    ev1 = O.log_spectrum(D, 1e-4, 1e1, rank=500, seed=4)
    ev2 = O.log_spectrum(D, 1e-4, 1e1, rank=700, seed=5)
    s1, s2, exact = O.commuting_pair(D, ev1, ev2, seed=6)
    r = fid.frechet_terms(np.zeros(D), s1, np.zeros(D), s2)
    print("sweeps", r.sweeps)
    check(r.trace_sqrt, exact, np.trace(s1) + np.trace(s2), O.trace_sqrt(s1, s2) - exact, "rank 500 / 700")


@pytest.mark.parametrize("n", [500, 5000])
def test_features_against_oracle_and_scipy(n):
    mu1, s1 = O.feature_stats(n, D, seed=10)
    mu2, s2 = O.feature_stats(n, D, seed=11)
    r = fid.frechet_terms(mu1, s1, mu2, s2)
    want, ts = O.frechet_distance(mu1, s1, mu2, s2)
    print("N=%d sweeps %s fid %.12g oracle %.12g" % (n, r.sweeps, r.fid, want))
    T = np.trace(s1) + np.trace(s2)
    if n == 5000:
        scipy_fid = fid.calculate_frechet_distance(mu1, s1, mu2, s2)
        print("N=5000 scipy %.12g, relative %.3e" % (scipy_fid, (r.fid - scipy_fid) / scipy_fid))
        assert r.fid == pytest.approx(scipy_fid, rel=1e-9)
        check(r.trace_sqrt, ts, T, (want - scipy_fid) / 2, "N=5000")
    else:
        # full rank needs N > d: here both covariances have rank 499, and tr sqrt sits on the fp64 floor of the square
        # roots of round-off-sized eigenvalues; the rule's second term is scipy's distance from the oracle
        scipy_ts = (np.trace(s1) + np.trace(s2) + (mu1 - mu2).dot(mu1 - mu2)
                    - fid.calculate_frechet_distance(mu1, s1, mu2, s2)) / 2
        check(r.trace_sqrt, ts, T, ts - scipy_ts, "N=500")


def test_feature_statistics_path_on_inception_features():
    net = fid.InceptionV3(weights=FO.seeded_state_dict(0))
    R, n = 256, 24
    pipe = migan_b200.EvalPipeline(MO.make_state_dict(R, seed=3), resolution=R, device=DEV, seed=0)
    rng = np.random.default_rng(5)
    s_r, s_c = fid.FeatureStatistics(device=DEV), fid.FeatureStatistics(device=DEV)
    for _ in range(3):
        real, composed = pipe.forward_batch([rng.integers(0, 256, size=(R, R, 3), dtype=np.uint8) for _ in range(n // 3)])
        s_r.add(net(real)[0])
        s_c.add(net(composed)[0])
    (mu_r, sg_r), (mu_c, sg_c) = s_r.mean_cov(), s_c.mean_cov()
    for st, (mu, sg) in ((s_r, (mu_r, sg_r)), (s_c, (mu_c, sg_c))):
        dmu, dsg = st.mean_cov_device()
        assert dmu.cpu().numpy().tobytes() == mu.tobytes() and dsg.cpu().numpy().tobytes() == sg.tobytes()
    got = s_r.frechet_distance(s_c)
    assert got == fid.frechet_distance(mu_r, sg_r, mu_c, sg_c)
    # 24 rows: both covariances have rank 23 of 2048.  scipy's sqrtm leaves an imaginary part here and
    # calculate_frechet_distance refuses the input; the oracle with the same numerical-rank cutoff is the reference.
    want, _ = O.frechet_distance(mu_r, sg_r, mu_c, sg_c, cutoff=True)
    floor, _ = O.frechet_distance(mu_r, sg_r, mu_c, sg_c)
    T = np.trace(sg_r) + np.trace(sg_c)
    print("inception features n=%d: fid %.12g, oracle with cutoff %.12g (error %.3e), without %.12g, T = %.4g"
          % (n, got, want, got - want, floor, T))
    assert abs(got - want) <= BOUND["inception"]


def test_bitwise_repeatable_across_calls_and_streams():
    mu1, s1 = O.feature_stats(3000, D, seed=20)
    mu2, s2 = O.feature_stats(3000, D, seed=21)
    t = [torch.from_numpy(x).to(DEV) for x in (mu1, s1, mu2, s2)]
    a = fid.frechet_terms(*t)
    b = fid.frechet_terms(*t)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        c = fid.frechet_terms(*t)
    assert a == b == c
    assert fid.frechet_terms(mu1, s1, mu2, s2) == a


def test_guard_bands_and_outputs():
    mu1, s1 = O.feature_stats(700, 300, seed=30)
    mu2, s2 = O.feature_stats(800, 300, seed=31)
    t = [torch.from_numpy(x).to(DEV) for x in (mu1, s1, mu2, s2)]
    L = fid.frechet_lib()
    need = L.fid_frechet_workspace_bytes(300)
    ws = torch.full((need + 65536,), 0xA5, dtype=torch.uint8, device=DEV)
    out = (ctypes.c_double * 6)(-7.25, 0, 0, 0, 0, -7.25)
    sweeps = (ctypes.c_int * 4)(-5, 0, 0, -5)
    _abi.check(L.fid_frechet_distance(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 300,
                                      ctypes.cast(ctypes.byref(out, 8), ctypes.POINTER(ctypes.c_double)),
                                      ctypes.cast(ctypes.byref(sweeps, 4), ctypes.POINTER(ctypes.c_int)), ws.data_ptr(),
                                      need, torch.cuda.current_stream().cuda_stream))
    assert bool((ws[need:] == 0xA5).all())
    assert out[0] == out[5] == -7.25 and sweeps[0] == sweeps[3] == -5
    assert out[4] == pytest.approx(O.trace_sqrt(s1, s2), rel=1e-11)


def test_refusals():
    L = fid.frechet_lib()
    mu, s = torch.zeros(64, dtype=torch.float64, device=DEV), torch.eye(64, dtype=torch.float64, device=DEV)
    need = L.fid_frechet_workspace_bytes(64)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = (ctypes.c_double * 4)()
    st = torch.cuda.current_stream().cuda_stream
    p = mu.data_ptr(), s.data_ptr(), mu.data_ptr(), s.data_ptr()
    assert L.fid_frechet_distance(*p, 64, out, None, ws.data_ptr(), need - 1, st) == _abi.ERR_WORKSPACE
    assert L.fid_frechet_distance(*p, 0, out, None, ws.data_ptr(), need, st) == _abi.ERR_INVALID
    assert L.fid_frechet_distance(*p, 4097, out, None, ws.data_ptr(), need, st) == _abi.ERR_INVALID
    assert L.fid_frechet_distance(None, *p[1:], 64, out, None, ws.data_ptr(), need, st) == _abi.ERR_INVALID
    bad = s.clone()
    bad[1, 2] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        fid.frechet_distance(mu, bad, mu, s)
    asym = s.clone()
    asym[1, 2] = 1e-6
    with pytest.raises(ValueError, match="not symmetric"):
        fid.frechet_distance(mu, asym, mu, s)
    with pytest.raises(ValueError, match="different dimensions"):
        fid.frechet_distance(mu, s, mu, torch.eye(63, dtype=torch.float64, device=DEV))
    with pytest.raises(ValueError, match="outside"):
        fid.frechet_distance(np.zeros(4097), np.eye(4097), np.zeros(4097), np.eye(4097))

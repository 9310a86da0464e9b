"""KID without a GPU: the float64 oracle against the textbook unbiased MMD^2, a hand-computed case and StyleGAN2-ADA's
float32 computation; the library's kernels in the emulation build (the same phases, DMMA tile products as loops in
their k order) against the oracle; every refusal of the C ABI; and `--kid` in the evaluation and scoring commands: its
argument handling, the line formats, and rank 0's merge, also through gloo at W = 2 and 3 against W = 1, with the
feature statistics, the distance and the scores replaced by stand-ins that record rows."""
import ctypes
import io
import math
import os
import socket
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, fid, ids, kid  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from migan_b200 import score_results as S  # noqa: E402
from oracle import kid_oracle as O  # noqa: E402

# Emulated terms and KID against the oracle, in units of each subset's cancellation scale
# ((|Sxx| + |Syy|) / (m - 1) + 2 |Sxy| / m) / m: both are float64 with sums in different orders; measured at most
# 1.5e-16 on the cases below.
BOUND = 1e-12
# StyleGAN2-ADA's float32 computation against the oracle, in units of the mean cancellation scale: measured 1.3e-8.
FLOAT32_BOUND = 1e-6
GUARD = -7.25


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(build_emul.CSRC, s) for s in ("kid.cu", "abi_error.cu")]
    L = kid.kid_lib(ctypes.CDLL(build_emul._compile("kid_emul", srcs)))
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


def raw_call(L, real, fake, real_idx, fake_idx, S, m, ws=None, nbytes=None, dtype=None, dim=None, terms=None,
             n_real=None, n_fake=None):
    """kid_subset_terms on host arrays: (return code, terms [S, 3] or the guard-filled buffer)."""
    if ws is None:
        ws = Workspace(max(L.kid_workspace_bytes(max(S, 1), max(m, 2)), 256))
    out = np.full((max(S, 1) + 2) * 3, GUARD)
    dtype = (ids.FLOAT64 if real.dtype == np.float64 else ids.FLOAT32) if dtype is None else dtype
    rc = L.kid_subset_terms(real.ctypes.data, len(real) if n_real is None else n_real, fake.ctypes.data,
                            len(fake) if n_fake is None else n_fake, real.shape[1] if dim is None else dim, dtype,
                            None if real_idx is None else real_idx.ctypes.data,
                            None if fake_idx is None else fake_idx.ctypes.data, S, m,
                            None if terms is False else out[3:].ctypes.data, ws.base,
                            ws.nbytes if nbytes is None else nbytes, None)
    return rc, out, ws


def emulated(L, real, fake, S, max_subset_size=1000, seed=0):
    """The library's terms [S, 3] and (KID, std) through the emulation build, with every guard checked."""
    m = O.subset_size(len(real), len(fake), max_subset_size)
    fi, ri = kid.draw_subsets(len(real), len(fake), S, m, seed)
    rc, out, ws = raw_call(L, real, fake, ri, fi, S, m)
    _abi.check(rc, L)
    assert ws.guard_intact() and (out[:3] == GUARD).all() and (out[-3:] == GUARD).all()
    T = out[3:-3].reshape(S, 3)
    return T, kid.finish(T, m)


def scale(T, m):
    """Each subset's cancellation scale."""
    return ((np.abs(T[:, 0]) + np.abs(T[:, 1])) / (m - 1) + 2 * np.abs(T[:, 2]) / m) / m


# -- the oracle -------------------------------------------------------------------------------------------------------

def textbook(x, y):
    """The unbiased MMD^2 estimate as the paper writes it."""
    m = len(x)
    kxx, kyy, kxy = O.kernel(x, x), O.kernel(y, y), O.kernel(x, y)
    off = ~np.eye(m, dtype=bool)
    return kxx[off].sum() / (m * (m - 1)) + kyy[off].sum() / (m * (m - 1)) - 2 * kxy.sum() / (m * m)


@pytest.mark.parametrize("n_r,n_f,d,max_subset", [(120, 90, 37, 1000), (300, 300, 2048, 64), (2, 3, 5, 1000)])
def test_oracle_is_the_unbiased_mmd(n_r, n_f, d, max_subset):
    real, fake = O.features(n_r, d, 1).astype(np.float64), O.features(n_f, d, 2, 0.2).astype(np.float64)
    res = O.kid(real, fake, 7, max_subset, seed=3)
    fi, ri = O.draw(n_r, n_f, 7, O.subset_size(n_r, n_f, max_subset), seed=3)
    for s in range(7):
        want = textbook(fake[fi[s]], real[ri[s]])
        assert abs(res.estimates[s] - want) <= 1e-13 * abs(want)
    assert res.kid == pytest.approx(np.mean(res.estimates), rel=1e-13)
    assert res.std == float(np.std(res.estimates))


def test_oracle_hand_case():
    # d = 1, m = 2, k(u, v) = (u v + 1)^3: Sxx = 2 k(0, 3) = 2, Syy = 2 k(1, 2) = 54,
    # Sxy = k(0, 1) + k(0, 2) + k(3, 1) + k(3, 2) = 1 + 1 + 64 + 343 = 409; e = ((2 + 54) / 1 - 2 * 409 / 2) / 2.
    real, fake = np.array([[1.0], [2.0]]), np.array([[0.0], [3.0]])
    res = O.kid(real, fake, 4)
    assert (res.terms == np.array([[2.0, 54.0, 409.0]] * 4)).all()
    assert res.kid == -176.5 and res.std == 0.0


def test_oracle_against_stylegan2_ada_float32():
    real, fake = O.features(500, 2048, 1), O.features(500, 2048, 2, 0.1)
    res = O.kid(real, fake, 10, 200)
    gap = abs(O.stylegan2_ada_float32(real, fake, 10, 200) - res.kid)
    assert gap <= FLOAT32_BOUND * scale(res.terms, 200).mean()


def test_draws_follow_the_contract():
    fi, ri = kid.draw_subsets(50, 70, 3, 20, seed=5)
    rng = np.random.RandomState(5)
    for s in range(3):
        assert (fi[s] == rng.choice(70, 20, replace=False)).all()
        assert (ri[s] == rng.choice(50, 20, replace=False)).all()
    assert fi.dtype == ri.dtype == np.int32
    ofi, ori = O.draw(50, 70, 3, 20, seed=5)
    assert (ofi == fi).all() and (ori == ri).all()


# -- the emulation build against the oracle ---------------------------------------------------------------------------

EMUL_CASES = [  # n_r, n_f, d, max_subset_size, dtype
    (2, 5, 37, 1000, np.float32),       # m = 2 = n_r
    (63, 63, 37, 1000, np.float64),     # m = 63 = n
    (100, 80, 37, 64, np.float32),      # m = 64
    (65, 90, 2048, 1000, np.float64),   # m = 65 = n_r
    (150, 130, 37, 1000, np.float32),   # m = 130 = n_f
    (140, 200, 2048, 130, np.float32),  # m = 130, d = 2048
]


@pytest.mark.parametrize("n_r,n_f,d,max_subset,dtype", EMUL_CASES)
def test_emulation_matches_the_oracle(emul, n_r, n_f, d, max_subset, dtype):
    real, fake = O.features(n_r, d, 11).astype(dtype), O.features(n_f, d, 12, 0.1).astype(dtype)
    T, (value, std) = emulated(emul, real, fake, 3, max_subset, seed=1)
    want = O.kid(real, fake, 3, max_subset, seed=1)
    m = O.subset_size(n_r, n_f, max_subset)
    c = scale(want.terms, m)
    diff = ((np.abs(T[:, 0] - want.terms[:, 0]) + np.abs(T[:, 1] - want.terms[:, 1])) / (m - 1)
            + 2 * np.abs(T[:, 2] - want.terms[:, 2]) / m) / m
    assert (diff <= BOUND * c).all()
    assert abs(value - want.kid) <= BOUND * c.mean()
    assert abs(std - want.std) <= BOUND * c.max()


def test_emulation_float32_is_float64_of_the_same_values(emul):
    real, fake = O.features(70, 100, 3), O.features(66, 100, 4, 0.3)
    T32, _ = emulated(emul, real, fake, 2)
    T64, _ = emulated(emul, real.astype(np.float64), fake.astype(np.float64), 2)
    assert T32.tobytes() == T64.tobytes()


def test_emulation_hand_case(emul):
    T, (value, std) = emulated(emul, np.array([[1.0], [2.0]]), np.array([[0.0], [3.0]]), 3)
    assert (T == np.array([[2.0, 54.0, 409.0]] * 3)).all() and (value, std) == (-176.5, 0.0)


# -- the C ABI's refusals ---------------------------------------------------------------------------------------------

def test_workspace_bytes(emul):
    assert emul.kid_workspace_bytes(0, 10) == 0 and emul.kid_workspace_bytes(1, 1) == 0
    assert emul.kid_workspace_bytes(2 ** 20, 4096) == 0                  # S x m reaches 2^31
    # S = 100, m = 1000: two tables of 100,000 ints, then 100 x 3 x 16^2 partials
    assert emul.kid_workspace_bytes(100, 1000) == 2 * 400128 + 614400
    assert emul.kid_workspace_bytes(1, 2) == 2 * 256 + 256


def test_refusals(emul):
    real, fake = O.features(10, 8, 1), O.features(12, 8, 2)
    fi, ri = kid.draw_subsets(10, 12, 2, 5)

    def refused(code, match, **kw):
        args = dict(real=real, fake=fake, real_idx=ri, fake_idx=fi, S=2, m=5)
        args.update(kw)
        rc, out, _ = raw_call(emul, args.pop("real"), args.pop("fake"), args.pop("real_idx"), args.pop("fake_idx"),
                              args.pop("S"), args.pop("m"), **args)
        assert rc == code, emul.migan_last_error()
        assert match in emul.migan_last_error().decode()
        assert (out == GUARD).all()

    invalid = _abi.ERR_INVALID
    refused(invalid, "null", real_idx=None)
    refused(invalid, "null", fake_idx=None)
    refused(invalid, "null", terms=False)
    refused(invalid, "null", ws=type("W", (), {"base": None, "nbytes": 1 << 20})())
    refused(invalid, "0 subsets", S=0)
    refused(invalid, "subsets of 1 rows", m=1)
    refused(invalid, "subsets of 11 rows", m=11, real_idx=np.zeros((2, 11), np.int32),
            fake_idx=np.zeros((2, 11), np.int32))
    refused(invalid, "from 4 real", n_real=4)
    refused(invalid, "and 3 fake", n_fake=3)
    refused(invalid, "reach 2^31", n_real=2 ** 31)
    refused(invalid, "dim 0 outside", dim=0)
    refused(invalid, "dim 4097 outside", dim=4097)
    refused(invalid, "dtype 2", dtype=2)
    refused(invalid, "dtype -1", dtype=-1)
    bad = fi.copy()
    bad[1, 3] = 12
    refused(invalid, "fake index 3 of subset 1 is 12", fake_idx=bad)
    bad = ri.copy()
    bad[0, 0] = -1
    refused(invalid, "real index 0 of subset 0 is -1", real_idx=bad)
    bad = ri.copy()
    bad[1, 4] = bad[1, 2]
    refused(invalid, "subset 1 draws real row %d twice" % ri[1, 2], real_idx=bad)
    ws = Workspace(emul.kid_workspace_bytes(2, 5) + 512)
    refused(_abi.ERR_WORKSPACE, "%d bytes" % (emul.kid_workspace_bytes(2, 5) - 1), ws=ws,
            nbytes=emul.kid_workspace_bytes(2, 5) - 1)
    shifted = type("W", (), {"base": ws.base + 8, "nbytes": ws.nbytes})()
    refused(_abi.ERR_WORKSPACE, "256-byte aligned", ws=shifted)


def test_python_checks_refuse_before_the_device():
    a = np.zeros((4, 8), np.float32)
    with pytest.raises(ValueError, match="at least 2 rows"):
        kid.kernel_inception_distance(a, a[:1])
    with pytest.raises(ValueError, match="at least 2 rows"):
        kid.kernel_inception_distance(a, a, max_subset_size=1)
    with pytest.raises(ValueError, match="width"):
        kid.kernel_inception_distance(a, np.zeros((4, 9)))
    with pytest.raises(ValueError, match="num_subsets"):
        kid.kernel_inception_distance(a, a, num_subsets=0)
    with pytest.raises(ValueError, match="outside 1..4096"):
        kid.kernel_inception_distance(np.zeros((4, 4097)), np.zeros((4, 4097)))
    with pytest.raises(ValueError, match=r"\[N, d\]"):
        kid.kernel_inception_distance(np.zeros(4), a)
    b = a.copy()
    b[2, 3] = np.inf
    with pytest.raises(ValueError, match="fake has non-finite"):
        kid.kernel_inception_distance(a, b)
    with pytest.raises(ValueError, match="real has non-finite"):
        kid.kernel_inception_distance(b * np.nan, a)
    with pytest.raises(ValueError, match=r"\[S, m\]"):
        kid.subset_terms(None, None, np.zeros((2, 3)), np.zeros((2, 4)))


# -- the commands -----------------------------------------------------------------------------------------------------

def _eval_argv(tmp_path, *extra):
    return ["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", str(tmp_path)] + list(extra)


def _score_argv(tmp_path, *extra):
    return ["--resolution", "256", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)] + list(extra)


def test_kid_flag_parses(tmp_path):
    assert not E.get_args(_eval_argv(tmp_path)).kid and E.get_args(_eval_argv(tmp_path, "--kid")).kid
    assert not S.get_args(_score_argv(tmp_path)).kid and S.get_args(_score_argv(tmp_path, "--kid")).kid


@pytest.mark.parametrize("command,argv", [(E, _eval_argv), (S, _score_argv)], ids=["evaluate_fid_lpips", "score_results"])
def test_kid_with_real_stats_is_refused_before_any_work(tmp_path, command, argv):
    missing = tmp_path / "nothing_here"          # no images, no model: the refusal comes first
    with pytest.raises(ValueError, match="--kid needs the real images' features.*--real-stats"):
        command.main(argv(missing, "--kid", "--real-stats", str(missing / "s.npz")))


def test_library_refusals_before_any_work(tmp_path):
    missing = tmp_path / "nothing_here"
    stats = (np.zeros(2048), np.eye(2048))
    with pytest.raises(ValueError, match="--kid needs"):
        E.evaluate("migan-256", missing / "m.pt", missing, real_stats=stats, kid=True)
    with pytest.raises(ValueError, match="--kid needs"):
        S.score(missing, missing, resolution=256, real_stats=stats, kid=True)
    with pytest.raises(ValueError, match="real features"):
        E.Merge(4, "cpu", real_features=False, kid=True)
    E.check_stats_args(stats, None, False, False)


class RowStats:
    """`fid.FeatureStatistics` stand-in: keeps its rows; its 'mean' is their column sum."""

    def __init__(self, dim=fid.FEATURES, device="cpu"):
        self.rows = []

    def add(self, feats):
        self.rows.append(feats.clone())

    def mean_cov_device(self):
        return torch.cat(self.rows).double().sum(0), None

    def frechet_distance(self, other):
        return 0.0


class BinnedRows:
    """`fid.BinnedFeatureStatistics` stand-in: keeps every (feats, bins) call."""

    def __init__(self, nbins, dim=fid.FEATURES, device="cpu"):
        self.nbins, self.calls = nbins, []

    def add(self, feats, bins):
        self.calls.append((feats.clone(), bins.clone()))

    def counts(self):
        b = torch.cat([c[1] for c in self.calls]).numpy()
        return np.bincount(b, minlength=self.nbins).astype(np.int64)

    def mean_cov_device(self, b, count=None):
        rows = torch.cat([f[k == b] for f, k in self.calls])
        return rows.double().sum(0), rows


def fake_distance(mu1, sigma1, mu2, sigma2):
    return float(mu2.sum())


class FakeScores:
    def __init__(self, p, u):
        self.p_ids, self.u_ids = p, u


def fake_ids(real, fake):
    return FakeScores(float(real.double().sum()), float(fake.double().mean()))


def fake_kid(real, fake):
    """A stand-in that sees which rows it got: all real rows, and the composed rows in dataset order."""
    r, f = real.double(), fake.double()
    return kid.KIDResult(float(r.sum()) * 1e-3 + float((f * torch.arange(1, len(f) + 1)[:, None]).sum()), 0.0, 100,
                         min(len(r), len(f), 1000))


def install_stand_ins():
    fid.FeatureStatistics, fid.BinnedFeatureStatistics, fid.frechet_distance = RowStats, BinnedRows, fake_distance
    ids.inception_discriminative_scores = fake_ids
    kid.kernel_inception_distance = fake_kid


@pytest.fixture
def stand_ins(monkeypatch):
    monkeypatch.setattr(fid, "FeatureStatistics", RowStats)
    monkeypatch.setattr(fid, "BinnedFeatureStatistics", BinnedRows)
    monkeypatch.setattr(fid, "frechet_distance", fake_distance)
    monkeypatch.setattr(ids, "inception_discriminative_scores", fake_ids)
    monkeypatch.setattr(kid, "kernel_inception_distance", fake_kid)


EDGES = (0.0, 0.25, 3 / 7, 0.6, 1.0)


def stand_in(j, chunks, extra_values):
    a, b = chunks[j]
    idx = torch.arange(a, b, dtype=torch.float32)[:, None]
    col = torch.arange(fid.FEATURES, dtype=torch.float32)[None]
    i = idx[:, 0]
    values = {"hole_fraction": (i % 8) / 7, "ssim": torch.cos(i * 0.3) * 0.4 + 0.5, "psnr": 12 + i / 3}
    extra = torch.stack([values[v] for v in extra_values], 1) if extra_values else None
    return E.ChunkResult(j, a, torch.sin(idx * 0.37 + col * 0.011), torch.cos(idx * 0.53 - col * 0.007) / 3,
                         torch.tanh(i / 9), extra)


def merged(n, batch, extra_values, edges, ids_on, kid_on, chunk_results=None):
    chunks = E.chunk_bounds(n, batch)
    merge = E.Merge(n, "cpu", True, keep_features=ids_on, extra_values=extra_values, hole_bins=edges, kid=kid_on)
    for c in chunk_results if chunk_results is not None else [stand_in(j, chunks, extra_values)
                                                              for j in range(len(chunks))]:
        merge.add(c)
    return merge.result()


def _printed(res, *flags, **kw):
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, *flags, **kw)
    return out.getvalue().splitlines()


def test_kid_line_and_its_place():
    res = E.EvalResult(1.5, 0.25, np.zeros(2), 2, p_ids=0.1, u_ids=0.2)
    res.kid = 0.0123
    assert _printed(res, True, kid=True) == ["FID: 1.5", "LPIPS:  0.25", "P-IDS: 0.1", "U-IDS: 0.2", "KID: 0.0123"]
    res.ssim, res.psnr, res.kid = 0.5, 30.0, -2.5e-05
    res.by_hole = (E.HoleBin(0.0, 1.0, 2, 3.0, 0.25, kid=0.125),)
    assert _printed(res, False, True, True, True) == ["FID: 1.5", "LPIPS:  0.25", "SSIM: 0.5", "PSNR: 30.0",
                                                      "KID: -2.5e-05", "HOLE [0.0, 1.0]: images 2 FID 3.0 LPIPS 0.25 "
                                                      "KID 0.125"]
    assert _printed(res, False, True, True) == ["FID: 1.5", "LPIPS:  0.25", "SSIM: 0.5", "PSNR: 30.0",
                                                "HOLE [0.0, 1.0]: images 2 FID 3.0 LPIPS 0.25 KID 0.125"]


def test_hole_line_with_kid():
    b = E.HoleBin(0.6, 1.0, 1, math.nan, 0.25, 0.5, math.inf, math.nan, math.nan, math.nan)
    assert E.hole_line(b, True) == ("HOLE [0.6, 1.0]: images 1 FID nan LPIPS 0.25 SSIM 0.5 PSNR inf P-IDS nan U-IDS nan "
                                    "KID nan")
    b = E.HoleBin(0.0, 0.1, 812, 3.52, 0.0412, kid=0.00125)
    assert E.hole_line(b, False) == "HOLE [0.0, 0.1): images 812 FID 3.52 LPIPS 0.0412 KID 0.00125"
    assert E.HoleBin(0.0, 0.1, 812, 3.52, 0.0412).kid is None


def test_merge_with_kid(stand_ins):
    n, batch = 29, 8
    chunks = E.chunk_bounds(n, batch)
    parts = [stand_in(j, chunks, ("hole_fraction",)) for j in range(len(chunks))]
    real, fake = torch.cat([p.real for p in parts]), torch.cat([p.fake for p in parts])
    res = merged(n, batch, ("hole_fraction",), EDGES, False, True)
    assert res.kid == fake_kid(real, fake).kid and res.p_ids is None and len(res) == 8
    h = torch.cat([p.extra[:, 0] for p in parts]).numpy().astype(np.float64)
    bins = np.searchsorted(np.array(EDGES[1:-1]), h, side="right")
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert b.kid == fake_kid(real, fake[idx]).kid and b.p_ids is None
    # with --ids too: both, from the same kept rows
    both = merged(n, batch, ("hole_fraction",), EDGES, True, True)
    assert both.kid == res.kid and both.p_ids == fake_ids(real, fake).p_ids
    assert [b.kid for b in both.by_hole] == [b.kid for b in res.by_hole]
    # below 2 images a bin's KID is nan
    small = merged(4, 2, ("hole_fraction",), (0.0, 0.1, 0.2, 0.3, 1.0), False, True)   # h = 0, 1/7, 2/7, 3/7
    assert all(b.count == 1 and math.isnan(b.kid) and b.p_ids is None for b in small.by_hole)


def test_without_kid_nothing_changes(stand_ins):
    res = merged(29, 8, ("hole_fraction",), EDGES, True, False)
    assert res.kid is None and all(b.kid is None for b in res.by_hole)
    plain = merged(20, 8, (), None, False, False)
    assert plain.kid is None and _printed(plain, False) == ["FID: 0.0", "LPIPS:  %r" % plain.lpips]
    assert E.Merge(4, "cpu", True).kept is None


# -- transport over gloo --------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


GLOO_CASES = [(70, 8, ("hole_fraction",), EDGES, True), (5, 2, (), None, False), (33, 32, ("hole_fraction",), EDGES, False)]


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    install_stand_ins()
    for case, (n, batch, extra_values, edges, ids_on) in enumerate(GLOO_CASES):
        chunks = E.chunk_bounds(n, batch)
        width = 2 * fid.FEATURES + 1 + len(extra_values)
        received = []
        for r in range(E.num_rounds(len(chunks), world)):
            j = E.round_chunk(r, rank, len(chunks), world)
            mine = None if j is None else stand_in(j, chunks, extra_values)
            received += E.gather_round(mine, r, chunks, width, "cpu", extra=len(extra_values))
        if rank == 0:
            res = merged(n, batch, extra_values, edges, ids_on, True, chunk_results=received)
            torch.save({"lines": _printed(res, ids_on, kid=True)}, os.path.join(out_dir, "case%d.pt" % case))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_print_the_kid_of_one_rank(tmp_path, stand_ins, world):
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for case, (n, batch, extra_values, edges, ids_on) in enumerate(GLOO_CASES):
        got = torch.load(tmp_path / ("case%d.pt" % case), weights_only=False)
        want = _printed(merged(n, batch, extra_values, edges, ids_on, True), ids_on, kid=True)
        assert got["lines"] == want and any(line.startswith("KID: ") for line in want)

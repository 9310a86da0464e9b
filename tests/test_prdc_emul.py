"""Precision, recall, density and coverage without a GPU: the library's kernels in the emulation build (the same phases,
DMMA tile products as loops in their k order) against the float64 oracle (squared differences summed directly), on
seeded ragged sets and on small integer-valued sets full of exact ties and duplicated rows; the exact identities (a
copy scores 1, swapping the sets swaps precision and recall, row order does not matter, the cached real radii give
the full call's counts); every refusal of the C ABI and of the Python checks; and `--prdc` in the evaluation and
scoring commands: the flag, the refusal with `--real-stats`, the line order, the per-bin nan rule, the real radii
computed once, and every output unchanged without `--prdc`, with the metrics replaced by stand-ins that record rows."""
import ctypes
import io
import math
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, fid, ids, prdc  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from migan_b200 import score_results as S  # noqa: E402
from oracle import prdc_oracle as O  # noqa: E402

GUARD = -7


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(build_emul.CSRC, s) for s in ("prdc.cu", "abi_error.cu")]
    L = prdc.prdc_lib(ctypes.CDLL(build_emul._compile("prdc_emul", srcs)))
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


def _dtype(x):
    return ids.FLOAT64 if x.dtype == np.float64 else ids.FLOAT32


def raw_call(L, real, fake, k, ws=None, nbytes=None, dtype=None, dim=None, out=True, n_real=None, n_fake=None,
             fn="prdc_counts"):
    """prdc_counts (or prdc_counts_with_real_radii) on host arrays: (return code, the guard-framed int64 buffer, ws)."""
    if ws is None:
        ws = Workspace(max(L.prdc_workspace_bytes(len(real), len(fake), real.shape[1], k), 256))
    buf = np.full(4 + 4, GUARD, dtype=np.int64)
    rc = getattr(L, fn)(real.ctypes.data, len(real) if n_real is None else n_real, fake.ctypes.data,
                        len(fake) if n_fake is None else n_fake, real.shape[1] if dim is None else dim,
                        _dtype(real) if dtype is None else dtype, k, buf[2:].ctypes.data if out else None, ws.base,
                        ws.nbytes if nbytes is None else nbytes, None)
    return rc, buf, ws


def emulated(L, real, fake, k=3):
    """The emulation build's four counts, with every guard checked."""
    rc, buf, ws = raw_call(L, real, fake, k)
    _abi.check(rc, L)
    assert ws.guard_intact() and (buf[:2] == GUARD).all() and (buf[-2:] == GUARD).all()
    return buf[2:6].copy()


# -- the emulation build against the oracle ---------------------------------------------------------------------------

EMUL_CASES = [  # n_r, n_f, d, k, dtype
    (150, 97, 37, 3, np.float32),       # N != M, neither a multiple of 64, d below one panel
    (70, 130, 100, 1, np.float64),      # d not a multiple of the panel width
    (65, 66, 130, 5, np.float32),
    (64, 128, 64, 3, np.float64),       # whole tiles and one whole panel
    (200, 201, 2048, 3, np.float32),    # pool3's width
    (6, 4, 9, 3, np.float64),           # k + 1 = M
]


@pytest.mark.parametrize("n_r,n_f,d,k,dtype", EMUL_CASES)
def test_emulation_matches_the_oracle(emul, n_r, n_f, d, k, dtype):
    real, fake = O.features(n_r, d, 11).astype(dtype), O.features(n_f, d, 12, 0.02).astype(dtype)
    got = emulated(emul, real, fake, k)
    want = O.prdc(real, fake, k)
    bound = O.rounding_bound(real, fake)
    print("N %d M %d d %d k %d: counts %s, margin %.3g, bound %.3g" % (n_r, n_f, d, k, got.tolist(), want.margin,
                                                                        bound))
    assert (got == want.counts).all(), (got, want.counts)
    assert want.margin > 1000 * bound


@pytest.mark.parametrize("k", [1, 3, 5])
@pytest.mark.parametrize("d", [1, 5, 70])
def test_integer_ties(emul, k, d):
    real = O.integer_features(150, d, 3)
    fake = O.integer_features(97, d, 4, dup_of=real, dups=30)
    want = O.prdc(real, fake, k)
    assert want.margin == 0.0          # ties at the thresholds: `<=` decides them
    assert (emulated(emul, real, fake, k) == want.counts).all()
    assert (emulated(emul, real.astype(np.float64), fake.astype(np.float64), k) == want.counts).all()


def test_copy_scores_one(emul):
    real = O.features(130, 40, 5)
    for k in (1, 3):
        c = emulated(emul, real, real.copy(), k)
        assert c[0] == c[1] == c[3] == 130 and c[2] >= 130 * k
        res = prdc.finish(c, k, 130, 130)
        assert res.precision == res.recall == res.coverage == 1.0


def test_swapping_the_sets_swaps_precision_and_recall(emul):
    real, fake = O.features(100, 50, 1), O.features(77, 50, 2, 0.02)
    a, b = emulated(emul, real, fake), emulated(emul, fake, real)
    assert (a[0], a[1]) == (b[1], b[0]) and 0 < a[0] < 77 and 0 < a[1] < 100


def test_row_order_does_not_matter(emul):
    real, fake = O.features(140, 70, 1), O.features(90, 70, 2, 0.02)
    rng = np.random.RandomState(0)
    a = emulated(emul, real, fake)
    b = emulated(emul, real[rng.permutation(140)].copy(), fake[rng.permutation(90)].copy())
    assert a.tobytes() == b.tobytes()
    ti, tf = O.integer_features(120, 4, 1), O.integer_features(80, 4, 2)
    c = emulated(emul, ti, tf)
    assert c.tobytes() == emulated(emul, ti[::-1].copy(), tf[rng.permutation(80)].copy()).tobytes()


def test_float32_counts_are_those_of_the_same_values_in_float64(emul):
    real, fake = O.features(90, 100, 3), O.features(70, 100, 4, 0.02)
    assert emulated(emul, real, fake).tobytes() == emulated(emul, real.astype(np.float64),
                                                            fake.astype(np.float64)).tobytes()


def test_cached_real_radii_give_the_full_counts(emul):
    real, fake = O.features(150, 37, 1), O.features(140, 37, 2, 0.02)
    k = 3
    ws = Workspace(emul.prdc_workspace_bytes(150, 140, 37, k))
    _abi.check(emul.prdc_real_radii(real.ctypes.data, 150, 37, ids.FLOAT32, k, ws.base, ws.nbytes, None), emul)
    for rows in (fake, fake[:4], fake[50:117]):
        rows = np.ascontiguousarray(rows)
        rc, buf, _ = raw_call(emul, real, rows, k, ws=ws, fn="prdc_counts_with_real_radii")
        _abi.check(rc, emul)
        assert (buf[2:6] == emulated(emul, real, rows, k)).all()
        assert (buf[2:6] == O.prdc(real, rows, k).counts).all()
    assert ws.guard_intact()


# -- the C ABI's refusals ---------------------------------------------------------------------------------------------

def test_workspace_bytes(emul):
    f = emul.prdc_workspace_bytes
    assert f(3, 4, 8, 3) == 0 and f(4, 3, 8, 3) == 0 and f(10, 10, 8, 0) == 0 and f(100, 100, 8, 33) == 0
    assert f(10, 10, 0, 3) == 0 and f(10, 10, 4097, 3) == 0 and f(2 ** 31, 10, 8, 3) == 0 and f(10, 2 ** 31, 8, 3) == 0
    # N = M = 10: 4 regions of 10 doubles and 2 of 10 ints (256 each), lists 1 x 1 x 4 x 256 doubles, 1 x 64 counters,
    # 2 x 2 int64 partials
    assert f(10, 10, 8, 3) == 6 * 256 + 8192 + 256 + 256
    # N = M = 36,500 (571 tiles, 8 splits), k = 3
    n = 36500
    a = lambda b: (b + 255) // 256 * 256  # noqa: E731
    assert f(n, n, 2048, 3) == 4 * a(8 * n) + 2 * a(4 * n) + 571 * 8 * 4 * 2048 + a(8 * 571 * 64 * 4) + a(2 * 571 * 16)


def test_refusals(emul):
    real, fake = O.features(10, 8, 1), O.features(12, 8, 2)

    def refused(code, match, fn="prdc_counts", **kw):
        rc, buf, _ = raw_call(emul, kw.pop("real", real), kw.pop("fake", fake), kw.pop("k", 3), fn=fn, **kw)
        assert rc == code, emul.migan_last_error()
        assert match in emul.migan_last_error().decode()
        assert (buf == GUARD).all()

    invalid = _abi.ERR_INVALID
    for fn in ("prdc_counts", "prdc_counts_with_real_radii"):
        refused(invalid, "null", fn, out=False)
        refused(invalid, "null", fn, ws=type("W", (), {"base": None, "nbytes": 1 << 20})())
        refused(invalid, "k 0 outside 1..32", fn, k=0)
        refused(invalid, "k 33 outside 1..32", fn, k=33)
        refused(invalid, "k + 1 = 11 neighbours from 10 real", fn, k=10)
        refused(invalid, "k + 1 = 4 neighbours from 10 real and 3 fake", fn, n_fake=3)
        refused(invalid, "k + 1 = 4 neighbours from 3 real", fn, n_real=3)
        refused(invalid, "2147483648 real / 12 fake rows reach 2^31", fn, n_real=2 ** 31)
        refused(invalid, "10 real / 2147483648 fake rows reach 2^31", fn, n_fake=2 ** 31)
        refused(invalid, "dim 0 outside", fn, dim=0)
        refused(invalid, "dim 4097 outside", fn, dim=4097)
        refused(invalid, "dtype 2", fn, dtype=2)
        refused(invalid, "dtype -1", fn, dtype=-1)
        need = emul.prdc_workspace_bytes(10, 12, 8, 3)
        ws = Workspace(need + 512)
        refused(_abi.ERR_WORKSPACE, "workspace of %d bytes, %d needed" % (need - 1, need), fn, ws=ws, nbytes=need - 1)
        refused(_abi.ERR_WORKSPACE, "256-byte aligned", fn, ws=type("W", (), {"base": ws.base + 8, "nbytes": need})())
    rc = emul.prdc_counts(None, 10, fake.ctypes.data, 12, 8, 0, 3, Workspace(8).base, Workspace(8).base, 1 << 20, None)
    assert rc == invalid and "null" in emul.migan_last_error().decode()
    ws = Workspace(1 << 16)
    assert emul.prdc_real_radii(real.ctypes.data, 10, 8, 0, 3, ws.base, 100, None) == _abi.ERR_WORKSPACE
    assert emul.prdc_real_radii(real.ctypes.data, 3, 8, 0, 3, ws.base, ws.nbytes, None) == invalid
    assert emul.prdc_real_radii(None, 10, 8, 0, 3, ws.base, ws.nbytes, None) == invalid


def test_python_checks_refuse_before_the_device():
    a = np.zeros((5, 8), np.float32)
    f = prdc.precision_recall_density_coverage
    with pytest.raises(ValueError, match="k = 3 needs at least k \\+ 1 = 4 fake rows, got 3"):
        f(a, a[:3])
    with pytest.raises(ValueError, match="4 real rows"):
        f(a[:3], a)
    with pytest.raises(ValueError, match="k must be in 1..32"):
        f(a, a, k=0)
    with pytest.raises(ValueError, match="k must be in 1..32"):
        f(a, a, k=33)
    with pytest.raises(ValueError, match="width"):
        f(a, np.zeros((5, 9)))
    with pytest.raises(ValueError, match="outside 1..4096"):
        f(np.zeros((5, 4097)), np.zeros((5, 4097)))
    with pytest.raises(ValueError, match=r"\[N, d\]"):
        f(np.zeros(4), a)
    b = a.copy()
    b[2, 3] = np.inf
    with pytest.raises(ValueError, match="fake has non-finite"):
        f(a, b)
    with pytest.raises(ValueError, match="real has non-finite"):
        f(b * np.nan, a)
    with pytest.raises(ValueError, match="real has non-finite"):
        prdc.RealRadii(b)


def test_finish():
    res = prdc.finish(np.array([3, 7, 20, 5], dtype=np.int64), 3, 10, 9)
    assert res == prdc.PRDCResult(3 / 9, 7 / 10, 20 / 27, 5 / 10, 3, 10, 9)
    assert all(type(v) is float for v in res[:4])


# -- the commands -----------------------------------------------------------------------------------------------------

def _eval_argv(tmp_path, *extra):
    return ["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", str(tmp_path)] + list(extra)


def _score_argv(tmp_path, *extra):
    return ["--resolution", "256", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)] + list(extra)


def test_prdc_flag_parses(tmp_path):
    assert not E.get_args(_eval_argv(tmp_path)).prdc and E.get_args(_eval_argv(tmp_path, "--prdc")).prdc
    assert not S.get_args(_score_argv(tmp_path)).prdc and S.get_args(_score_argv(tmp_path, "--prdc")).prdc


@pytest.mark.parametrize("command,argv", [(E, _eval_argv), (S, _score_argv)], ids=["evaluate_fid_lpips", "score_results"])
def test_prdc_with_real_stats_is_refused_before_any_work(tmp_path, command, argv):
    missing = tmp_path / "nothing_here"          # no images, no model: the refusal comes first
    with pytest.raises(ValueError, match="--prdc needs the real images' features.*--real-stats"):
        command.main(argv(missing, "--prdc", "--real-stats", str(missing / "s.npz")))


def test_library_refusals_before_any_work(tmp_path):
    missing = tmp_path / "nothing_here"
    stats = (np.zeros(2048), np.eye(2048))
    with pytest.raises(ValueError, match="--prdc needs"):
        E.evaluate("migan-256", missing / "m.pt", missing, real_stats=stats, prdc=True)
    with pytest.raises(ValueError, match="--prdc needs"):
        S.score(missing, missing, resolution=256, real_stats=stats, prdc=True)
    with pytest.raises(ValueError, match="real features"):
        E.Merge(4, "cpu", real_features=False, prdc=True)


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


class FakeRadii:
    """`prdc.RealRadii` stand-in: counts its constructions and keeps the real rows."""
    made = 0

    def __init__(self, real, k=3, max_fake=None):
        FakeRadii.made += 1
        self.rows, self.k, self.max_fake = real.clone(), k, max_fake


def fake_prdc(radii, fake, k=3):
    """A stand-in that sees which rows it got: all real rows, and the composed rows in dataset order."""
    assert isinstance(radii, FakeRadii) and len(fake) <= radii.max_fake
    r, f = radii.rows.double(), fake.double()
    w = (f * torch.arange(1, len(f) + 1)[:, None]).sum()
    return prdc.PRDCResult(float(w), float(r.sum()) * 1e-3, float(f.mean()), float(len(f)) / 7, radii.k, len(r),
                           len(f))


@pytest.fixture
def stand_ins(monkeypatch):
    monkeypatch.setattr(fid, "FeatureStatistics", RowStats)
    monkeypatch.setattr(fid, "BinnedFeatureStatistics", BinnedRows)
    monkeypatch.setattr(fid, "frechet_distance", fake_distance)
    monkeypatch.setattr(prdc, "RealRadii", FakeRadii)
    monkeypatch.setattr(prdc, "precision_recall_density_coverage", fake_prdc)
    FakeRadii.made = 0


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


def merged(n, batch, extra_values, edges, prdc_on, names=None):
    chunks = E.chunk_bounds(n, batch)
    merge = E.Merge(n, "cpu", True, extra_values=extra_values, hole_bins=edges, prdc=prdc_on, names=names)
    for j in range(len(chunks)):
        merge.add(stand_in(j, chunks, extra_values))
    return merge.result()


def _printed(res, *flags, **kw):
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, *flags, **kw)
    return out.getvalue().splitlines()


def test_prdc_lines_and_their_place():
    res = E.EvalResult(1.5, 0.25, np.zeros(2), 2, p_ids=0.1, u_ids=0.2)
    res.kid, res.ssim = 0.0123, 0.5
    res.prdc = prdc.PRDCResult(0.75, 0.5, 1.0833333333333333, 0.625, 3, 8, 4)
    res.by_hole = (E.HoleBin(0.0, 1.0, 2, 3.0, 0.25, kid=0.125, precision=0.5, recall=1.0, density=0.25,
                             coverage=math.nan),)
    assert _printed(res, True, True, False, True, True) == [
        "FID: 1.5", "LPIPS:  0.25", "SSIM: 0.5", "P-IDS: 0.1", "U-IDS: 0.2", "KID: 0.0123", "Precision: 0.75",
        "Recall: 0.5", "Density: 1.0833333333333333", "Coverage: 0.625",
        "HOLE [0.0, 1.0]: images 2 FID 3.0 LPIPS 0.25 KID 0.125 Precision 0.5 Recall 1.0 Density 0.25 Coverage nan"]
    assert _printed(res, False, prdc=True)[2:6] == ["Precision: 0.75", "Recall: 0.5", "Density: 1.0833333333333333",
                                                    "Coverage: 0.625"]


def test_hole_line_with_prdc():
    b = E.HoleBin(0.6, 1.0, 3, math.nan, 0.25, 0.5, math.inf, math.nan, math.nan, math.nan, math.nan, math.nan,
                  math.nan, math.nan)
    assert E.hole_line(b, True) == ("HOLE [0.6, 1.0]: images 3 FID nan LPIPS 0.25 SSIM 0.5 PSNR inf P-IDS nan U-IDS nan "
                                    "KID nan Precision nan Recall nan Density nan Coverage nan")
    b = E.HoleBin(0.0, 0.1, 812, 3.52, 0.0412, precision=0.75, recall=0.5, density=1.25, coverage=0.625)
    assert E.hole_line(b, False) == ("HOLE [0.0, 0.1): images 812 FID 3.52 LPIPS 0.0412 Precision 0.75 Recall 0.5 "
                                     "Density 1.25 Coverage 0.625")
    b = E.HoleBin(0.0, 0.1, 812, 3.52, 0.0412)
    assert (b.precision, b.recall, b.density, b.coverage) == (None,) * 4
    assert E.HoleBin._fields[-5:] == ("kid", "precision", "recall", "density", "coverage")


def test_merge_with_prdc(stand_ins):
    n, batch = 29, 8
    chunks = E.chunk_bounds(n, batch)
    parts = [stand_in(j, chunks, ("hole_fraction",)) for j in range(len(chunks))]
    real, fake = torch.cat([p.real for p in parts]), torch.cat([p.fake for p in parts])
    res = merged(n, batch, ("hole_fraction",), EDGES, True)
    assert FakeRadii.made == 1                  # once per command, for the overall value and every bin
    radii = FakeRadii(real, 3, n)
    assert res.prdc == fake_prdc(radii, fake) and res.kid is None and res.p_ids is None and len(res) == 8
    h = torch.cat([p.extra[:, 0] for p in parts]).numpy().astype(np.float64)
    bins = np.searchsorted(np.array(EDGES[1:-1]), h, side="right")
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert b.count == len(idx) > 3
        assert tuple(b[-4:]) == tuple(fake_prdc(radii, fake[idx])[:4]) and b.kid is None
    # at k = 3 images or fewer a bin's four values are nan; at 4 they are computed
    FakeRadii.made = 0
    small = merged(15, 4, ("hole_fraction",), (0.0, 0.1, 0.2, 0.5, 1.0), True)   # h = i % 8 / 7
    assert FakeRadii.made == 1
    assert [b.count for b in small.by_hole] == [2, 2, 4, 7]
    assert all(math.isnan(v) for b in small.by_hole[:2] for v in b[-4:])
    assert all(not math.isnan(v) for b in small.by_hole[2:] for v in b[-4:])


def test_without_prdc_nothing_changes(stand_ins, tmp_path):
    names = ["img_%02d" % i for i in range(29)]
    on = merged(29, 8, ("hole_fraction", "ssim", "psnr"), EDGES, True, names)
    off = merged(29, 8, ("hole_fraction", "ssim", "psnr"), EDGES, False, names)
    assert off.prdc is None and all(b[-4:] == (None,) * 4 for b in off.by_hole)
    assert (on.fid, on.lpips, on.count, on.ssim, on.psnr) == (off.fid, off.lpips, off.count, off.ssim, off.psnr)
    assert on.lpips_values.tobytes() == off.lpips_values.tobytes()
    assert [b[:-4] for b in on.by_hole] == [b[:-4] for b in off.by_hole]
    lines_on = _printed(on, False, True, True, False, True)
    lines_off = _printed(off, False, True, True)
    assert [ln for ln in lines_on if ln.split(":")[0] not in ("Precision", "Recall", "Density", "Coverage")
            and not ln.startswith("HOLE")] == [ln for ln in lines_off if not ln.startswith("HOLE")]
    assert [ln.split(" Precision ")[0] for ln in lines_on if ln.startswith("HOLE")] == \
        [ln for ln in lines_off if ln.startswith("HOLE")]
    assert _printed(off, False, True, True) == _printed(off, False, True, True, False, False)
    E.write_per_image(tmp_path / "on.csv", on.per_image)
    E.write_per_image(tmp_path / "off.csv", off.per_image)
    assert (tmp_path / "on.csv").read_bytes() == (tmp_path / "off.csv").read_bytes()
    assert FakeRadii.made == 1 and E.Merge(4, "cpu", True).kept is None

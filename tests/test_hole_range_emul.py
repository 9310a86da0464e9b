"""Hole-range masks and binned feature statistics without a GPU, in the emulation builds.

- migan_mask_plan_range + b200_mask_raster + b200_mask_compact_range, driven as RandomMaskStream drives them, equal
  tests/golden/masks_hole_range.npz (the reference's RandomMask(s, hole_range)): masks or digests, hole counts,
  attempts and the final numpy state;
- hole_range [0, 1] through the new entry points equals the old ones on tests/golden/masks.npz;
- migan_mask_hole_bounds equals the float64 predicate at every hole count at s = 32 and around each fixture range's
  bounds at 512, and refuses the ranges RandomMask cannot draw;
- oracle/masks_range_oracle.py reproduces the fixture at s = 32;
- fid_stats_update_binned equals fid_stats_update on each bin's rows, bit for bit."""
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
from oracle import masks_oracle as M  # noqa: E402
from oracle import masks_range_oracle as MR  # noqa: E402

NAMES = ("migan_np_seed", "migan_mask_plan", "b200_mask_raster", "b200_mask_compact", "migan_mask_plan_range",
         "migan_mask_hole_bounds", "b200_mask_compact_range")
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "masks_hole_range.npz"))
OLD = np.load(os.path.join(ROOT, "tests", "golden", "masks.npz"))
RANGES = [tuple(r) for r in GOLDEN["ranges"]]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), [s for s in _abi.SYMBOLS if s[0] in NAMES])


def bounds(lib, s, lo, hi):
    a, b = ctypes.c_int(), ctypes.c_int()
    rc = lib.migan_mask_hole_bounds(s, lo, hi, ctypes.byref(a), ctypes.byref(b))
    return rc, a.value, b.value


def emul_stream(lib, s, n, hole_range=None, call=None):
    """The emulated RandomMaskStream, in calls of `call` masks; hole_range None drives the [0, 1] entry points.
    Returns (masks, attempts, final state)."""
    st = _abi.NpRandom()
    assert lib.migan_np_seed(ctypes.byref(st), 0) == 0
    if hole_range is None:
        h_min, h_max = 1, s * s - 1
    else:
        rc, h_min, h_max = bounds(lib, s, *hole_range)
        assert rc == 0
    out, attempts = [], 0
    for c0 in range(0, n, call or n):
        want, got = min(call or n, n - c0), 0
        while got < want:
            need = want - got
            a = 4 * need + 8
            recs, states = (_abi.MaskRecord * a)(), (_abi.NpRandom * a)()
            cur = _abi.NpRandom.from_buffer_copy(st)
            if hole_range is None:
                assert lib.migan_mask_plan(ctypes.byref(cur), s, a, recs, states) == 0
            else:
                assert lib.migan_mask_plan_range(ctypes.byref(cur), s, hole_range[0], hole_range[1], a, recs, states) == 0
            att = np.empty((a, s, s), np.uint8)
            holes = np.empty(a, np.int32)
            assert lib.b200_mask_raster(recs, a, s, att.ctypes.data, holes.ctypes.data, None) == 0
            o = np.full((need, s, s), 7, np.uint8)
            if hole_range is None:
                assert lib.b200_mask_compact(att.ctypes.data, holes.ctypes.data, a, s, need, o.ctypes.data, None) == 0
            else:
                assert lib.b200_mask_compact_range(att.ctypes.data, holes.ctypes.data, a, s, h_min, h_max, need,
                                                   o.ctypes.data, None) == 0
            ok = np.flatnonzero((holes >= h_min) & (holes <= h_max))
            took = min(need, len(ok))
            used = int(ok[need - 1]) + 1 if len(ok) >= need else a
            np.testing.assert_array_equal(o[:took], att[ok[:took]])
            out.append(o[:took])
            st = _abi.NpRandom.from_buffer_copy(states[used - 1])
            attempts += used
            got += took
    return np.concatenate(out), attempts, st


def assert_state(st, key, golden=GOLDEN):
    rest = golden[key + "_rest"]
    np.testing.assert_array_equal(np.array(st.key, np.uint32), golden[key + "_state"])
    assert (st.pos, st.has_gauss, st.gauss) == (int(rest[0]), int(rest[1]), float(rest[2]))


def check_masks(masks, key, s):
    n = masks.shape[0]
    assert np.array_equal((masks == 0).reshape(n, -1).sum(1), GOLDEN[key + "_holes"])
    if s == 32:
        bits = np.unpackbits(GOLDEN[key], axis=1, count=s * s).reshape(-1, s, s)
        assert np.array_equal(masks, np.where(bits == 1, 255, 0).astype(np.uint8))
    else:
        got = np.frombuffer(b"".join(M.digest(m) for m in masks), np.uint8).reshape(n, 8)
        assert np.array_equal(got, GOLDEN[key + "_digest"])


@pytest.mark.parametrize("s", [32, 256, 512])
@pytest.mark.parametrize("i", range(5))
def test_emulated_stream_equals_fixture(emul, i, s):
    key = "r%d_%d" % (i, s)
    n = GOLDEN[key + "_holes"].shape[0]
    masks, attempts, st = emul_stream(emul, s, n, RANGES[i], call=None if s > 32 else 7)
    check_masks(masks, key, s)
    assert attempts == int(GOLDEN[key + "_attempts"])
    assert_state(st, key)


@pytest.mark.parametrize("s", [32, 64])
def test_full_range_through_new_entry_points_equals_old(emul, s):
    n = OLD["m0_%d" % s].shape[0]
    new = emul_stream(emul, s, n, (0.0, 1.0))
    old = emul_stream(emul, s, n, None)
    assert np.array_equal(new[0], old[0]) and new[1] == old[1] == int(OLD["m0_%d_attempts" % s])
    bits = np.unpackbits(OLD["m0_%d" % s], axis=1, count=s * s).reshape(-1, s, s)
    assert np.array_equal(new[0], np.where(bits == 1, 255, 0).astype(np.uint8))
    assert_state(new[2], "m0_%d" % s, OLD)
    assert bounds(emul, s, 0.0, 1.0) == (0, 1, s * s - 1)


def test_hole_bounds_equal_the_predicate(emul):
    s = 32
    ranges = RANGES + [(0.0, 1.0), (0.3, 0.30001), (0.5, 0.5 + 2 ** -40), (0.1, 1.0), (0.0, 0.9990234375)]
    for lo, hi in ranges:
        keep = [not (MR.hole_ratio(h, s) <= lo or MR.hole_ratio(h, s) >= hi) for h in range(s * s + 1)]
        rc, h_min, h_max = bounds(emul, s, lo, hi)
        assert rc == 0
        assert keep == [h_min <= h <= h_max for h in range(s * s + 1)], (lo, hi, h_min, h_max)
    s = 512
    for lo, hi in RANGES:
        rc, h_min, h_max = bounds(emul, s, lo, hi)
        assert rc == 0 and h_min <= h_max
        for h in (h_min - 1, h_min, h_min + 1, h_max - 1, h_max, h_max + 1):
            r = MR.hole_ratio(h, s)
            assert (not (r <= lo or r >= hi)) == (h_min <= h <= h_max), (lo, hi, h)


@pytest.mark.parametrize("lo,hi", [(0.2, 0.2), (0.5, 0.4), (-0.1, 0.5), (0.5, 1.5), (float("nan"), 1.0),
                                   (0.0, float("inf")), (0.0, 0.1), (0.05, 0.149)])
def test_refused_ranges(emul, lo, hi):
    assert bounds(emul, 32, lo, hi)[0] != 0
    st = _abi.NpRandom()
    emul.migan_np_seed(ctypes.byref(st), 0)
    before = bytes(st)
    recs = (_abi.MaskRecord * 1)()
    assert emul.migan_mask_plan_range(ctypes.byref(st), 32, lo, hi, 1, recs, None) != 0
    assert bytes(st) == before                                           # nothing drawn


def test_smallest_range_numpy_draws(emul):
    assert MR.tries((0.0, 0.2)) == (2, 1, 4) and bounds(emul, 32, 0.0, 0.2)[0] == 0
    assert MR.tries((0.05, 0.1499)) == (1, 0, 3)


@pytest.mark.parametrize("i", range(5))
def test_oracle_equals_fixture(i):
    key = "r%d_32" % i
    n = GOLDEN[key + "_holes"].shape[0]
    masks, attempts = MR.random_masks(32, n, RANGES[i])
    check_masks(masks, key, 32)
    assert attempts == int(GOLDEN[key + "_attempts"])


# ---- binned feature statistics ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def incep():
    path = build_emul._compile("inception_emul", [os.path.join(build_emul.CSRC, s) for s in ("inception_abi.cu",
                                                                                              "abi_error.cu")])
    return fid.lib(ctypes.CDLL(path))


@pytest.mark.parametrize("dim,nbins,sizes", [(64, 2, [1, 32, 1, 5]), (64, 32, [32, 32, 1, 17]), (2048, 3, [1, 32, 4]),
                                             (64, 7, [32] * 3)])
def test_binned_statistics_equal_per_bin_updates(incep, dim, nbins, sizes):
    rng = np.random.default_rng(dim + nbins)
    shift, s1 = np.zeros((nbins, dim)), np.zeros((nbins, dim))
    s2, count = np.zeros((nbins, dim, dim)), np.zeros(nbins, np.int64)
    want = [[np.zeros(dim), np.zeros(dim), np.zeros((dim, dim)), 0] for _ in range(nbins)]
    for call, n in enumerate(sizes):
        x = np.ascontiguousarray((rng.normal(size=(n, dim)) * 2 + 500).astype(np.float32))
        # the first call leaves the upper bins empty, so they first get rows in a later call; -1 rows go nowhere
        top = max(1, nbins // 2) if call == 0 else nbins
        bins = rng.integers(-1, top, n).astype(np.int32)
        rc = incep.fid_stats_update_binned(x.ctypes.data, bins.ctypes.data, n, dim, nbins, shift.ctypes.data,
                                           s1.ctypes.data, s2.ctypes.data, count.ctypes.data, None)
        _abi.check(rc, incep)
        for b in range(nbins):
            rows = np.ascontiguousarray(x[bins == b])
            if not len(rows):
                continue
            w = want[b]
            _abi.check(incep.fid_stats_update(rows.ctypes.data, len(rows), dim, w[0].ctypes.data, w[1].ctypes.data,
                                              w[2].ctypes.data, int(w[3] == 0), None), incep)
            w[3] += len(rows)
    for b in range(nbins):
        assert count[b] == want[b][3]
        assert np.array_equal(shift[b], want[b][0]) and np.array_equal(s1[b], want[b][1])
        assert np.array_equal(s2[b], want[b][2]), b
    assert (count > 0).sum() >= min(nbins, 2)


def test_binned_statistics_refusals(incep):
    x, bins = np.zeros((2, 4), np.float32), np.zeros(2, np.int32)
    buf, cnt = np.zeros(40 * 16), np.zeros(40, np.int64)
    for nbins in (0, fid.MAX_BINS + 1):
        assert incep.fid_stats_update_binned(x.ctypes.data, bins.ctypes.data, 2, 4, nbins, buf.ctypes.data,
                                             buf.ctypes.data, buf.ctypes.data, cnt.ctypes.data, None) != 0
    with pytest.raises(ValueError, match="bins"):
        fid.BinnedFeatureStatistics(fid.MAX_BINS + 1, device="cpu")

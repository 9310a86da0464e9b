"""CPU checks of the free-form mask generator (mi-gan_b200/csrc/masks.cu) and its oracle (oracle/masks_oracle.py).

- the planner (the product's host code: numpy's MT19937 and legacy distributions, the RandomMask attempt walk) makes the
  oracle's draws on np.random.RandomState for several seeds and sizes: every record, and the state after every attempt
  equals np.random.get_state()'s;
- the emulation build of the rasterizer (the same block functions, threads in turn) equals Pillow's ImageDraw on a sweep
  of single wide lines, including vertices on and beyond the canvas edge, and its disc stamps equal ImageDraw.ellipse;
- the emulated stream (plan, raster, compact, rewind, plan again) equals tests/golden/masks.npz byte for byte at every
  stored size, with the attempts and the final state, when it is split into small calls (repeated planning at s = 32),
  and its digests of the first 2000 masks at 512 and 1000 at 256 match;
- the oracle equals the fixture, and where Pillow is installed its rasterizer equals Pillow's on the fixture's attempts."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

from migan_b200 import _abi  # noqa: E402
from oracle import masks_oracle as M  # noqa: E402
import build_emul  # noqa: E402

NAMES = ("migan_np_seed", "migan_mask_plan", "b200_mask_raster", "b200_mask_compact")
SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "masks.npz"))
LISTS = [(0, 32), (0, 64), (0, 256), (0, 512), (7, 128)]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), SYMBOLS)


def seeded(lib, seed):
    st = _abi.NpRandom()
    assert lib.migan_np_seed(ctypes.byref(st), seed) == 0
    return st


def state_tuple(st):
    return np.array(st.key, np.uint32), st.pos, st.has_gauss, st.gauss


def assert_state(st, np_state):
    key, pos, has_gauss, gauss = state_tuple(st)
    assert np_state[0] == "MT19937"
    np.testing.assert_array_equal(key, np_state[1])
    assert (pos, has_gauss, gauss) == (np_state[2], np_state[3], np_state[4])


def plan(lib, st, s, a):
    recs, states = (_abi.MaskRecord * a)(), (_abi.NpRandom * a)()
    assert lib.migan_mask_plan(ctypes.byref(st), s, a, recs, states) == 0
    return recs, states


def record_attempt(r: _abi.MaskRecord):
    """(rects, quads, discs, flips) of one record, comparable with the oracle's Attempt."""
    rects = [tuple(r.rects[i]) for i in range(r.n_rects)]
    quads = [tuple(r.quads[i]) for i in range(r.n_segments)]
    discs = [tuple(r.discs[i])[:3] for i in range(r.n_discs)]
    return rects, quads, discs, (bool(r.flips & 1), bool(r.flips & 2))


def oracle_quad(x0, y0, x1, y1, w):
    v = M.quad(x0, y0, x1, y1, w)
    return tuple([x0, y0] * 4) if v is None else tuple(c for p in v for c in p)


def raster(lib, recs, a, s):
    att = np.empty((a, s, s), np.uint8)
    holes = np.empty(a, np.int32)
    assert lib.b200_mask_raster(recs, a, s, att.ctypes.data, holes.ctypes.data, None) == 0
    return att, holes


def emul_stream(lib, s, n, seed=0, call=None, round_max=None):
    """The emulated RandomMaskStream: n masks in calls of `call` (all at once when None), at most `round_max` attempts
    planned per round.  Returns (masks, attempts, final state)."""
    st = seeded(lib, seed)
    out, attempts = [], 0
    for c0 in range(0, n, call or n):
        want = min(call or n, n - c0)
        got = 0
        while got < want:
            need = want - got
            a = need + need // 8 + 2 if round_max is None else min(round_max, need + 2)
            recs, states = plan(lib, _abi.NpRandom.from_buffer_copy(st), s, a)
            att, holes = raster(lib, recs, a, s)
            o = np.full((need, s, s), 7, np.uint8)
            assert lib.b200_mask_compact(att.ctypes.data, holes.ctypes.data, a, s, need, o.ctypes.data, None) == 0
            ok = np.flatnonzero((holes > 0) & (holes < s * s))
            took = min(need, len(ok))
            used = int(ok[need - 1]) + 1 if len(ok) >= need else a
            np.testing.assert_array_equal(o[:took], att[ok[:took]])
            out.append(o[:took])
            st = _abi.NpRandom.from_buffer_copy(states[used - 1])
            attempts += used
            got += took
    return np.concatenate(out), attempts, st


def golden_masks(seed, s):
    bits = GOLDEN["m%d_%d" % (seed, s)]
    return np.where(np.unpackbits(bits, axis=1, count=s * s).reshape(-1, s, s) == 1, 255, 0).astype(np.uint8)


def golden_state(prefix):
    rest = GOLDEN[prefix + "_rest"]
    return ("MT19937", GOLDEN[prefix + "_state"], int(rest[0]), int(rest[1]), float(rest[2]))


# ---- the planner: numpy's draws ------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,s", [(0, 2), (0, 3), (1, 32), (12345, 100), (0, 512), (2**32 - 1, 4096)])
def test_planner_draws_equal_numpy(emul, seed, s):
    a = 25
    recs, states = plan(emul, seeded(emul, seed), s, a)
    rs = np.random.RandomState(seed)
    for k in range(a):
        want = M.plan_attempt(rs, s)
        rects, quads, discs, flips = record_attempt(recs[k])
        assert rects == want.rects
        assert quads == [oracle_quad(*seg) for seg in want.segments]
        assert discs == want.discs
        assert flips == (want.flip_rows, want.flip_cols)
        assert_state(states[k], rs.get_state())


def test_seed_equals_numpy(emul):
    for seed in (0, 1, 2**31, 2**32 - 1):
        assert_state(seeded(emul, seed), np.random.RandomState(seed).get_state())


def test_planner_refuses_sizes(emul):
    st = seeded(emul, 0)
    recs = (_abi.MaskRecord * 1)()
    for s in (1, 0, -3, 4097):
        assert emul.migan_mask_plan(ctypes.byref(st), s, 1, recs, None) == _abi.ERR_INVALID
    assert emul.migan_mask_plan(ctypes.byref(st), 64, 0, recs, None) == _abi.ERR_INVALID
    assert_state(st, np.random.RandomState(0).get_state())       # a refused call draws nothing


# ---- the rasterizer: Pillow's wide lines and ellipses --------------------------------------------------------------
def one_segment_record(x0, y0, x1, y1, w):
    r = _abi.MaskRecord()
    r.n_segments = 1
    for i, c in enumerate(oracle_quad(x0, y0, x1, y1, w)):
        r.quads[0][i] = c
    return r


def test_raster_segments_equal_pillow(emul):
    Image = pytest.importorskip("PIL.Image")
    ImageDraw = pytest.importorskip("PIL.ImageDraw")
    rng = np.random.default_rng(5)
    for s in (16, 33, 64, 160):
        n = 300
        recs = (_abi.MaskRecord * n)()
        segs = []
        for k in range(n):
            w = int(rng.integers(12, 48))
            x0, y0 = (int(v) for v in rng.integers(0, s + 1, 2))
            kind = k % 4
            if kind == 0:
                x1, y1 = x0, y0
            elif kind == 1:
                x1, y1 = x0 + int(rng.integers(-3, 4)), y0 + int(rng.integers(-3, 4))
            elif kind == 2:
                x1, y1 = (x0, int(rng.integers(0, s + 1))) if k % 8 == 2 else (int(rng.integers(0, s + 1)), y0)
            else:
                x1, y1 = (int(v) for v in rng.integers(0, s + 1, 2))
            segs.append((x0, y0, x1, y1, w))
            recs[k] = one_segment_record(x0, y0, x1, y1, w)
        att, holes = raster(emul, recs, n, s)
        for k, (x0, y0, x1, y1, w) in enumerate(segs):
            img = Image.new("L", (s, s), 0)
            ImageDraw.Draw(img).line([(x0, y0), (x1, y1)], fill=1, width=w)
            want = np.where(np.asarray(img) == 1, 0, 255)
            np.testing.assert_array_equal(att[k], want, err_msg="segment %s on %d x %d" % ((x0, y0, x1, y1, w), s, s))
            assert holes[k] == int((want == 0).sum())


def test_disc_table_equals_pillow():
    Image = pytest.importorskip("PIL.Image")
    ImageDraw = pytest.importorskip("PIL.ImageDraw")
    for r in range(M.DISC_R_MIN, M.DISC_R_MAX + 1):
        for cx, cy in ((50, 50), (0, 3), (99, 97), (-5, 40)):
            img = Image.new("L", (100, 100), 0)
            ImageDraw.Draw(img).ellipse((cx - r, cy - r, cx + r, cy + r), fill=1)
            want = np.zeros((100, 100), np.uint8)
            M._paint_spans(want, M.disc_spans(cx, cy, r))
            np.testing.assert_array_equal(np.asarray(img), want, err_msg="r = %d at (%d, %d)" % (r, cx, cy))


def test_raster_discs_and_flips(emul):
    """Discs at the canvas edges and every flip combination: the emulated raster equals the oracle's."""
    rs = np.random.RandomState(3)
    s, a = 48, 24
    recs, _ = plan(emul, seeded(emul, 3), s, a)
    att, holes = raster(emul, recs, a, s)
    for k in range(a):
        want = M.raster(M.plan_attempt(rs, s), s)
        np.testing.assert_array_equal(att[k], want)
        assert holes[k] == int((want == 0).sum())


# ---- the stream against the reference's masks ----------------------------------------------------------------------
@pytest.mark.parametrize("seed,s", LISTS)
def test_emul_stream_equals_fixture(emul, seed, s):
    want = golden_masks(seed, s)
    got, attempts, st = emul_stream(emul, s, len(want), seed)
    np.testing.assert_array_equal(got, want)
    assert attempts == int(GOLDEN["m%d_%d_attempts" % (seed, s)])
    assert_state(st, golden_state("m%d_%d" % (seed, s)))


@pytest.mark.parametrize("call,round_max", [(1, None), (7, 3), (32, 16)])
def test_emul_stream_split_at_32(emul, call, round_max):
    """At s = 32 most attempts are all-hole, so every call plans again; the bytes do not depend on the split."""
    want = golden_masks(0, 32)
    got, attempts, st = emul_stream(emul, 32, len(want), 0, call=call, round_max=round_max)
    np.testing.assert_array_equal(got, want)
    assert attempts == int(GOLDEN["m0_32_attempts"])
    assert_state(st, golden_state("m0_32"))


@pytest.mark.parametrize("s", [256, 512])
def test_emul_stream_digests(emul, s):
    want = GOLDEN["digest0_%d" % s]
    got, attempts, st = emul_stream(emul, s, len(want), 0, call=250)
    digests = np.frombuffer(b"".join(M.digest(m) for m in got), np.uint8).reshape(-1, 8)
    np.testing.assert_array_equal(digests, want)
    assert attempts == int(GOLDEN["digest0_%d_attempts" % s])
    assert_state(st, golden_state("digest0_%d" % s))


# ---- the oracle against the reference's masks ----------------------------------------------------------------------
@pytest.mark.parametrize("seed,s,n", [(0, 32, 200), (0, 64, 40), (0, 256, 6), (0, 512, 3), (7, 128, 12)])
def test_oracle_equals_fixture(seed, s, n):
    got, _ = M.random_masks(s, n, seed)
    np.testing.assert_array_equal(got, golden_masks(seed, s)[:n])


def test_oracle_pillow_path_equals_fixture():
    pytest.importorskip("PIL.ImageDraw")
    got, attempts = M.random_masks(32, 200, 0, pillow=True)
    np.testing.assert_array_equal(got, golden_masks(0, 32))
    assert attempts == int(GOLDEN["m0_32_attempts"])

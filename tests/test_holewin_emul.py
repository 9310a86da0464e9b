"""CPU checks of the hole-window request path (mi-gan_b200/csrc/holewin.cu, the window kernels of fullres.cu).

- the window planner (migan_hole_windows, host code) equals oracle/holewin_oracle.py on a few
  hundred seeded random cell grids and on named cases, and every result keeps the invariants: windows disjoint and inside
  the photo, every hole cell's pixels covered, every side a valid forward_fc size or the photo's side, the count within
  migan_hole_windows_max;
- the emulation build of the cells kernel (the same block functions, threads in turn) equals the oracle's cells for every
  mask channel count, both invert values, partial cells and unaligned mask rows;
- the emulated window pre- and post-processing equal the full-resolution oracle on each window's crop, pasted into the
  photo, byte for byte; nothing outside the windows is written."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

from migan_b200 import _abi  # noqa: E402
from oracle import fullres_oracle as F  # noqa: E402
from oracle import holewin_oracle as HW  # noqa: E402
import build_emul  # noqa: E402

NAMES = ("b200_hole_cells_bytes", "b200_hole_cells", "b200_window_preprocess", "b200_window_postprocess",
         "migan_hole_windows", "migan_hole_windows_max", "migan_last_error")
SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), SYMBOLS)


# ---- the window planner (host code) ---------------------------------------------------------------
def plan(lib, cells, H, W, R, margin=1):
    mx = ctypes.c_int()
    _abi.check(lib.migan_hole_windows_max(H, W, R, ctypes.byref(mx)))
    assert mx.value == HW.max_windows(H, W, R)
    buf = (ctypes.c_int * (4 * mx.value))()
    cnt = ctypes.c_int()
    cells = np.ascontiguousarray(cells, np.uint8)
    _abi.check(lib.migan_hole_windows(cells.ctypes.data, H, W, R, margin, buf, mx.value, ctypes.byref(cnt)))
    return [tuple(buf[4 * k:4 * k + 4]) for k in range(cnt.value)]


def check_invariants(wins, cells, H, W, R):
    q = R // 4
    cover = np.zeros((H, W), np.int32)
    for y0, x0, h, w in wins:
        assert 0 <= y0 and y0 + h <= H and 0 <= x0 and x0 + w <= W, (y0, x0, h, w)
        for side, n in ((h, H), (w, W)):
            assert side == n or (side % q == 0 and side >= R), (side, n)
        cover[y0:y0 + h, x0:x0 + w] += 1
    assert cover.max(initial=0) <= 1, "windows overlap"
    hole_px = np.kron(cells, np.ones((q, q), np.int32))[:H, :W] > 0
    assert np.all(cover[hole_px] == 1), "a hole cell is not covered"
    assert len(wins) <= HW.max_windows(H, W, R)
    assert wins == sorted(wins)


def _grid(H, W, R):
    q = R // 4
    return np.zeros((-(-H // q), -(-W // q)), np.uint8)


@pytest.mark.parametrize("seed", range(300))
def test_planner_random_grids(emul, seed):
    rng = np.random.default_rng(seed)
    R = int(rng.choice([16, 64, 256]))
    H, W = int(rng.integers(1, 12 * R)), int(rng.integers(1, 12 * R))
    margin = int(rng.integers(0, 3))
    g = _grid(H, W, R)
    g[...] = rng.random(g.shape) < float(rng.choice([0.002, 0.02, 0.1, 0.5]))
    wins = plan(emul, g, H, W, R, margin)
    assert wins == HW.windows(g, H, W, R, margin), (R, H, W, margin)
    check_invariants(wins, g, H, W, R)


def test_planner_empty_mask_gives_no_windows(emul):
    assert plan(emul, _grid(3024, 4032, 512), 3024, 4032, 512) == []


def test_planner_all_hole_gives_the_whole_photo(emul):
    for R, H, W in [(512, 3024, 4032), (256, 1000, 1001), (64, 30, 70)]:
        g = _grid(H, W, R) + 1
        assert plan(emul, g, H, W, R) == [(0, 0, H, W)]


def test_planner_distant_and_close_holes(emul):
    R, H, W = 512, 2160, 3840
    g = _grid(H, W, R)
    g[2, 2] = g[14, 26] = 1                              # opposite ends: two windows of R x R around the cells
    wins = plan(emul, g, H, W, R)
    assert wins == [(64, 64, 512, 512), (1600, 3136, 512, 512)]
    check_invariants(wins, g, H, W, R)
    g[...] = 0
    g[5, 5] = g[5, 9] = 1                                # windows [448, 960) and [960, 1472) only touch: two windows
    assert plan(emul, g, H, W, R) == [(448, 448, 512, 512), (448, 960, 512, 512)]
    g[5, 9], g[5, 8] = 0, 1                              # [448, 960) and [832, 1344) overlap: one window over cells 5..8
    wins = plan(emul, g, H, W, R)
    assert wins == HW.windows(g, H, W, R) == [(448, 512, 512, 768)]
    check_invariants(wins, g, H, W, R)


@pytest.mark.parametrize("where", ["tl", "tr", "bl", "br", "top", "bottom", "left", "right"])
def test_planner_corners_and_edges(emul, where):
    R, H, W = 256, 1000, 1500                            # sides not multiples of q = 64: partial last cells
    g = _grid(H, W, R)
    gh, gw = g.shape
    pos = {"tl": (0, 0), "tr": (0, gw - 1), "bl": (gh - 1, 0), "br": (gh - 1, gw - 1), "top": (0, gw // 2),
           "bottom": (gh - 1, gw // 2), "left": (gh // 2, 0), "right": (gh // 2, gw - 1)}[where]
    g[pos] = 1
    wins = plan(emul, g, H, W, R)
    assert wins == HW.windows(g, H, W, R) and len(wins) == 1
    check_invariants(wins, g, H, W, R)


def test_planner_photo_smaller_than_R_and_margin_0(emul):
    R = 512
    g = _grid(300, 400, R)
    g[1, 1] = 1
    assert plan(emul, g, 300, 400, R) == [(0, 0, 300, 400)]
    R, H, W = 256, 777, 1333                             # q = 64
    g = _grid(H, W, R)
    g[5, 10:13] = 1                                      # three cells: 5 with the margin (320 wide), 3 without (256)
    assert plan(emul, g, H, W, R, 1) == HW.windows(g, H, W, R, 1) == [(224, 576, 256, 320)]
    wins = plan(emul, g, H, W, R, 0)
    assert wins == HW.windows(g, H, W, R, 0) == [(224, 608, 256, 256)]
    check_invariants(wins, g, H, W, R)


def test_planner_refusals(emul):
    mx = ctypes.c_int()
    assert emul.migan_hole_windows_max(0, 5, 256, ctypes.byref(mx)) == _abi.ERR_INVALID
    assert emul.migan_hole_windows_max(5, 5, 100, ctypes.byref(mx)) == _abi.ERR_INVALID
    g = np.ones((1, 1), np.uint8)
    buf, cnt = (ctypes.c_int * 4)(), ctypes.c_int()
    assert emul.migan_hole_windows(g.ctypes.data, 5, 5, 256, -1, buf, 1, ctypes.byref(cnt)) == _abi.ERR_INVALID
    assert emul.migan_hole_windows(g.ctypes.data, 5, 5, 256, 1, buf, 0, ctypes.byref(cnt)) == _abi.ERR_INVALID
    assert "room" in emul.migan_last_error().decode()


# ---- the cells kernel (emulation build) ----------------------------------------------------------------------------
def _mask(rng, H, W, C, hole_frac=0.002):
    m = np.where(rng.random((H, W, C)) < 0.5, 255, rng.choice(np.array([0, 1, 254], np.uint8), (H, W, C))).astype(np.uint8)
    ch = {1: 0, 2: 1, 3: 0, 4: 3}[C]
    sel = rng.random((H, W)) >= hole_frac
    m[..., ch] = np.where(sel, 255, rng.choice(np.array([0, 7, 254], np.uint8), (H, W)))
    return m


def run_cells(lib, masks, inverts, R, offset=0):
    """Emulated b200_hole_cells over one batch; each mask is copied `offset` bytes into a buffer (unaligned rows)."""
    n = len(masks)
    table = (_abi.CellsRequest * n)()
    keep = []
    for r, m, inv in zip(table, masks, inverts):
        buf = np.zeros(m.size + offset + 16, np.uint8)
        buf[offset:offset + m.size] = m.reshape(-1)
        keep.append(buf)
        r.mask, r.H, r.W = buf.ctypes.data + offset, m.shape[0], m.shape[1]
        r.mask_channels, r.invert = 1 if m.ndim == 2 else m.shape[2], int(inv)
    total = lib.b200_hole_cells_bytes(table, n, R)
    cells = np.full(total, 77, np.uint8)
    assert lib.b200_hole_cells(table, n, R, cells.ctypes.data, None) == 0
    out, off = [], 0
    for m in masks:
        gh, gw = -(-m.shape[0] // (R // 4)), -(-m.shape[1] // (R // 4))
        out.append(cells[off:off + gh * gw].reshape(gh, gw))
        off += gh * gw
    assert off == total
    return out


@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("inv", [False, True])
def test_cells_equal_oracle(emul, C, inv):
    rng = np.random.default_rng(10 * C + inv)
    sizes = [(300, 500), (257, 129), (64, 64), (1, 1000), (1000, 1), (77, 33), (130, 700)]
    for R in (16, 64, 256):
        masks = []
        for H, W in sizes:
            m = _mask(rng, H, W, C)
            if inv:
                m = 255 - m
            masks.append(np.ascontiguousarray(m[..., 0]) if C == 1 else m)
        for offset in (0, 5):
            got = run_cells(emul, masks, [inv] * len(masks), R, offset)
            for k, m in enumerate(masks):
                want = HW.cells(m, inv, R)
                assert np.array_equal(got[k], want), (R, sizes[k], offset)


def test_cells_single_hole_pixel_in_partial_cell(emul):
    R, H, W = 256, 200, 333                                 # q = 64: the last cell column is 13 pixels wide
    for y, x in [(0, 0), (199, 332), (130, 320), (63, 64), (64, 63)]:
        m = np.full((H, W, 4), 255, np.uint8)
        m[y, x, 3] = 0
        m[y, x, :3] = 0                                     # other channels do not matter
        got = run_cells(emul, [m], [False], R)[0]
        want = np.zeros_like(got)
        want[y // 64, x // 64] = 1
        assert np.array_equal(got, want), (y, x)


def test_cells_batch_of_32(emul):
    rng = np.random.default_rng(32)
    masks, invs = [], []
    for k in range(32):
        H, W, C = int(rng.integers(1, 400)), int(rng.integers(1, 400)), int(rng.integers(1, 5))
        m = _mask(rng, H, W, C, 0.01)
        masks.append(np.ascontiguousarray(m[..., 0]) if C == 1 else m)
        invs.append(False)
    got = run_cells(emul, masks, invs, 64, offset=3)
    for k, m in enumerate(masks):
        assert np.array_equal(got[k], HW.cells(m, False, 64)), k


# ---- the window pre- and post-processing (emulation build) ---------------------------------------------------------
def run_windows(lib, img, mask, inv, wins, ys, R):
    """Emulated window pre / post over one pass of windows of one photo, written into a copy of it."""
    n = len(wins)
    table = (_abi.WindowRequest * n)()
    out = img.copy()
    xs, yb = [], []
    for r, win, y in zip(table, wins, ys):
        Hp, Wp = F.extent(win[2], win[3], R)
        x = np.full((4, Hp, Wp), np.nan, np.float32)
        xs.append(x)
        yb.append(np.ascontiguousarray(y, np.float32))
        r.img, r.mask, r.H, r.W = img.ctypes.data, mask.ctypes.data, img.shape[0], img.shape[1]
        r.mask_channels, r.invert = 1 if mask.ndim == 2 else mask.shape[2], int(inv)
        r.y0, r.x0, r.h, r.w = win
        r.x, r.y, r.Hp, r.Wp, r.out = x.ctypes.data, yb[-1].ctypes.data, Hp, Wp, out.ctypes.data
    assert lib.b200_window_preprocess(table, n, None) == 0
    assert lib.b200_window_postprocess(table, n, None) == 0
    return xs, out


@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("inv", [False, True])
def test_windows_equal_oracle(emul, C, inv):
    rng = np.random.default_rng(100 + 10 * C + inv)
    R, H, W = 64, 300, 460                               # q = 16
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    m = _mask(rng, H, W, C, 0.0)
    ch = {1: 0, 2: 1, 3: 0, 4: 3}[C]
    for y0, x0, h, w in [(5, 7, 20, 30), (200, 400, 90, 55), (150, 0, 3, 460)]:
        m[y0:y0 + h, x0:x0 + w, ch] = 0
    if inv:
        m = 255 - m
    mask = np.ascontiguousarray(m[..., 0]) if C == 1 else m
    g = HW.cells(mask, inv, R)
    wins = HW.windows(g, H, W, R)
    assert len(wins) >= 2 and (0, 0, H, W) not in wins
    ys = [(rng.standard_normal((3,) + F.extent(h, w, R)) * 0.8).astype(np.float32) for _, _, h, w in wins]
    xs, out = run_windows(emul, img, mask, inv, wins, ys, R)
    for k, win in enumerate(wins):
        want_x = F.preprocess(HW.crop(img, win), HW.crop(mask, win), inv, R)[0].numpy()
        assert np.array_equal(xs[k], want_x), win
    want = HW.compose(img, mask, wins, lambda k, ci, cm: F.postprocess(torch.from_numpy(ys[k]), ci, cm, inv))
    assert np.array_equal(out, want)
    inside = np.zeros((H, W), bool)
    for y0, x0, h, w in wins:
        inside[y0:y0 + h, x0:x0 + w] = True
    assert np.array_equal(out[~inside], img[~inside])


def test_whole_photo_window_pads_like_fullres(emul):
    """A window that is the whole photo at a side that is not a valid size is reflect-padded as the full-resolution path
    pads the photo; a window of a valid size is not padded."""
    rng = np.random.default_rng(7)
    R, H, W = 64, 70, 90
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    mask = _mask(rng, H, W, 2, 0.1)
    for win in [(0, 0, H, W), (6, 10, 64, 80)]:
        y = (rng.standard_normal((3,) + F.extent(win[2], win[3], R))).astype(np.float32)
        xs, out = run_windows(emul, img, mask, False, [win], [y], R)
        assert xs[0].shape[1:] == F.extent(win[2], win[3], R)
        assert np.array_equal(xs[0], F.preprocess(HW.crop(img, win), HW.crop(mask, win), False, R)[0].numpy())
        want = HW.compose(img, mask, [win], lambda k, ci, cm: F.postprocess(torch.from_numpy(y), ci, cm, False))
        assert np.array_equal(out, want)


def test_window_argument_checks(emul):
    img = np.zeros((40, 50, 3), np.uint8)
    mask = np.zeros((40, 50), np.uint8)
    x = np.zeros((4, 64, 64), np.float32)
    t = (_abi.WindowRequest * 1)()
    t[0].img, t[0].mask, t[0].H, t[0].W, t[0].mask_channels = img.ctypes.data, mask.ctypes.data, 40, 50, 1
    t[0].y0, t[0].x0, t[0].h, t[0].w = 0, 0, 40, 50
    t[0].x, t[0].Hp, t[0].Wp = x.ctypes.data, 64, 64
    assert emul.b200_window_preprocess(t, 1, None) == 0
    assert emul.b200_window_postprocess(t, 1, None) == _abi.ERR_INVALID        # no y, no output
    t[0].x0 = 1                                                                  # window past the right edge
    assert emul.b200_window_preprocess(t, 1, None) == _abi.ERR_INVALID
    t[0].x0, t[0].y0, t[0].h = 0, -1, 20
    assert emul.b200_window_preprocess(t, 1, None) == _abi.ERR_INVALID
    t[0].y0, t[0].Hp = 0, 10                                                     # extent smaller than the window
    assert emul.b200_window_preprocess(t, 1, None) == _abi.ERR_INVALID
    c = (_abi.CellsRequest * 1)()
    c[0].mask, c[0].H, c[0].W, c[0].mask_channels = mask.ctypes.data, 40, 50, 1
    assert emul.b200_hole_cells_bytes(c, 1, 64) == 3 * 4
    assert emul.b200_hole_cells_bytes(c, 1, 96) == 0                             # not a power of two
    c[0].mask_channels = 5
    assert emul.b200_hole_cells_bytes(c, 1, 64) == 0

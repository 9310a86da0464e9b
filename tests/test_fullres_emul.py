"""CPU checks of the full-resolution request path (mi-gan_b200/csrc/fullres.cu, migan_b200.fullres).

- the emulation build of fullres.cu (the same item functors, host loops) equals oracle/fullres_oracle.py (np.pad reflect +
  oracle/prepost_oracle.py) byte for byte: valid sizes, sides below R, pads longer than the side, 1-pixel sides, odd
  sizes, every mask channel count and invert;
- a mixed pass of 32 equals its requests run one at a time;
- the pass planner (grouping order, chunks, slots, passes of 32) and the extent rule of the product library."""
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
from migan_b200.fullres import Chunk, plan_passes  # noqa: E402
from oracle import fullres_oracle as F  # noqa: E402
import build_emul  # noqa: E402

NAMES = ("b200_fullres_preprocess", "b200_fullres_postprocess")
SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]

# (R, H, W, mask channels, invert)
CASES = [(256, 256, 256, 1, False), (256, 320, 448, 3, True), (256, 100, 700, 4, False), (256, 700, 90, 2, True),
         (256, 50, 600, 1, False), (256, 600, 50, 3, False), (256, 1, 300, 4, True), (256, 300, 1, 2, False),
         (256, 1, 1, 1, False), (256, 257, 511, 3, True), (512, 333, 777, 4, False), (512, 1080, 1920, 1, True),
         (64, 17, 23, 2, False), (16, 5, 7, 1, True)]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), SYMBOLS)


def _request(rng, H, W, C):
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    m = np.where(rng.random((H, W, C)) < 0.6, 255, rng.choice(np.array([0, 1, 254], np.uint8), (H, W, C))).astype(np.uint8)
    m[-max(1, H // 4):, -max(1, W // 5):] = 0       # a hole at the bottom-right border
    return img, np.ascontiguousarray(m[..., 0] if C == 1 else m)


def run(lib, reqs, R, ys=None):
    """One emulated pass over reqs = [(img, mask, invert)], each in a chunk of its own extent: (xs [4,Hp,Wp], outs)."""
    n = len(reqs)
    table = (_abi.FullResRequest * n)()
    xs, yb, outs = [], [], []
    for r, (img, mask, inv) in zip(table, reqs):
        H, W = img.shape[:2]
        Hp, Wp = F.extent(H, W, R)
        x = np.full((4, Hp, Wp), np.nan, np.float32)
        out = np.full((H, W, 3), 77, np.uint8)
        xs.append(x)
        outs.append(out)
        r.img, r.mask, r.H, r.W = img.ctypes.data, mask.ctypes.data, H, W
        r.mask_channels, r.invert = 1 if mask.ndim == 2 else mask.shape[2], int(inv)
        r.x, r.Hp, r.Wp, r.out = x.ctypes.data, Hp, Wp, out.ctypes.data
    assert lib.b200_fullres_preprocess(table, n, None) == 0
    if ys is not None:
        for r, y in zip(table, ys):
            yb.append(np.ascontiguousarray(y, np.float32))
            r.y = yb[-1].ctypes.data
        assert lib.b200_fullres_postprocess(table, n, None) == 0
    return xs, outs


def _y(rng, R, H, W):
    return (rng.standard_normal((3,) + F.extent(H, W, R)) * 0.8).astype(np.float32)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_equals_oracle(emul, case):
    R, H, W, C, inv = CASES[case]
    rng = np.random.default_rng(case)
    img, mask = _request(rng, H, W, C)
    y = _y(rng, R, H, W)
    xs, outs = run(emul, [(img, mask, inv)], R, [y])
    want_x = F.preprocess(img, mask, inv, R)[0].numpy()
    assert np.array_equal(xs[0], want_x), CASES[case]
    assert np.array_equal(outs[0], F.postprocess(torch.from_numpy(y), img, mask, inv)), CASES[case]


def test_hole_at_the_border_continues_into_the_pad(emul):
    """The known-mask is reflected with the photo: a hole on the right edge stays a hole (mask - 0.5 = -0.5, img * mask =
    0) in its mirror image inside the pad."""
    R, H, W = 256, 256, 300
    img = np.full((H, W, 3), 200, np.uint8)
    mask = np.full((H, W), 255, np.uint8)
    mask[:, -10:] = 0
    xs, _ = run(emul, [(img, mask, False)], R)
    x = xs[0]
    assert x.shape == (4, 256, 320)
    assert np.all(x[0, :, 290:300] == -0.5) and np.all(x[0, :, 300:309] == -0.5)     # 300..308 mirror 298..290
    assert np.all(x[0, :, 309:] == 0.5) and np.all(x[1:, :, 300:309] == 0)


def test_mixed_pass_of_32_equals_single_requests(emul):
    rng = np.random.default_rng(32)
    R = 64
    reqs, ys = [], []
    for k in range(32):
        H, W = int(rng.integers(1, 200)), int(rng.integers(1, 200))
        img, mask = _request(rng, H, W, int(rng.integers(1, 5)))
        reqs.append((img, mask, bool(k % 3 == 0)))
        ys.append(_y(rng, R, H, W))
    xs, outs = run(emul, reqs, R, ys)
    for k in range(32):
        x1, o1 = run(emul, [reqs[k]], R, [ys[k]])
        assert np.array_equal(xs[k], x1[0], equal_nan=True) and np.array_equal(outs[k], o1[0]), k


def test_argument_checks(emul):
    img = np.zeros((4, 4, 3), np.uint8)
    mask = np.zeros((4, 4), np.uint8)
    x = np.zeros((4, 64, 64), np.float32)
    t = (_abi.FullResRequest * 1)()
    t[0].img, t[0].mask, t[0].H, t[0].W, t[0].mask_channels = img.ctypes.data, mask.ctypes.data, 4, 4, 1
    t[0].x, t[0].Hp, t[0].Wp = x.ctypes.data, 64, 64
    assert emul.b200_fullres_preprocess(t, 1, None) == 0
    assert emul.b200_fullres_preprocess(t, 0, None) == _abi.ERR_INVALID
    assert emul.b200_fullres_postprocess(t, 1, None) == _abi.ERR_INVALID        # no y, no output
    t[0].mask_channels = 5
    assert emul.b200_fullres_preprocess(t, 1, None) == _abi.ERR_INVALID
    t[0].mask_channels, t[0].Hp = 1, 3                                           # extent smaller than the photo
    assert emul.b200_fullres_preprocess(t, 1, None) == _abi.ERR_INVALID


# ---- the pass planner -----------------------------------------------------------------------------------------------
def test_plan_groups_in_order_of_first_appearance():
    a, b, c = (512, 512), (768, 1280), (1152, 1920)
    passes = plan_passes([b, a, b, c, a, b], {a: 8, b: 8, c: 8})
    assert passes == [[Chunk(768, 1280, [0, 2, 5]), Chunk(512, 512, [1, 4]), Chunk(1152, 1920, [3])]]


def test_plan_splits_chunks_at_max_n():
    a, b = (512, 512), (3072, 4096)
    passes = plan_passes([b] * 7 + [a] * 3, {a: 128, b: 2})
    assert passes == [[Chunk(3072, 4096, [0, 1]), Chunk(3072, 4096, [2, 3]), Chunk(3072, 4096, [4, 5]),
                       Chunk(3072, 4096, [6]), Chunk(512, 512, [7, 8, 9])]]


def test_plan_passes_of_32():
    exts = [(512, 512 + 128 * (i % 3)) for i in range(70)]
    passes = plan_passes(exts, {e: 100 for e in exts})
    assert [sum(len(c.requests) for c in p) for p in passes] == [32, 32, 6]
    for k, p in enumerate(passes):
        got = sorted(i for c in p for i in c.requests)
        assert got == list(range(32 * k, min(32 * k + 32, 70)))
        for c in p:                                        # slot s of a chunk is its s-th request, all of its extent
            assert all(exts[i] == (c.Hp, c.Wp) for i in c.requests) and c.requests == sorted(c.requests)
    assert [c.requests[:2] for c in passes[0]] == [[0, 3], [1, 4], [2, 5]]


# ---- the extent rule (product library, description-only context) -----------------------------------------------------
@pytest.fixture(scope="module")
def ctx512(lib):
    h = ctypes.c_void_p()
    _abi.check(lib.migan_create(512, -1, ctypes.byref(h)))
    yield h
    lib.migan_destroy(h)


def _extent(lib, ctx, H, W):
    Hp, Wp, mx = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = lib.migan_fullres_extent(ctx, H, W, ctypes.byref(Hp), ctypes.byref(Wp), ctypes.byref(mx))
    return rc, (Hp.value, Wp.value), mx.value


@pytest.mark.parametrize("H,W,want", [(1080, 1920, (1152, 1920)), (720, 1280, (768, 1280)), (3024, 4032, (3072, 4096)),
                                      (2160, 3840, (2176, 3840)), (300, 400, (512, 512)), (1, 1, (512, 512)),
                                      (512, 640, (512, 640)), (513, 513, (640, 640))])
def test_extent_rule(lib, ctx512, H, W, want):
    rc, ext, mx = _extent(lib, ctx512, H, W)
    assert rc == 0 and ext == want
    assert ext == F.extent(H, W, 512)
    assert lib.migan_workspace_bytes_hw(ctx512, mx, *ext) > 0           # the largest batch is accepted ...
    assert lib.migan_workspace_bytes_hw(ctx512, mx + 1, *ext) == 0      # ... and one more is not


def test_extent_refuses_a_photo_too_large_for_one_forward(lib, ctx512):
    # ch(512) = 64: a padded extent of 2^31 / 64 = 2^25 pixels or more is refused; 4096 x 8192 is exactly 2^25
    assert _extent(lib, ctx512, 4096, 8191)[0] == _abi.ERR_INVALID
    msg = lib.migan_last_error().decode()
    assert "4096 x 8191" in msg and "4096 x 8192" in msg, msg
    rc, ext, mx = _extent(lib, ctx512, 4096, 8064)
    assert rc == 0 and ext == (4096, 8064) and mx == 1
    assert _extent(lib, ctx512, 0, 5)[0] == _abi.ERR_INVALID

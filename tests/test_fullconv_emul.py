"""Fully convolutional forward (any H x W that is a multiple of R/4 and at least R), checked without a GPU.

* The oracle's fully convolutional form (oracle/fullconv_oracle.py) against tests/golden/fullconv.npz, which the reference
  itself wrote with its `filter_const` / `noise_const` buffers made size-dependent (tests/golden/make_golden_fullconv.py);
  at H = W = R it equals `generator_forward` bit for bit.
* The shape rule of the C ABI (`migan_workspace_bytes_hw` on a description-only context): accepted and refused shapes,
  the nearest-valid-size message and the 2^31 element limit.
* The uint8 pre/post kernels at rectangular shapes in the emulation build, against demo.py's torch expressions.
* The UP / STEM pre-stages of the tensor-core kernel on tiles at the right / bottom edge of a rectangular image.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from migan_b200 import _abi
from oracle import fullconv_oracle as FC
from oracle import migan_oracle as O
from oracle import prepost_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import build_emul  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "fullconv.npz")
SQRT2 = np.float32(np.sqrt(2))


def _ptr(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def _cases():
    z = np.load(GOLD)
    return [i for i in range(int(z["num_cases"]))]


@pytest.mark.parametrize("case", _cases())
def test_oracle_matches_reference_fixture(case):
    z = np.load(GOLD)
    R, N, H, W, wseed, xseed = [int(v) for v in z["case%d_meta" % case]]
    sd = O.make_state_dict(R, seed=wseed)
    assert abs(sum(float(v.double().abs().sum()) for v in sd.values()) - float(z["case%d_w_checksum" % case])) < 1e-6 * float(
        z["case%d_w_checksum" % case])
    x = FC.make_input_hw(R, N, H, W, seed=xseed)
    assert abs(float(x.double().abs().sum()) - float(z["case%d_x_checksum" % case])) < 1e-6 * float(z["case%d_x_checksum" % case])
    y = FC.generator_forward_fc(sd, x, R)
    assert tuple(y.shape) == (N, 3, H, W)
    rows = torch.from_numpy(z["case%d_rows" % case])
    assert torch.equal(rows, FC.fixture_rows(H))
    assert float((y[:, :, rows] - torch.from_numpy(z["case%d_y" % case])).abs().max()) <= 1e-5


@pytest.mark.parametrize("R,n", [(64, 2), (256, 1)])
def test_oracle_at_model_resolution_is_the_fixed_forward(R, n):
    sd = O.make_state_dict(R, seed=1)
    x = O.make_input(R, n, seed=5)
    assert torch.equal(FC.generator_forward_fc(sd, x, R), O.generator_forward(sd, x, R))
    assert FC.fullconv_state_dict(sd, R, R, R).keys() == sd.keys()
    assert all(torch.equal(a, b) for a, b in zip(FC.fullconv_state_dict(sd, R, R, R).values(), sd.values()))


def test_tiled_noise_and_zero_insertion():
    nc = torch.arange(16.0).reshape(4, 4)
    t = FC.tiled_noise(nc, 5, 7)
    assert tuple(t.shape) == (5, 7)
    assert all(t[i, j] == nc[i % 4, j % 4] for i in range(5) for j in range(7))
    f = FC.zero_insertion(6, 10)[0, 0]
    assert all(f[i, j] == (1.0 if (i % 2 == 0 and j % 2 == 0) else 0.0) for i in range(6) for j in range(10))


# ---- shape rule through the C ABI ------------------------------------------------------------------------------------------
@pytest.fixture
def ctx512(lib):
    h = ctypes.c_void_p()
    _abi.check(lib.migan_create(512, -1, ctypes.byref(h)))   # description-only context: sizes, no device
    yield h
    lib.migan_destroy(h)


@pytest.mark.parametrize("n,H,W", [(1, 512, 512), (32, 512, 512), (8, 640, 896), (4, 1024, 1536), (2, 2048, 2048), (3, 768, 512),
                                   (1, 512, 3968)])
def test_accepted_shapes(lib, ctx512, n, H, W):
    nbytes = lib.migan_workspace_bytes_hw(ctx512, n, H, W)
    assert nbytes > 0, lib.migan_last_error()
    assert FC.fullconv_shape_error(512, n, H, W) is None
    if (H, W) == (512, 512):
        assert nbytes == lib.migan_workspace_bytes(ctx512, n)
    else:   # the activations scale with the area; the tiled noise planes come on top
        assert nbytes > lib.migan_workspace_bytes(ctx512, n) * (H * W) / (512 * 512)


@pytest.mark.parametrize("n,H,W,nearest", [
    (1, 640, 600, (b"640 x 512", b"640 x 640")),      # not a multiple of 128
    (1, 384, 512, (b"512 x 512", b"512 x 512")),      # below R
    (1, 700, 1000, (b"640 x 896", b"768 x 1024")),
    (1, 0, 512, (b"512 x 512", b"512 x 512")),
])
def test_refused_shapes_name_the_nearest_valid_sizes(lib, ctx512, n, H, W, nearest):
    assert lib.migan_workspace_bytes_hw(ctx512, n, H, W) == 0
    msg = lib.migan_last_error()
    assert b"multiples of 128" in msg and b"at least 512" in msg, msg
    for s in nearest:
        assert s in msg, msg
    assert FC.fullconv_shape_error(512, n, H, W) is not None


def test_element_limit(lib, ctx512):
    # 8 x 2048 x 2048 x 64 = 2^31 elements in the largest activation: one too many for 32-bit offsets
    assert 8 * 2048 * 2048 * 64 == 2 ** 31
    assert lib.migan_workspace_bytes_hw(ctx512, 8, 2048, 2048) == 0
    msg = lib.migan_last_error()
    assert b"2^31 - 1" in msg and b"largest batch is 7" in msg, msg
    assert lib.migan_workspace_bytes_hw(ctx512, 7, 2048, 2048) > 0
    assert FC.fullconv_shape_error(512, 8, 2048, 2048) is not None and FC.fullconv_shape_error(512, 7, 2048, 2048) is None
    assert lib.migan_workspace_bytes_hw(ctx512, 0, 512, 512) == 0


def test_rule_at_other_resolutions(lib):
    for R, ok, bad in [(256, [(256, 384), (320, 256), (640, 320)], [(256, 200), (192, 256)]),
                       (128, [(160, 224), (128, 128)], [(160, 100), (96, 128)])]:
        h = ctypes.c_void_p()
        _abi.check(lib.migan_create(R, -1, ctypes.byref(h)))
        try:
            for H, W in ok:
                assert lib.migan_workspace_bytes_hw(h, 1, H, W) > 0, (R, H, W)
            for H, W in bad:
                assert lib.migan_workspace_bytes_hw(h, 1, H, W) == 0, (R, H, W)
                assert ("multiples of %d" % (R // 4)).encode() in lib.migan_last_error()
        finally:
            lib.migan_destroy(h)


# ---- uint8 pre/post kernels at H x W (emulation build: the same item functors on the host) ----------------------------------
@pytest.fixture(scope="module")
def prepost():
    return _abi.bind(ctypes.CDLL(build_emul.build()), _abi.PREPOST_SYMBOLS)


@pytest.mark.parametrize("n,H,W", [(2, 48, 80), (1, 96, 40), (3, 17, 23)])
def test_prepost_u8_hw_match_demo_expressions(prepost, n, H, W):
    rng = np.random.RandomState(H * 1000 + W)
    img = np.ascontiguousarray(rng.randint(0, 256, size=(n, H, W, 3)).astype(np.uint8))
    mask = np.ascontiguousarray(rng.choice(np.array([0, 7, 254, 255, 255], np.uint8), size=(n, H, W)))
    x = np.empty((n, 4, H, W), np.float32)
    assert prepost.b200_preprocess_u8_hw(_ptr(img), _ptr(mask), _ptr(x), n, H, W, None) == 0
    assert np.array_equal(x, P.preprocess(img, mask).numpy())
    y = np.ascontiguousarray(rng.uniform(-1.3, 1.3, size=(n, 3, H, W)).astype(np.float32))
    out = np.empty((n, H, W, 3), np.uint8)
    assert prepost.b200_postprocess_u8_hw(_ptr(y), _ptr(img), _ptr(mask), _ptr(out), n, H, W, None) == 0
    assert np.array_equal(out, P.postprocess(torch.from_numpy(y), img, mask))


def test_prepost_u8_hw_at_square_equals_r_entry_points(prepost):
    rng = np.random.RandomState(3)
    n, r = 2, 32
    img = np.ascontiguousarray(rng.randint(0, 256, size=(n, r, r, 3)).astype(np.uint8))
    mask = np.ascontiguousarray(rng.choice(np.array([0, 255], np.uint8), size=(n, r, r)))
    x1, x2 = np.empty((n, 4, r, r), np.float32), np.empty((n, 4, r, r), np.float32)
    prepost.b200_preprocess_u8(_ptr(img), _ptr(mask), _ptr(x1), n, r, None)
    prepost.b200_preprocess_u8_hw(_ptr(img), _ptr(mask), _ptr(x2), n, r, r, None)
    assert np.array_equal(x1, x2)
    y = np.ascontiguousarray(rng.uniform(-1.2, 1.2, size=(n, 3, r, r)).astype(np.float32))
    o1, o2 = np.empty((n, r, r, 3), np.uint8), np.empty((n, r, r, 3), np.uint8)
    prepost.b200_postprocess_u8(_ptr(y), _ptr(img), _ptr(mask), _ptr(o1), n, r, None)
    prepost.b200_postprocess_u8_hw(_ptr(y), _ptr(img), _ptr(mask), _ptr(o2), n, r, r, None)
    assert np.array_equal(o1, o2)


# ---- UP / STEM pre-stages on an H x W image, tiles at the right / bottom edge ---------------------------------------------
@pytest.fixture(scope="module")
def stages():
    L = ctypes.CDLL(build_emul.build_harness("stages_hw_emul.cpp"))
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.emul_prestage_up_hw.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci, ci]
    L.emul_prestage_stem_hw.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci, ci]
    return L


def tma_box(t, starts, box):
    """TMA tile load emulation (out-of-bounds elements zero); starts / box innermost-first."""
    out = np.zeros(box[::-1], dtype=t.dtype)
    src, dst = [], []
    for ax in range(t.ndim):
        k = t.ndim - 1 - ax
        lo, n, size = starts[k], box[k], t.shape[ax]
        a, b = max(lo, 0), min(lo + n, size)
        if a >= b:
            return out
        src.append(slice(a, b))
        dst.append(slice(a - lo, b - lo))
    out[tuple(dst)] = t[tuple(src)]
    return out


# (H, W): 40 x 48 puts the last tile column at 32..47 (full) and the last tile row at 32..39; 36 x 52 gives partial tiles
# in both directions (the kernel's tiles are 8 x 16 with the origin on a multiple of the tile shape)
EDGE_TILES = [(40, 48, 32, 32), (40, 48, 0, 32), (36, 52, 32, 48), (36, 52, 32, 0), (36, 52, 16, 48), (36, 52, 0, 0)]


@pytest.mark.parametrize("H,W,y0,x0", EDGE_TILES)
@pytest.mark.parametrize("fir", ["constructor", "asymmetric"])
def test_prestage_up_hw_edge_tiles(stages, H, W, y0, x0, fir):
    C = 32
    g = torch.Generator().manual_seed(H + W + y0 + x0)
    t = torch.randn(1, C, H // 2, W // 2, generator=g) * 3
    skip = torch.randn(1, C, H, W, generator=g)
    noise = torch.randn(H, W, generator=g) * 0.3
    if fir == "constructor":   # symmetric: blind to flipped or transposed taps
        taps = O.setup_filter([1, 3, 3, 1], gain=4.0)
    else:                      # one asymmetric filter, as a trained checkpoint may carry
        taps = O.random_fir(1, 4.0, torch.Generator().manual_seed(11))[0, 0]
    want = O.lrelu_agc(O.upsample2d(t, taps[None, None].repeat(C, 1, 1, 1), FC.zero_insertion(H, W)) + noise) + skip
    want = F.pad(want, (1, 17, 1, 9))[0].permute(1, 2, 0).numpy()          # zero outside the image, index +1
    t_hwc = np.ascontiguousarray(t[0].permute(1, 2, 0).numpy())
    skip_hwc = np.ascontiguousarray(skip[0].permute(1, 2, 0).numpy())
    pitch = (W + 3) // 4 * 4
    nz = np.zeros((H, pitch), np.float32)
    nz[:, :W] = noise.numpy() * SQRT2
    taps16 = np.ascontiguousarray((taps.numpy().reshape(16) * SQRT2).astype(np.float32))
    in_stage = tma_box(skip_hwc, (0, x0 - 1, y0 - 1), (32, 18, 10)).copy()
    t_area = tma_box(t_hwc, (0, x0 // 2 - 1, y0 // 2 - 1), (32, 10, 6)).copy()
    nz_area = tma_box(nz[:, :W], (x0 - 4, y0 - 1), (24, 10)).copy()
    stages.emul_prestage_up_hw(_ptr(in_stage), _ptr(t_area), _ptr(nz_area), _ptr(taps16), y0, x0, H, W, 1)
    ref = want[y0:y0 + 10, x0:x0 + 18, :]
    assert np.abs(in_stage - ref).max() < 2e-5 * max(1.0, np.abs(ref).max())
    rows_out, cols_out = max(0, y0 + 9 - H), max(0, x0 + 17 - W)           # IN rows / columns at or past the edge
    if rows_out:
        assert not in_stage[10 - rows_out:].any()
    if cols_out:
        assert not in_stage[:, 18 - cols_out:].any()


@pytest.mark.parametrize("H,W,y0,x0", EDGE_TILES)
def test_prestage_stem_hw_edge_tiles(stages, H, W, y0, x0):
    C0 = 64
    g = torch.Generator().manual_seed(H * W + y0 + x0)
    x = torch.randn(1, 4, H, W, generator=g)
    w = torch.randn(C0, 4, 1, 1, generator=g)
    b = torch.randn(C0, generator=g) * 0.1
    want = O.lrelu_agc(F.conv2d(x, w, b))
    want = F.pad(want, (1, 17, 1, 9))[0].permute(1, 2, 0).numpy()
    ws = (w.numpy().reshape(C0, 4) * SQRT2).astype(np.float32)
    ws = np.ascontiguousarray(ws.reshape(C0 // 2, 2, 4).transpose(0, 2, 1))
    bs = np.ascontiguousarray((b.numpy() * SQRT2).astype(np.float32))
    xn = np.ascontiguousarray(x[0].numpy())
    for cg0 in (0, 32):
        in_stage = np.full((10, 18, 32), np.nan, np.float32)
        x_area = tma_box(xn, (x0 - 4, y0 - 1, 0), (24, 10, 4)).copy()
        stages.emul_prestage_stem_hw(_ptr(in_stage), _ptr(x_area), _ptr(ws), _ptr(bs), cg0, y0, x0, H, W)
        ref = want[y0:y0 + 10, x0:x0 + 18, cg0:cg0 + 32]
        assert np.isfinite(in_stage).all()
        assert np.abs(in_stage - ref).max() < 2e-6 * max(1.0, np.abs(ref).max())

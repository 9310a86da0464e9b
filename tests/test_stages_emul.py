"""CPU check of the shared-memory stages of the fused SeparableConv2d kernel (mi-gan_b200/csrc/sepconv_stages.cuh).

The stage functions are compiled as plain C++ (tests/emul/build_emul.py) and run over host buffers filled the way the
TMA unit fills a pipeline stage (box layout, out-of-bounds zero fill).  Checked against the oracle's torch ops:
  * UP pre-stage   == lrelu_agc(Upsample2d(t) + noise) + skip on the halo'd tile, ZERO outside the image
  * STEM pre-stage == lrelu_agc(fromrgb(x) + b) on the halo'd tile, ZERO outside the image
  * depthwise prologue -> A operand (fp16 hi/lo, SWIZZLE_128B K-major) == 64 * lrelu_agc(dw3x3(in) + b)
for tiles at every image corner / edge / interior position.  The UP pre-stage runs with the constructor's symmetric filter
and with an asymmetric one, which shows flipped or transposed taps.  No GPU involved.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import migan_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emul"))
import build_emul  # noqa: E402

SQRT2 = np.float32(np.sqrt(2))


@pytest.fixture(scope="module")
def lib():
    L = ctypes.CDLL(build_emul.build_harness("stages_emul.cpp"))
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.emul_prologue_chunk.argtypes = [ci, vp, vp, vp, vp, vp, ci, ci, ci]
    L.emul_prestage_up.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci]
    L.emul_prestage_stem.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci]
    return L


def ptr(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def tma_box(t, starts, box):
    """Emulate a TMA tile load: t is indexed [d_last]...[d0]; starts/box are given innermost-first like the tensor-map
    coordinates.  Out-of-bounds elements are zero."""
    out = np.zeros(box[::-1], dtype=t.dtype)
    rank = t.ndim
    src, dst = [], []
    for ax in range(rank):                       # ax 0 = outermost numpy axis = last TMA coordinate
        k = rank - 1 - ax
        lo, n, size = starts[k], box[k], t.shape[ax]
        a, b = max(lo, 0), min(lo + n, size)
        if a >= b:
            return out
        src.append(slice(a, b))
        dst.append(slice(a - lo, b - lo))
    out[tuple(dst)] = t[tuple(src)]
    return out


def decode_a(a_hi, a_lo):
    """A operand planes (bytes) -> float [128 rows][64 k]: (hi + lo) of the SWIZZLE_128B K-major layout."""
    hi = np.frombuffer(a_hi.tobytes(), dtype=np.float16).astype(np.float32)
    lo = np.frombuffer(a_lo.tobytes(), dtype=np.float16).astype(np.float32)
    out = np.zeros((128, 64), np.float32)
    for m in range(128):
        for j in range(8):
            off = ((m >> 3) * 1024 + (m & 7) * 128 + ((j ^ (m & 7)) << 4)) // 2   # in halves
            out[m, j * 8:(j + 1) * 8] = hi[off:off + 8] + lo[off:off + 8]
    return out


TILE_POS = [(0, 0), (0, 16), (8, 0), (24, 48), (56, 48), (56, 0), (0, 48), (16, 32)]   # R = 64: corners, edges, interior


def up_taps(fir):
    """The 4x4 up-sampling filter (gain 4) the pre-stage gets: the constructor's [1,3,3,1] (symmetric, so blind to a
    flip or a transpose) or one asymmetric filter, as a trained checkpoint may carry."""
    if fir == "constructor":
        return O.setup_filter([1, 3, 3, 1], gain=4.0)
    return O.random_fir(1, 4.0, torch.Generator().manual_seed(11))[0, 0]


@pytest.mark.parametrize("y0,x0", TILE_POS)
@pytest.mark.parametrize("has_noise", [1, 0])
@pytest.mark.parametrize("fir", ["constructor", "asymmetric"])
def test_prestage_up_matches_oracle(lib, y0, x0, has_noise, fir):
    R, C = 64, 64
    g = torch.Generator().manual_seed(7)
    t = torch.randn(1, C, R // 2, R // 2, generator=g) * 3
    skip = torch.randn(1, C, R, R, generator=g)
    noise = torch.randn(R, R, generator=g) * 0.3 if has_noise else torch.zeros(R, R)
    taps = up_taps(fir)
    fw = taps[None, None].repeat(C, 1, 1, 1)
    fconst = torch.zeros(1, 1, R, R); fconst[:, :, ::2, ::2] = 1
    want = O.lrelu_agc(O.upsample2d(t, fw, fconst) + noise) + skip            # [1, C, R, R]
    want = F.pad(want, (1, 1, 1, 1))[0].permute(1, 2, 0).numpy()              # zero halo, HWC, index +1

    t_hwc = np.ascontiguousarray(t[0].permute(1, 2, 0).numpy())
    skip_hwc = np.ascontiguousarray(skip[0].permute(1, 2, 0).numpy())
    nz = np.ascontiguousarray((noise.numpy() * SQRT2).astype(np.float32))
    taps16 = np.ascontiguousarray((taps.numpy().reshape(16) * SQRT2).astype(np.float32))
    for cg0 in (0, 32):
        in_stage = tma_box(skip_hwc, (cg0, x0 - 1, y0 - 1), (32, 18, 10)).copy()
        t_area = tma_box(t_hwc, (cg0, x0 // 2 - 1, y0 // 2 - 1), (32, 10, 6)).copy()
        nz_area = tma_box(nz, (x0 - 4, y0 - 1), (24, 10)).copy()
        lib.emul_prestage_up(ptr(in_stage), ptr(t_area), ptr(nz_area), ptr(taps16), y0, x0, R, has_noise)
        ref = want[y0:y0 + 10, x0:x0 + 18, cg0:cg0 + 32]
        err = np.abs(in_stage - ref).max()
        assert err < 2e-5 * max(1.0, np.abs(ref).max()), (y0, x0, cg0, err)
        # pixels outside the image are exactly zero (the depthwise conv's padding)
        if y0 == 0:
            assert not in_stage[0].any()
        if x0 == 0:
            assert not in_stage[:, 0].any()
        if y0 + 8 == R:
            assert not in_stage[9].any()
        if x0 + 16 == R:
            assert not in_stage[:, 17].any()


def test_prestage_up_clamps(lib):
    """Values beyond the +-256 clamp of lrelu_agc saturate before the skip is added."""
    R, C, y0, x0 = 32, 32, 8, 16
    t = torch.full((1, C, R // 2, R // 2), 500.0)
    t[:, 1::2] = -5000.0
    skip = torch.ones(1, C, R, R) * 0.5
    taps = O.setup_filter([1, 3, 3, 1], gain=4.0)
    fconst = torch.zeros(1, 1, R, R); fconst[:, :, ::2, ::2] = 1
    want = O.lrelu_agc(O.upsample2d(t, taps[None, None].repeat(C, 1, 1, 1), fconst)) + skip
    assert float(want.max()) == 256.5 and float(want.min()) == -255.5
    want = F.pad(want, (1, 1, 1, 1))[0].permute(1, 2, 0).numpy()
    t_hwc = np.ascontiguousarray(t[0].permute(1, 2, 0).numpy())
    skip_hwc = np.ascontiguousarray(skip[0].permute(1, 2, 0).numpy())
    in_stage = tma_box(skip_hwc, (0, x0 - 1, y0 - 1), (32, 18, 10)).copy()
    t_area = tma_box(t_hwc, (0, x0 // 2 - 1, y0 // 2 - 1), (32, 10, 6)).copy()
    nz_area = np.zeros((10, 24), np.float32)
    taps16 = np.ascontiguousarray((taps.numpy().reshape(16) * SQRT2).astype(np.float32))
    lib.emul_prestage_up(ptr(in_stage), ptr(t_area), ptr(nz_area), ptr(taps16), y0, x0, R, 0)
    assert np.abs(in_stage - want[y0:y0 + 10, x0:x0 + 18, :32]).max() < 1e-3
    assert in_stage.max() == 256.5 and in_stage.min() == -255.5


@pytest.mark.parametrize("y0,x0", TILE_POS)
def test_prestage_stem_matches_oracle(lib, y0, x0):
    R, C0 = 64, 64
    g = torch.Generator().manual_seed(9)
    x = torch.randn(1, 4, R, R, generator=g)
    w = torch.randn(C0, 4, 1, 1, generator=g)
    w = w / w.flatten(1).norm(dim=1).view(-1, 1, 1, 1)
    b = torch.randn(C0, generator=g) * 0.1
    want = O.lrelu_agc(F.conv2d(x, w, b))
    want = F.pad(want, (1, 1, 1, 1))[0].permute(1, 2, 0).numpy()
    ws = (w.numpy().reshape(C0, 4) * SQRT2).astype(np.float32)
    ws = np.ascontiguousarray(ws.reshape(C0 // 2, 2, 4).transpose(0, 2, 1))      # pair-interleaved [C0/2][plane][2], as the kernel stages it
    bs = np.ascontiguousarray((b.numpy() * SQRT2).astype(np.float32))
    xn = np.ascontiguousarray(x[0].numpy())                                   # [4][R][R]
    for cg0 in (0, 32):
        in_stage = np.full((10, 18, 32), np.nan, np.float32)                  # the stage is NOT pre-filled in this mode
        x_area = tma_box(xn, (x0 - 4, y0 - 1, 0), (24, 10, 4)).copy()
        lib.emul_prestage_stem(ptr(in_stage), ptr(x_area), ptr(ws), ptr(bs), cg0, y0, x0, R)
        ref = want[y0:y0 + 10, x0:x0 + 18, cg0:cg0 + 32]
        assert np.isfinite(in_stage).all()
        err = np.abs(in_stage - ref).max()
        assert err < 2e-6 * max(1.0, np.abs(ref).max()), (y0, x0, cg0, err)


@pytest.mark.parametrize("tile_w,res", [(16, 64), (8, 8), (4, 4)])
def test_depthwise_prologue_a_operand(lib, tile_w, res):
    """The depthwise stage writes 64 * lrelu_agc(dw3x3(in) + b) as fp16 hi + lo into the swizzled A operand."""
    C = 64
    tile_h = 8 if res >= 8 else res
    tile_n = 128 // (tile_w * tile_h)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(tile_n, C, res, res, generator=g) * 2
    w = torch.randn(C, 1, 3, 3, generator=g)
    w = w / w.flatten(1).norm(dim=1).view(-1, 1, 1, 1)
    b = torch.randn(C, generator=g) * 0.1
    want = O.lrelu_agc(F.conv2d(x, w, b, padding=1, groups=C)).permute(0, 2, 3, 1).numpy()   # NHWC
    S = np.float32(64.0) * SQRT2
    w9 = np.ascontiguousarray((w.numpy().reshape(C, 9).T * S).astype(np.float32))              # [9][C]
    bias = np.ascontiguousarray((b.numpy() * S).astype(np.float32))
    x_nhwc = np.ascontiguousarray(x.permute(0, 2, 3, 1).numpy())
    for (y0, x0) in [(0, 0)] + ([(res - tile_h, res - tile_w), (8, 16)] if res >= 32 else []):
        a_hi = np.zeros(128 * 64 * 2, np.uint8)
        a_lo = np.zeros(128 * 64 * 2, np.uint8)
        for gi in (0, 1):
            in_stage = tma_box(x_nhwc, (gi * 32, x0 - 1, y0 - 1, 0), (32, tile_w + 2, tile_h + 2, tile_n)).copy()
            lib.emul_prologue_chunk(tile_w, ptr(in_stage), ptr(a_hi), ptr(a_lo), ptr(w9), ptr(bias), C, gi * 32, gi)
        got = decode_a(a_hi, a_lo) / 64.0
        ref = want[:, y0:y0 + tile_h, x0:x0 + tile_w, :].reshape(128, C)
        err = np.abs(got - ref).max()
        assert err < 1e-5 * max(1.0, np.abs(ref).max()), (tile_w, y0, x0, err)

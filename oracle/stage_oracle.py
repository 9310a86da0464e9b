"""One launch of a CUDA-core stage kernel of the forward (elementwise.cu), restated on the CPU.  TEST INFRASTRUCTURE.

The kernels: `stem_fromrgb`, `dw3x3_act`, the three down-sampling forms (`dw3x3_down` fp32, `dw3x3_down_split` and
`dw3x3_down_tma`, which write the tensor-core GEMM's fp16 hi/lo operand), `up2_noise_act_skip`, `torgb_img`, `noise_tile`
and `add_inplace`.  Two references per launch (DESIGN.md section 4.2):

* `stage_op`     the operation in float64, built from the `migan_oracle` ops (Downsample2d, Upsample2d, lrelu_agc, the
                 torgb 1x1), in activation units.  The kernel must stay within the contract bound of it.
* `stage_model`  the kernel's fp32 chain in float64 on the tables the loader packs (fp32), with a per-element bound
                 c * 2^-24 * M: M is the float64 sum of magnitudes along the chain, c the count of roundings on it (the
                 depthwise FFMAs from the bias, the 0.2 v multiply, the gain, the FIR / up-sampling FFMAs, the noise and
                 skip adds, the torgb dot product and its shuffle reduction).  The activation is 1-Lipschitz in the
                 tensor-core feed's scaled units and sqrt 2-Lipschitz in activation units.  A split output adds the fp16
                 rounding of lo, 2^-11 ulp(hi).

Bitwise properties where the arithmetic allows them: the split forms' hi is the fp16 nearest to hi + lo; the DW split
output is numpy's split of its own fp32 output * 64; `noise_tile` is numpy's tiling; `add_inplace` one fp32 add.

`CASES` is the shape matrix the GPU test runs (tests/test_stages_gpu.py) and `make_case` its seeded operands; the CPU
tests (tests/test_stage_oracle.py) pin the references to the generator oracle and check the matrix against what
production forwards launch.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import migan_oracle as O

STEM, DW, DOWN, UP2, TORGB, NOISE_TILE, ADD = range(7)
KIND_NAMES = {STEM: "stem", DW: "dw", DOWN: "down", UP2: "up2", TORGB: "torgb", NOISE_TILE: "noise_tile", ADD: "add"}
AUTO, F32, SPLIT, TMA = -1, 0, 1, 2
FORM_NAMES = {F32: "f32", SPLIT: "split", TMA: "tma"}
U = 2.0 ** -24
SPLIT_SCALE = 64.0
F32_SQRT2 = np.float32(1.41421356237309515)
F32_ALPHA = float(np.float32(0.2))
LIM = 256.0
# contract bounds: max |kernel - float64 op| / max(|op|max, 1), per kernel; about 3x the largest value measured on the
# H100 (DESIGN.md section 4.2).  The saturation cases set dw's and up2's: pre-activation sums of 1e4 and more carry fp32
# rounding of that size into outputs clamped at 256.
OP_BOUND = {"stem": 2e-6, "dw": 1e-5, "down_f32": 1e-6, "down_split": 1e-6, "down_tma": 1e-6, "up2": 1.2e-4, "torgb": 4e-7}
LOBES = torch.tensor([-1.0, 2.0, 2.0, -1.0]) / 2          # outer(LOBES, LOBES): sum |f| = 9


@dataclass
class Case:
    kind: int
    n: int
    h: int                        # the kernel's input extent (UP2: the low-resolution side; NOISE_TILE: the tiled plane)
    w: int
    c: int = 4
    form: int = F32               # DOWN: F32 / SPLIT / TMA; DW: F32 (fp32 out) or SPLIT (fp32 and hi/lo out)
    noise: bool = False           # UP2
    skip: bool = False            # UP2
    img_lo: bool = False          # TORGB
    fir: str = "random"           # DOWN / UP2: "constructor", "uniform", "random" (per channel), "lobes"
    sat: bool = False             # inputs scaled until the clamp and the negative lrelu branch are both hit
    r: int = 0                    # NOISE_TILE: side of the source plane
    seed: int = 0
    t: dict = field(default_factory=dict, repr=False)

    @property
    def name(self):
        """The kernel's row in the report."""
        return KIND_NAMES[self.kind] + ("_" + FORM_NAMES[self.form] if self.kind == DOWN else "")

    @property
    def id(self):
        s = "%s-n%d-%dx%d-c%d" % (self.name, self.n, self.h, self.w, self.c)
        if self.kind == DW and self.form == SPLIT:
            s += "-split"
        for flag in ("noise", "skip", "img_lo", "sat"):
            if getattr(self, flag):
                s += "-" + flag
        if self.kind in (DOWN, UP2):
            s += "-fir" + self.fir
        if self.kind == NOISE_TILE:
            s = "noise_tile-r%d-%dx%d" % (self.r, self.h, self.w)
        return s

    @property
    def noise_pitch(self):
        w = 2 * self.w if self.kind == UP2 else self.w
        return (w + 3) // 4 * 4 + (4 if self.kind == UP2 else 0)   # UP2: a padded row, as the sepconv matrix does

    @property
    def rs(self):
        """Rows per thread of the DW / DOWN kernels."""
        rows = self.h // 2 if self.kind == DOWN else self.h
        return 8 if rows >= 8 else 4

    def out_shape(self):
        n, h, w, c = self.n, self.h, self.w, self.c
        return {STEM: (n, h, w, c), DW: (n, h, w, c), DOWN: (n, h // 2, w // 2, c), UP2: (n, 2 * h, 2 * w, c),
                TORGB: (n, 3, h, w), NOISE_TILE: (h, self.noise_pitch), ADD: (n, h, w, c)}[self.kind]


def _matrix():
    c = []
    # stem: C0 = 64 .. 512
    c += [Case(STEM, 1, 8, 12, 64), Case(STEM, 2, 16, 16, 128), Case(STEM, 1, 8, 12, 256), Case(STEM, 1, 16, 16, 512),
          Case(STEM, 1, 8, 12, 64, sat=True)]
    # dw3x3: RS 4 and 8, odd W, H not a multiple of RS; 512 channels with the split output too
    c += [Case(DW, 1, 5, 7, 64), Case(DW, 2, 13, 9, 64), Case(DW, 1, 4, 4, 512), Case(DW, 3, 6, 5, 512, SPLIT),
          Case(DW, 2, 12, 9, 512, SPLIT), Case(DW, 1, 12, 9, 512, SPLIT, sat=True)]
    # down split: C = 512; RS 4 (H2 = 4, 5) and 8 (H2 = 12); odd and even W2; n = 1, 3
    c += [Case(DOWN, 1, 8, 10, 512, SPLIT), Case(DOWN, 3, 10, 12, 512, SPLIT), Case(DOWN, 1, 24, 10, 512, SPLIT),
          Case(DOWN, 3, 24, 16, 512, SPLIT), Case(DOWN, 1, 24, 16, 512, SPLIT, sat=True),
          Case(DOWN, 2, 24, 16, 512, SPLIT, fir="lobes", sat=True)]
    # down TMA: RS 8; C = 64 .. 512 (1, 2, 4, 8 slabs); W2 = 16, 24, 40 (a partial 16-column tile); H2 = 16, 20
    for ch in (64, 128, 256, 512):
        c += [Case(DOWN, 1, 32, 32, ch, TMA), Case(DOWN, 3, 40, 48, ch, TMA), Case(DOWN, 1, 40, 80, ch, TMA)]
    c += [Case(DOWN, 1, 32, 48, 64, TMA, sat=True), Case(DOWN, 2, 32, 32, 128, TMA, fir="lobes", sat=True),
          Case(DOWN, 1, 32, 32, 512, TMA, fir="constructor")]
    # down fp32 (CUDA-core path): RS 4 and 8, odd W2, C = 64 and 512
    c += [Case(DOWN, 1, 8, 10, 64), Case(DOWN, 2, 24, 14, 64), Case(DOWN, 1, 12, 10, 512), Case(DOWN, 2, 24, 18, 512),
          Case(DOWN, 1, 24, 18, 64, sat=True)]
    # up2: C = 64 .. 512; 4x4, 5x7, 8x12; noise and skip on / off; channel-uniform and per-channel taps
    c += [Case(UP2, 1, 4, 4, 512, noise=True, skip=True, fir="uniform"), Case(UP2, 2, 5, 7, 256, noise=True),
          Case(UP2, 1, 8, 12, 64, skip=True), Case(UP2, 3, 8, 12, 128, noise=True, skip=True, fir="uniform"),
          Case(UP2, 1, 4, 4, 512, fir="constructor"), Case(UP2, 1, 5, 7, 64, noise=True, skip=True, sat=True)]
    # torgb: G = 16 (C = 64) and 32 (C = 128, 512); img_lo on / off; pixel counts that leave a warp partly idle
    c += [Case(TORGB, 3, 5, 7, 64), Case(TORGB, 1, 6, 10, 64, img_lo=True), Case(TORGB, 2, 8, 8, 128),
          Case(TORGB, 1, 6, 10, 512, img_lo=True), Case(TORGB, 3, 4, 4, 512, img_lo=True)]
    # noise_tile and add: planes r does not divide; odd tails
    c += [Case(NOISE_TILE, 1, 20, 28, r=16), Case(NOISE_TILE, 1, 5, 7, r=4), Case(NOISE_TILE, 1, 40, 24, r=32)]
    c += [Case(ADD, 1, 5, 7, 64), Case(ADD, 3, 3, 5, 4), Case(ADD, 2, 20, 28, 128)]
    for i, case in enumerate(c):
        case.seed = 2000 + i
    return c


CASES = _matrix()


def _fir(kind_gain, mode, c, g):
    if mode == "constructor":
        f = O.setup_filter([1, 3, 3, 1], gain=kind_gain)
        return f.expand(c, 1, 4, 4).contiguous()
    if mode == "lobes":
        return torch.outer(LOBES, LOBES).expand(c, 1, 4, 4).contiguous()
    f = O.random_fir(1 if mode == "uniform" else c, kind_gain, g)
    return f.expand(c, 1, 4, 4).contiguous()


def _signs(h, w):
    """+-1 with period 4 along both axes: the sign pattern of outer(LOBES, LOBES) at every other output."""
    s = torch.tensor([1.0, 1.0, -1.0, -1.0])
    return s[torch.arange(h) % 4][:, None] * s[torch.arange(w) % 4][None, :]


def make_case(case: Case) -> Case:
    """Seeded operands of `case`: CPU float32 tensors in the layouts the hook takes (migan_stage_io)."""
    if case.t:
        return case
    g = torch.Generator().manual_seed(case.seed)
    n, h, w, c = case.n, case.h, case.w, case.c
    t = case.t
    big = 3000.0 if case.sat else 1.0
    if case.kind == STEM:
        t["in"] = (torch.rand(n, 4, h, w, generator=g) * 2 - 1) * big
        t["fromrgb_w"] = torch.randn(c, 4, generator=g) / 2
        t["fromrgb_b"] = 0.1 * torch.randn(c, generator=g)
    elif case.kind in (DW, DOWN):
        t["in"] = torch.randn(n, h, w, c, generator=g) * big
        t["dw_w"] = torch.randn(c, 1, 3, 3, generator=g) / 3
        t["dw_b"] = 0.1 * torch.randn(c, generator=g)
        if case.kind == DOWN:
            t["fir"] = _fir(1.0, case.fir, c, g)
            if case.fir == "lobes":
                # identity depthwise taps and inputs far past the clamp in the filter's sign pattern: every other output is
                # 9 * 256 * 64 in the tensor-core feed's units, past fp16's 65504 unless the taps are scaled down
                t["dw_w"] = torch.zeros(c, 1, 3, 3)
                t["dw_w"][:, 0, 1, 1] = 1.0
                t["dw_b"] = torch.zeros(c)
                t["in"] = (_signs(h, w)[None, :, :, None] * 1e5).expand(n, h, w, c).contiguous()
    elif case.kind == UP2:
        t["in"] = torch.randn(n, h, w, c, generator=g) * (300.0 * big if case.sat else 1.0)
        t["fir"] = _fir(4.0, case.fir, c, g)
        if case.noise:
            t["noise"] = torch.randn(2 * h, case.noise_pitch, generator=g)
        if case.skip:
            t["skip"] = torch.randn(n, 2 * h, 2 * w, c, generator=g)
    elif case.kind == TORGB:
        t["in"] = torch.randn(n, h, w, c, generator=g)
        t["rgb_w"] = torch.randn(3, c, generator=g) / np.sqrt(c)
        t["rgb_b"] = 0.1 * torch.randn(3, generator=g)
        t["fir"] = O.random_fir(3, 4.0, g)
        if case.img_lo:
            t["img_lo"] = torch.randn(n, 3, h // 2, w // 2, generator=g)
    elif case.kind == NOISE_TILE:
        t["in"] = torch.randn(case.r, case.r, generator=g)
    else:
        t["in"] = torch.randn(n, h, w, c, generator=g)
        t["out"] = torch.randn(n, h, w, c, generator=g)
    return case


def _d(x):
    return torch.as_tensor(np.asarray(x)).to(torch.float64) if not isinstance(x, torch.Tensor) else x.to(torch.float64)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _zero_insertion(h, w):
    fc = torch.zeros(1, 1, h, w, dtype=torch.float64)
    fc[..., ::2, ::2] = 1.0
    return fc


def fir_shift(fir) -> int:
    """m of the loader's pack_down_fir: the least m >= 0 with max_c sum_t |f[c][t]| * 2^-m <= 2."""
    s = float(np.abs(np.asarray(fir, dtype=np.float64)).reshape(-1, 16).sum(1).max())
    m = 0
    while m < 64 and s * 2.0 ** -m > 2.0:
        m += 1
    return m


def out_scale(case: Case) -> float:
    """Activation units -> the split output's units (64 * 2^-m)."""
    return SPLIT_SCALE * 2.0 ** -fir_shift(make_case(case).t["fir"]) if case.kind == DOWN else SPLIT_SCALE


def stage_op(case: Case):
    """The operation in float64, in the kernel's output layout and activation units."""
    t = make_case(case).t
    if case.kind == STEM:
        return _nhwc(O.lrelu_agc(F.conv2d(_d(t["in"]), _d(t["fromrgb_w"])[:, :, None, None], _d(t["fromrgb_b"]))))
    if case.kind in (DW, DOWN):
        a = O.lrelu_agc(F.conv2d(_nchw(_d(t["in"])), _d(t["dw_w"]), _d(t["dw_b"]), padding=1, groups=case.c))
        return _nhwc(a if case.kind == DW else O.downsample2d(a, _d(t["fir"])))
    if case.kind == UP2:
        x = O.upsample2d(_nchw(_d(t["in"])), _d(t["fir"]), _zero_insertion(2 * case.h, 2 * case.w))
        if case.noise:
            x = x + _d(t["noise"])[: 2 * case.h, : 2 * case.w]
        x = O.lrelu_agc(x)
        if case.skip:
            x = x + _nchw(_d(t["skip"]))
        return _nhwc(x)
    if case.kind == TORGB:
        img = F.conv2d(_nchw(_d(t["in"])), _d(t["rgb_w"])[:, :, None, None], _d(t["rgb_b"]))
        if case.img_lo:
            img = img + O.upsample2d(_d(t["img_lo"]), _d(t["fir"]), _zero_insertion(case.h, case.w))
        return img
    if case.kind == NOISE_TILE:
        return tile_noise(case).astype(np.float64)
    return _d(t["out"]) + _d(t["in"])


def tile_noise(case: Case):
    """noise_tile's plane: the r x r plane tiled over h x w, rows noise_pitch floats apart, padding columns zero."""
    src = make_case(case).t["in"].numpy()
    out = np.zeros((case.h, case.noise_pitch), np.float32)
    out[:, : case.w] = np.tile(src, (case.h // case.r + 1, case.w // case.r + 1))[: case.h, : case.w]
    return out


VARIANTS = ("drop_lo", "fir_flip", "fir_transpose", "dw_transpose", "clamp_256", "row_shift", "noise_pitch_w")


def variant_applies(case: Case, v: str) -> bool:
    split = case.kind == DOWN and case.form != F32
    return {"drop_lo": split,
            "fir_flip": case.kind in (DOWN, UP2) and case.fir not in ("constructor", "lobes"),
            "fir_transpose": case.kind in (DOWN, UP2) and case.fir not in ("constructor", "lobes"),
            "dw_transpose": case.kind in (DW, DOWN) and case.fir != "lobes",
            "clamp_256": split and case.sat,
            "row_shift": case.kind in (DW, DOWN) and case.out_shape()[1] > 8,
            "noise_pitch_w": case.kind == UP2 and case.noise}[v]


def _act(v, lim, gain=1.0):
    """max(v, 0.2 v) * gain, clamped: lrelu_agc (gain sqrt 2, lim 256) or the tensor-core feed's form (gain folded into
    the taps, lim 256 * 64)."""
    a = torch.maximum(v, F32_ALPHA * v)
    return torch.clamp(a * gain if gain != 1.0 else a, -lim, lim)


def stage_model(case: Case, variant: Optional[str] = None):
    """The kernel's fp32 chain in float64 on the packed tables: {"out": values in the output's units (split forms: the
    value hi + lo carries), "bound": c * 2^-24 * M (+ the lo rounding)}.  variant: the model of a subtly wrong kernel."""
    t = make_case(case).t
    f32 = np.float32
    gain = float(F32_SQRT2)
    if case.kind == STEM:
        x, wt, b = _d(t["in"]), _d(t["fromrgb_w"]), _d(t["fromrgb_b"])
        v = F.conv2d(x, wt[:, :, None, None], b)
        mag = F.conv2d(x.abs(), wt.abs()[:, :, None, None], b.abs())
        return {"out": _nhwc(_act(v, LIM, gain)), "bound": _nhwc(7 * U * gain * mag)}
    if case.kind in (DW, DOWN):
        split = case.kind == DOWN and case.form != F32
        dw = t["dw_w"].numpy()
        if variant == "dw_transpose":
            dw = dw.transpose(0, 1, 3, 2)
        if split:   # pack_dw_tc: taps and bias * (64 * sqrt 2) in fp32
            S = f32(64.0) * F32_SQRT2
            w9, b9 = _d(dw * S), _d(t["dw_b"].numpy() * S)
            g_act, lim = 1.0, LIM * SPLIT_SCALE
        else:
            w9, b9 = _d(dw), _d(t["dw_b"])
            g_act, lim = gain, LIM
        if variant == "clamp_256":
            lim = LIM
        x = _nchw(_d(t["in"]))
        v = F.conv2d(x, w9, b9, padding=1, groups=case.c)
        mag = g_act * F.conv2d(x.abs(), w9.abs(), b9.abs(), padding=1, groups=case.c)
        a = _act(v, lim, g_act)
        if case.kind == DW:
            out, bound = a, 11 * U * mag
        else:
            fir = t["fir"].numpy()
            if split:
                fir = np.ldexp(fir, -fir_shift(fir)).astype(f32)
            fir = _d(fir)
            if variant == "fir_flip":
                fir = fir.flip([2, 3])
            if variant == "fir_transpose":
                fir = fir.transpose(2, 3)
            out = O.downsample2d(a, fir)
            bound = (27 if not split else 26) * U * O.downsample2d(mag, fir.abs())
        out, bound = _nhwc(out), _nhwc(bound)
        if variant == "row_shift":
            out = out.clone()
            out[:, 8] = out[:, 7]
        if split:
            hi = out.numpy().astype(np.float32).astype(np.float16).astype(np.float64)
            ulp = np.spacing(np.abs(hi).astype(np.float16)).astype(np.float64)
            bound = bound + 2.0 ** -11 * torch.from_numpy(ulp) + 2.0 ** -25
            if variant == "drop_lo":
                out = torch.from_numpy(hi)
        return {"out": out, "bound": bound}
    if case.kind == UP2:
        fir = _d(t["fir"])
        if variant == "fir_flip":
            fir = fir.flip([2, 3])
        if variant == "fir_transpose":
            fir = fir.transpose(2, 3)
        fc = _zero_insertion(2 * case.h, 2 * case.w)
        x = _nchw(_d(t["in"]))
        acc = O.upsample2d(x, fir, fc)
        mag = O.upsample2d(x.abs(), fir.abs(), fc)
        if case.noise:
            p = _d(t["noise"])
            nz = (p.reshape(-1)[: 4 * case.h * case.w].reshape(2 * case.h, 2 * case.w) if variant == "noise_pitch_w"
                  else p[: 2 * case.h, : 2 * case.w])
            acc, mag = acc + nz, mag + nz.abs()
        out, mag = _act(acc, LIM, gain), gain * mag
        if case.skip:
            sk = _nchw(_d(t["skip"]))
            out, mag = out + sk, mag + sk.abs() + out.abs()
        return {"out": _nhwc(out), "bound": _nhwc(8 * U * mag)}
    if case.kind == TORGB:
        G = 32 if case.c // 4 >= 32 else 16
        x, wt, b = _nchw(_d(t["in"])), _d(t["rgb_w"]), _d(t["rgb_b"])
        img = F.conv2d(x, wt[:, :, None, None], b)
        mag = F.conv2d(x.abs(), wt.abs()[:, :, None, None], b.abs())
        if case.img_lo:
            fc = _zero_insertion(case.h, case.w)
            lo, fir = _d(t["img_lo"]), _d(t["fir"])
            img = img + O.upsample2d(lo, fir, fc)
            mag = mag + O.upsample2d(lo.abs(), fir.abs(), fc)
        c_round = case.c // G + int(np.log2(G)) + 6
        return {"out": img, "bound": c_round * U * mag}
    raise ValueError("%s has a bitwise reference, not a model" % case.id)


def kernel_value(case: Case, out=None, hi=None, lo=None):
    """The kernel's result in the model's units, float64: fp32 out, or hi + lo of a split form."""
    if case.kind == DOWN and case.form != F32:
        return _d(np.asarray(hi, np.float16).astype(np.float64) + np.asarray(lo, np.float16).astype(np.float64))
    return _d(out)


def model_ratio(case: Case, got, model=None) -> float:
    """max |kernel - model| / bound (NaN -> inf)."""
    m = model or stage_model(case)
    q = (_d(got) - m["out"]).abs() / m["bound"].clamp_min(1e-30)
    q = torch.where(torch.isnan(q), torch.full_like(q, float("inf")), q)
    return float(q.max())


def op_error(case: Case, got) -> float:
    """max |kernel - float64 op| / max(|op|max, 1), in activation units (split forms: (hi + lo) / (64 * 2^-m))."""
    want = stage_op(case)
    v = _d(got)
    if case.kind == DOWN and case.form != F32:
        v = v / out_scale(case)
    return float((v - want).abs().max() / max(float(want.abs().max()), 1.0))


def split_is_nearest(hi, lo) -> bool:
    """hi is the fp16 nearest to hi + lo: |lo| <= ulp(hi) / 2 (ties excepted at exactly half)."""
    hi = np.asarray(hi, np.float16)
    lo64 = np.asarray(lo, np.float16).astype(np.float64)
    half = np.spacing(np.abs(hi)).astype(np.float64) / 2
    # below fp16's smallest normal the spacing of hi is that of the subnormals, which the rounding of s used too
    return bool(np.all(np.abs(lo64) <= half))


def split_f16(v, scale):
    """split_f16 of common.cuh in numpy: s = v * scale (fp32), hi = fp16(s), lo = fp16(s - hi)."""
    s = (np.asarray(v, np.float32) * np.float32(scale)).astype(np.float32)
    hi = s.astype(np.float16)
    lo = (s - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def saturation(case: Case):
    """(clamp hit, negative lrelu branch hit) of the float64 operation's activation."""
    t = make_case(case).t
    if case.kind == STEM:
        pre = F.conv2d(_d(t["in"]), _d(t["fromrgb_w"])[:, :, None, None], _d(t["fromrgb_b"]))
    elif case.kind in (DW, DOWN):
        pre = F.conv2d(_nchw(_d(t["in"])), _d(t["dw_w"]), _d(t["dw_b"]), padding=1, groups=case.c)
    elif case.kind == UP2:
        pre = O.upsample2d(_nchw(_d(t["in"])), _d(t["fir"]), _zero_insertion(2 * case.h, 2 * case.w))
    else:
        return False, False
    act = O.lrelu_agc(pre)
    return bool((act.abs() == LIM).any()), bool(((pre < 0) & (act.abs() < LIM)).any())

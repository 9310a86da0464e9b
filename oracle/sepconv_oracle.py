"""One launch of the tensor-core SeparableConv2d kernel (`sepconv_tc_kernel`), restated on the CPU.  TEST INFRASTRUCTURE.

Two references for the same operation (DESIGN.md section 3):

* `sepconv_op`     the operation in float64, built from the `migan_oracle` pieces: the prologue's source (NHWC tensor,
                   up-sampled low-resolution tensor + noise + skip, fromrgb stem, or a pre-split operand), depthwise 3x3
                   + bias + lrelu_agc, the 1x1 conv, the epilogue (noise, activation) and the optional fused torgb +
                   image up-sampling.  The kernel must stay within the float64 contract bound of it.
* `sepconv_model`  the arithmetic the kernel claims to perform, exactly: the activation A = 64 sqrt2 (depthwise + bias)
                   after lrelu and the +-256 * 64 clamp, split by truncation into fp16 hi / lo; the weights B = w * 2^k2
                   split by rounding (k2 as the weight loader picks it); the fp16 products summed in float64
                   (Ah Bh + Ah Bl + Al Bh for 3 passes, Ah Bh for 1).  It also returns a per-element error bound:
                   c * 2^-22 * sum_k |A_k| |B_k| (fp32 accumulation; the tensor core truncates on accumulate), plus the
                   fp32 rounding of the prologue and the epilogue, which the model does not reproduce bit for bit.  At 1
                   pass the fp16 hi of an activation depends on the last bit of the kernel's fp32 depthwise sum, so an
                   element within fp32 rounding of a truncation boundary may fall either way; the bound allows both.

`CASES` is the shape matrix the GPU test runs (tests/test_sepconv_tc_gpu.py) and `make_case` its seeded operands; the
CPU tests (tests/test_sepconv_oracle.py) check the references and the matrix's schedule coverage on the same cases.
"""
from __future__ import annotations

from dataclasses import dataclass, field
import numpy as np
import torch
import torch.nn.functional as F

from oracle import migan_oracle as O

NHWC, SPLIT, UP, STEM = 0, 1, 2, 3
SOURCE_NAMES = {NHWC: "nhwc", SPLIT: "split", UP: "up", STEM: "stem"}
SPLIT_SCALE = 64.0                               # kActSplitScale: activations * 64 before the fp16 split
F32_SQRT2 = np.float32(1.41421356237309515)      # the sqrt 2 the packing multiplies by (fp32)
# c of the model bound c * 2^-22 * sum |A||B|; measured and recorded in DESIGN.md section 3
MODEL_C = 12.0
# contract bounds: max |kernel - float64 op| / max(|op|max, 1), by passes; measured and recorded in DESIGN.md section 3
OP_BOUND = {3: 2e-5, 1: 2e-2}


def split_trunc(s):
    """Prologue split (sepconv_stages.cuh split_pack2): hi = s with the low 13 mantissa bits cleared, lo = fp16(s - hi).
    hi is exact in fp16 for 2^-14 <= |s| <= 16384; below, it rounds to the fp16 subnormal grid as the kernel's conversion
    does (lo is still taken from the fp32 hi)."""
    s = np.asarray(s).astype(np.float32)
    hi32 = (s.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    hi = hi32.astype(np.float16)
    lo = (s - hi32).astype(np.float16)
    return hi, lo


def split_round(s):
    """Weight split (migan_abi.cu pack_pw_split): hi = fp16(s), lo = fp16(s - hi)."""
    s = np.asarray(s).astype(np.float32)
    hi = s.astype(np.float16)
    lo = (s - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def weight_k2(w) -> int:
    """The power-of-two weight scale of pack_pw_split: max |w 2^k2| in [8192, 16384), k2 in [-14, 24]."""
    w = np.asarray(w, dtype=np.float32)
    m = float(np.abs(w[np.isfinite(w)]).max()) if w.size else 0.0
    k2 = int(np.floor(np.log2(16384.0 / m))) if m > 0 else 0
    return max(-14, min(24, k2))


# --------------------------------------------------------------------------------------------------------------- #
# One launch's operands
# --------------------------------------------------------------------------------------------------------------- #
@dataclass
class Case:
    source: int
    n: int
    h: int
    w: int
    cin: int
    cout: int
    passes: int = 3
    act: int = 1
    noise: bool = False           # epilogue noise plane
    up_noise: bool = False        # UP: prologue noise plane
    torgb: bool = False
    img_lo: bool = False
    store_out: int = 1
    fir: str = "constructor"      # UP: "constructor" ([1,3,3,1]) or "random" (asymmetric, channel-uniform)
    seed: int = 0
    t: dict = field(default_factory=dict, repr=False)   # tensors, filled by make_case

    @property
    def id(self):
        s = "%s-n%d-%dx%d-%d-%d-p%d" % (SOURCE_NAMES[self.source], self.n, self.h, self.w, self.cin, self.cout, self.passes)
        for flag in ("noise", "up_noise", "torgb", "img_lo"):
            if getattr(self, flag):
                s += "-" + flag
        if not self.store_out:
            s += "-nostore"
        if self.fir != "constructor":
            s += "-fir" + self.fir
        return s

    @property
    def noise_pitch(self):
        return (self.w + 3) // 4 * 4 + 4           # padded rows, as the workspace's noise planes (>= w, 16-byte rows)


def _matrix():
    c = []
    for p in (3, 1):
        c += [Case(NHWC, 1, 4, 4, 512, 512, p), Case(NHWC, 3, 5, 7, 512, 512, p, noise=True),
              Case(NHWC, 2, 9, 13, 64, 64, p), Case(NHWC, 4, 32, 32, 256, 512, p),
              Case(NHWC, 2, 40, 56, 128, 128, p, noise=True, torgb=True, img_lo=True),
              Case(NHWC, 1, 64, 96, 256, 256, p, torgb=True),
              Case(UP, 2, 16, 16, 256, 256, p, noise=True, up_noise=True, torgb=True, img_lo=True),
              Case(UP, 1, 40, 56, 128, 128, p, fir="random"),
              Case(UP, 3, 32, 48, 64, 64, p, up_noise=True),
              Case(STEM, 2, 16, 16, 64, 64, p), Case(STEM, 2, 16, 16, 128, 128, p), Case(STEM, 1, 64, 96, 64, 64, p),
              Case(SPLIT, 2, 8, 8, 512, 512, p), Case(SPLIT, 1, 10, 14, 512, 512, p),
              Case(SPLIT, 4, 64, 64, 256, 512, p), Case(SPLIT, 1, 128, 256, 64, 128, p)]
        # added for schedule coverage: the widest stationary group, torgb with nothing stored, a raw (act = 0) output
        c += [Case(NHWC, 4, 64, 64, 128, 512, p),
              Case(NHWC, 3, 24, 40, 64, 128, p, noise=True, torgb=True, img_lo=True, store_out=0),
              Case(NHWC, 5, 6, 6, 128, 256, p, act=0)]
    for i, case in enumerate(c):
        case.seed = 1000 + i
        if case.passes == 1 and case.cout > 128:
            # one pass at cout 256: a resident A next to 128-channel B stages does not fit, so torgb is not fused there
            case.torgb = case.img_lo = False
    return c


CASES = _matrix()


def _wide_range_pw(g, cout, cin):
    """Pointwise weights whose per-output-channel scales span 1e-3 .. 1, with three channels 30x larger: those set k2,
    and their outputs saturate the epilogue's +-256 clamp."""
    w = torch.randn(cout, cin, generator=g, dtype=torch.float64) / np.sqrt(cin)
    scale = torch.logspace(-3, 0, cout, dtype=torch.float64)[torch.randperm(cout, generator=g)]
    scale[torch.randperm(cout, generator=g)[:3]] = 30.0
    return (w * scale[:, None]).float()


def _activations(g, shape, big_dim):
    """randn values with a few channels (dimension big_dim) scaled by 300: the depthwise sums there saturate the prologue's
    +-256 clamp."""
    x = torch.randn(shape, generator=g)
    idx = torch.randperm(shape[big_dim], generator=g)[:3]
    x.index_fill_(big_dim, idx, 0.0)
    sel = [slice(None)] * len(shape)
    sel[big_dim] = idx
    x[tuple(sel)] = torch.randn(x[tuple(sel)].shape, generator=g) * 300.0
    return x


def make_case(case: Case) -> Case:
    """Seeded operands of `case`: CPU float32 tensors in the reference layouts (SPLIT: fp16 hi / lo numpy arrays).
    Noise planes are [h + 2][noise_pitch]: the padding columns and the rows past h hold values the kernel must not read."""
    if case.t:
        return case
    g = torch.Generator().manual_seed(case.seed)
    n, h, w, cin, cout = case.n, case.h, case.w, case.cin, case.cout
    t = case.t
    if case.source == NHWC:
        t["in"] = _activations(g, (n, h, w, cin), 3)
    elif case.source == UP:
        t["in"] = torch.randn(n, h, w, cin, generator=g)                     # the skip tensor
        t["up_t"] = _activations(g, (n, h // 2, w // 2, cin), 3)
        f = O.setup_filter([1, 3, 3, 1], gain=4) if case.fir == "constructor" else O.random_fir(1, 4.0, g)[0, 0]
        t["up_fir"] = f.reshape(4, 4).contiguous()
        if case.up_noise:
            t["up_noise"] = torch.randn(h + 2, case.noise_pitch, generator=g)
    elif case.source == STEM:
        t["x"] = torch.rand(n, 4, h, w, generator=g) * 2 - 1
        t["fromrgb_w"] = _activations(g, (cin, 4), 0) / 2            # a few channels saturate the stem's clamp
        t["fromrgb_b"] = 0.1 * torch.randn(cin, generator=g)
    else:
        a = _activations(g, (n, h, w, cin), 3).clamp(-256, 256)          # post-activation range
        t["a_hi"], t["a_lo"] = split_trunc((a * SPLIT_SCALE).numpy())
    if case.source != SPLIT:
        t["dw_w"] = torch.randn(cin, 1, 3, 3, generator=g) / 3
        t["dw_b"] = 0.1 * torch.randn(cin, generator=g)
    t["pw_w"] = _wide_range_pw(g, cout, cin)
    if case.noise:
        t["noise"] = torch.randn(h + 2, case.noise_pitch, generator=g)
    if case.torgb:
        t["rgb_w"] = torch.randn(3, cout, generator=g) / np.sqrt(cout)
        t["rgb_b"] = 0.1 * torch.randn(3, generator=g)
        t["rgb_fir"] = O.random_fir(3, 4.0, g)[:, 0].contiguous()      # [3,4,4], asymmetric, one per colour
        if case.img_lo:
            t["img_lo"] = torch.randn(n, 3, h // 2, w // 2, generator=g)
    return case


def _d(x):
    return torch.as_tensor(np.asarray(x)).to(torch.float64) if not isinstance(x, torch.Tensor) else x.to(torch.float64)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _zero_insertion(h, w):
    fc = torch.zeros(1, 1, h, w, dtype=torch.float64)
    fc[..., ::2, ::2] = 1.0
    return fc


def _plane(p, h, w, pitch_w=False):
    """Rows 0..h-1, columns 0..w-1 of a [rows][pitch] noise plane; pitch_w: read it as if its pitch were w (a bug)."""
    p = _d(p)
    return p.reshape(-1)[: h * w].reshape(h, w) if pitch_w else p[:h, :w]


def _image(case, out, rgb_w, rgb_b, fir):
    """torgb(out) + b [+ Upsample2d(img_lo)] (migan_inference.py:308-313), NCHW float64; also the magnitude sum."""
    t = case.t
    img = F.conv2d(out, rgb_w[:, :, None, None], rgb_b)
    mag = F.conv2d(out.abs(), rgb_w.abs()[:, :, None, None], rgb_b.abs())
    if case.img_lo:
        fc = _zero_insertion(case.h, case.w)
        img = img + O.upsample2d(_d(t["img_lo"]), fir[:, None], fc)
        mag = mag + O.upsample2d(_d(t["img_lo"]).abs(), fir.abs()[:, None], fc)
    return img, mag


def sepconv_op(case: Case):
    """The operation in float64: (out NHWC [n,h,w,cout], img NCHW [n,3,h,w] or None)."""
    t = make_case(case).t
    h, w, cin = case.h, case.w, case.cin
    if case.source == SPLIT:
        a = _nchw((_d(t["a_hi"]) + _d(t["a_lo"])) / SPLIT_SCALE)
    else:
        if case.source == NHWC:
            x = _nchw(_d(t["in"]))
        elif case.source == UP:
            up = O.upsample2d(_nchw(_d(t["up_t"])), _d(t["up_fir"]).expand(cin, 1, 4, 4), _zero_insertion(h, w))
            if case.up_noise:
                up = up + _plane(t["up_noise"], h, w)
            x = O.lrelu_agc(up) + _nchw(_d(t["in"]))
        else:
            x = O.lrelu_agc(F.conv2d(_d(t["x"]), _d(t["fromrgb_w"])[:, :, None, None], _d(t["fromrgb_b"])))
        a = O.lrelu_agc(F.conv2d(x, _d(t["dw_w"]), _d(t["dw_b"]), padding=1, groups=cin))
    y = F.conv2d(a, _d(t["pw_w"])[:, :, None, None])
    if case.noise:
        y = y + _plane(t["noise"], h, w)
    out = O.lrelu_agc(y) if case.act else y
    img = _image(case, out, _d(t["rgb_w"]), _d(t["rgb_b"]), _d(t["rgb_fir"]))[0] if case.torgb else None
    return out.permute(0, 2, 3, 1), img


VARIANTS = ("drop_corr", "dw_transpose", "k2_off", "noise_pitch_w", "rgb_swap", "fir_unflipped")


def variant_applies(case: Case, variant: str) -> bool:
    """Whether `variant` (a wrong kernel, see sepconv_model) is distinguishable in principle on `case`."""
    return {"drop_corr": case.passes == 3,
            "dw_transpose": case.source != SPLIT,
            "k2_off": True,
            "noise_pitch_w": (case.noise or case.up_noise) and case.noise_pitch != case.w,
            "rgb_swap": case.torgb,
            "fir_unflipped": case.torgb and case.img_lo}[variant]


def _act(v, lim):
    return torch.clamp(torch.maximum(v, 0.2 * v), -lim, lim)


def _trunc_hi(s):
    return split_trunc(s.numpy().astype(np.float32))[0].astype(np.float64)


def sepconv_model(case: Case, variant: Optional[str] = None, c: float = MODEL_C):
    """The kernel's arithmetic, exactly (module docstring).  Returns {"out", "bound"} (NHWC [n,h,w,cout]) and, with
    torgb, {"img", "img_bound"} (NCHW): |kernel - model| <= bound element by element.

    variant: the model of a subtly wrong kernel -- "drop_corr" drops Al Bh, "dw_transpose" transposes the depthwise taps,
    "k2_off" undoes 2^(k2 - 1) instead of 2^k2, "noise_pitch_w" reads the noise planes at pitch w, "rgb_swap" swaps the
    first two torgb colours, "fir_unflipped" applies the image FIR without the flip of a convolution."""
    t = make_case(case).t
    f32 = np.float32
    n, h, w, cin, cout = case.n, case.h, case.w, case.cin, case.cout
    pitch_w = variant == "noise_pitch_w"
    if case.source == SPLIT:
        ah, al = _d(t["a_hi"]).reshape(-1, cin), _d(t["a_lo"]).reshape(-1, cin)
        d_a = torch.zeros_like(ah)
        d_ah = torch.zeros_like(ah)
    else:
        # the prologue's tables, packed as pack_dw_tc / scale_sqrt2 do (fp32)
        S = f32(64.0) * F32_SQRT2
        dw = t["dw_w"].numpy()
        if variant == "dw_transpose":
            dw = dw.transpose(0, 1, 3, 2)
        w9, b9 = _d(dw * S), _d(t["dw_b"].numpy() * S)
        if case.source == NHWC:
            x = _nchw(_d(t["in"]))
            xmag = torch.zeros_like(x)
        elif case.source == UP:
            f2 = _d(t["up_fir"].numpy() * F32_SQRT2).expand(cin, 1, 4, 4)
            fc = _zero_insertion(h, w)
            tt = _nchw(_d(t["up_t"]))
            acc = O.upsample2d(tt, f2, fc)
            xmag = O.upsample2d(tt.abs(), f2.abs(), fc)
            if case.up_noise:
                nz = _plane(_d(t["up_noise"].numpy() * F32_SQRT2), h, w, pitch_w)
                acc, xmag = acc + nz, xmag + nz.abs()
            skip = _nchw(_d(t["in"]))
            x = _act(acc, 256.0) + skip
            xmag = xmag + skip.abs()
        else:
            sw, sb = _d(t["fromrgb_w"].numpy() * F32_SQRT2), _d(t["fromrgb_b"].numpy() * F32_SQRT2)
            xx = _d(t["x"])
            x = _act(F.conv2d(xx, sw[:, :, None, None], sb), 256.0)
            xmag = F.conv2d(xx.abs(), sw.abs()[:, :, None, None], sb.abs())
        v = F.conv2d(x, w9, b9, padding=1, groups=cin)
        # fp32 rounding of the prologue (pre-stage + 10-term FMA chain): a generous 16 ulp of the magnitude sum
        delta = 2.0 ** -20 * F.conv2d(x.abs() + xmag, w9.abs(), b9.abs(), padding=1, groups=cin)
        lim = 256.0 * SPLIT_SCALE
        s = _act(v, lim)
        hi, lo = split_trunc(s.permute(0, 2, 3, 1).numpy())
        ah, al = _d(hi).reshape(-1, cin), _d(lo).reshape(-1, cin)
        dl = delta.permute(0, 2, 3, 1).reshape(-1, cin)
        # 3 passes: hi + lo follows the fp32 sum, and lo's rounding may differ by one of its ulps (<= 2^-21 |s|)
        d_a = dl + 2.0 ** -21 * (ah + al).abs()
        # 1 pass: hi may be the truncation of any value within delta of s
        s_up = _act(v + delta, lim).permute(0, 2, 3, 1)
        s_dn = _act(v - delta, lim).permute(0, 2, 3, 1)
        d_ah = torch.maximum((_d(_trunc_hi(s_up)).reshape(-1, cin) - ah).abs(),
                             (_d(_trunc_hi(s_dn)).reshape(-1, cin) - ah).abs())
    # the weights, packed as pack_pw_split does
    pw = t["pw_w"].numpy().astype(f32)
    k2 = weight_k2(pw)
    wscale = f32(2.0 ** k2)
    bh, bl = split_round(pw * wscale)
    bh, bl = _d(bh), _d(bl)
    inv = float(f32(1.0) / (wscale * f32(64.0)))
    if variant == "k2_off":
        inv *= 2.0
    acc = ah @ bh.T
    if case.passes == 3:
        acc = acc + ah @ bl.T
        if variant != "drop_corr":
            acc = acc + al @ bh.T
        abs_a, abs_b = ah.abs() + al.abs(), bh.abs() + bl.abs()
        bound = c * 2.0 ** -22 * (abs_a @ abs_b.T) + d_a @ abs_b.T
    else:
        bound = c * 2.0 ** -22 * (ah.abs() @ bh.abs().T) + d_ah @ bh.abs().T
    vo = (acc * inv).reshape(n, h, w, cout)
    bound = (bound * inv).reshape(n, h, w, cout)
    nz = _plane(t["noise"], h, w, pitch_w)[None, :, :, None] if case.noise else torch.zeros(1, 1, 1, 1, dtype=torch.float64)
    if case.act:
        out = _act((vo + nz) * O.SQRT2, 256.0)
        gain = O.SQRT2
    else:
        out, gain = vo + nz, 1.0
    bound = gain * (bound + 2.0 ** -22 * (vo.abs() + nz.abs()))
    res = {"out": out, "bound": bound}
    if case.torgb:
        rgb_w, rgb_b, fir = _d(t["rgb_w"]), _d(t["rgb_b"]), _d(t["rgb_fir"])
        if variant == "rgb_swap":
            rgb_w, rgb_b = rgb_w[[1, 0, 2]], rgb_b[[1, 0, 2]]
        if variant == "fir_unflipped":
            fir = fir.flip([1, 2])
        o = _nchw(out)
        img, mag = _image(case, o, rgb_w, rgb_b, fir)
        res["img"] = img
        res["img_bound"] = F.conv2d(_nchw(bound), rgb_w.abs()[:, :, None, None]) + 2.0 ** -20 * mag
    return res


def op_error(case: Case, out, img=None):
    """max |kernel - float64 op| / max(|op|max, 1) over the output (when stored) and the image."""
    want_out, want_img = sepconv_op(case)
    err = 0.0
    if case.store_out or not case.torgb:
        err = float((_d(out) - want_out).abs().max() / max(float(want_out.abs().max()), 1.0))
    if case.torgb:
        err = max(err, float((_d(img) - want_img).abs().max() / max(float(want_img.abs().max()), 1.0)))
    return err


def model_ratio(case: Case, out, img=None, model=None):
    """max |kernel - model| / bound over the output (when stored) and the image (NaN -> inf)."""
    m = model or sepconv_model(case)
    r = 0.0
    pairs = []
    if case.store_out or not case.torgb:
        pairs.append((_d(out), m["out"], m["bound"]))
    if case.torgb:
        pairs.append((_d(img), m["img"], m["img_bound"]))
    for got, want, bound in pairs:
        q = (got - want).abs() / bound.clamp_min(1e-30)
        q = torch.where(torch.isnan(q), torch.full_like(q, float("inf")), q)
        r = max(r, float(q.max()))
    return r

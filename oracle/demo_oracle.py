"""numpy model of the reference demo's request path (scripts/demo.py:26-66, :120-143) at any image size.

Three resamplers, each reproducing its library's uint8 arithmetic bit for bit, so tests need neither PIL nor OpenCV:

- `pil_bicubic`: Pillow's `Image.resize(..., BICUBIC)` (separable, a = -0.5, 22-bit fixed-point taps, uint8
  intermediate; the horizontal pass runs only if the width changes, the vertical only if the height does).
- `pil_nearest_index`: the source index of Pillow's NEAREST resize, which maps coordinates by accumulating the scale
  in double (`xo = s/2; xo += s` per output), not by multiplying.
- `cv_cubic`: OpenCV's scalar `cv2.resize(..., INTER_CUBIC)` path (A = -0.75 float coefficients quantised to 1/2048,
  integer horizontal pass, float vertical pass rounded half to even).

`demo_request` composes them into what demo.py saves for one photo.
"""
from __future__ import annotations

import numpy as np

PIL_BITS = 22


def resized_size(w: int, h: int, max_size: int):
    """demo.py `resize`: the (w, h) of the image after the down-scale to at most max_size (unchanged when it fits)."""
    if w > max_size or h > max_size:
        ratio = max_size / w if w > h else max_size / h
        return int(w * ratio), int(h * ratio)
    return w, h


def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def pil_coeffs(in_size: int, out_size: int):
    """(xmin [out], k [out, ksize] int32) of Pillow's bicubic table in_size -> out_size; taps past the end are 0."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    xmin = np.zeros(out_size, np.int64)
    k = np.zeros((out_size, ksize), np.int64)
    for x in range(out_size):
        center = (x + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - lo
        w = np.array([float(_bicubic((i + lo - center + 0.5) * ss)) for i in range(n)])
        tot = 0.0
        for v in w:
            tot += v
        if tot != 0.0:
            w = w / tot
        k[x, :n] = [int(-0.5 + v * (1 << PIL_BITS)) if v < 0 else int(0.5 + v * (1 << PIL_BITS)) for v in w]
        xmin[x] = lo
    return xmin, k


def _pil_pass(img: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    a = np.moveaxis(img, axis, 0).astype(np.int64)
    xmin, k = pil_coeffs(a.shape[0], out_size)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], a.shape[0] - 1)
    acc = np.full((out_size,) + a.shape[1:], 1 << (PIL_BITS - 1), np.int64)
    for t in range(k.shape[1]):
        acc += a[idx[:, t]] * k[:, t].reshape((-1,) + (1,) * (a.ndim - 1))
    acc = np.clip(acc >> PIL_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(acc, 0, axis)


def pil_bicubic(img: np.ndarray, w: int, h: int) -> np.ndarray:
    """`Image.fromarray(img).resize((w, h), BICUBIC)` for uint8 [H, W] or [H, W, C]."""
    out = img
    if w != img.shape[1]:
        out = _pil_pass(out, w, 1)
    if h != img.shape[0]:
        out = _pil_pass(out, h, 0)
    return np.ascontiguousarray(out)


def pil_nearest_index(in_size: int, out_size: int) -> np.ndarray:
    """Source index of every output of Pillow's NEAREST resize along one axis."""
    if in_size == out_size:
        return np.arange(out_size)
    s = float(in_size) / out_size
    xo = 0.0 + s * 0.5
    idx = np.empty(out_size, np.int64)
    for x in range(out_size):
        idx[x] = -1 if xo < 0.0 else int(xo)
        xo += s
    return np.clip(idx, 0, in_size - 1)


def pil_nearest(img: np.ndarray, w: int, h: int) -> np.ndarray:
    return np.ascontiguousarray(img[pil_nearest_index(img.shape[0], h)][:, pil_nearest_index(img.shape[1], w)])


def cv_coeffs(in_size: int, out_size: int):
    """(sx [out], short coefficients [out, 4]) of OpenCV's INTER_CUBIC table in_size -> out_size (scalar path)."""
    scale = 1.0 / (out_size / in_size)
    f32 = np.float32
    A = f32(-0.75)
    sx = np.empty(out_size, np.int64)
    c = np.empty((out_size, 4), np.int64)
    for d in range(out_size):
        f = f32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        x = f32(f - f32(s))
        x1 = f32(x + f32(1))
        c0 = f32(f32(f32(f32(f32(f32(A * x1) - f32(5) * A) * x1) + f32(8) * A) * x1) - f32(4) * A)
        c1 = f32(f32(f32(f32(f32(A + f32(2)) * x) - f32(A + f32(3))) * x) * x) + f32(1)
        y = f32(f32(1) - x)
        c2 = f32(f32(f32(f32(f32(A + f32(2)) * y) - f32(A + f32(3))) * y) * y) + f32(1)
        c3 = f32(f32(f32(f32(1) - c0) - c1) - c2)
        sx[d] = s
        c[d] = [int(np.rint(f32(v * f32(2048)))) for v in (c0, c1, c2, c3)]
    return sx, c


CV_LANES = 8      # int16 lanes of OpenCV's 128-bit baseline SIMD: the vertical pass's vector body steps 8 values


def cv_cubic(img: np.ndarray, w: int, h: int) -> np.ndarray:
    """`cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC)` with `cv2.setUseOptimized(False)`, uint8 [H, W, C].

    The vertical pass of a row of w*C values runs its vector body (float, ((S3 b3 + S2 b2) + S1 b1) + S0 b0, round half
    to even) on the first 8 * floor(w*C / 8) values and the scalar fixed-point tail ((sum S b + 2^21) >> 22) on the rest."""
    H, W = img.shape[:2]
    if (H, W) == (h, w):
        return img.copy()
    img3 = img.reshape(H, W, -1)
    C = img3.shape[2]
    sx, cx = cv_coeffs(W, w)
    sy, cy = cv_coeffs(H, h)
    a = img3.astype(np.int64)
    S = np.zeros((H, w, C), np.int64)
    for t in range(4):
        S += a[:, np.clip(sx - 1 + t, 0, W - 1)] * cx[:, t].reshape(1, -1, 1)
    Sf = S.astype(np.float32)
    b = (cy.astype(np.float32) * np.float32(1.0 / (2048.0 * 2048.0))).astype(np.float32)
    rows = [np.clip(sy - 1 + t, 0, H - 1) for t in range(4)]
    shape = (-1, 1, 1)
    acc = Sf[rows[3]] * b[:, 3].reshape(shape) + Sf[rows[2]] * b[:, 2].reshape(shape)
    acc = acc + Sf[rows[1]] * b[:, 1].reshape(shape)
    acc = acc + Sf[rows[0]] * b[:, 0].reshape(shape)
    vec = np.clip(np.rint(acc), 0, 255)
    tail = np.clip((sum(S[rows[t]] * cy[:, t].reshape(shape) for t in range(4)) + (1 << 21)) >> 22, 0, 255)
    e = np.arange(w * C).reshape(1, w, C)
    out = np.where(e < (w * C // CV_LANES) * CV_LANES, vec, tail).astype(np.uint8)
    return out.reshape((h, w) + img.shape[2:])


def mask_known(mask: np.ndarray, invert: bool) -> np.ndarray:
    """read_mask's per-pixel steps: channel selection (alpha of LA / RGBA, R of RGB, L itself), optional invert, then
    `v < 255 -> 0`.  Returns uint8 0 / 255 [H, W]."""
    if mask.ndim == 2:
        v = mask
    else:
        v = mask[..., {4: 3, 2: 1, 3: 0, 1: 0}[mask.shape[2]]]
    if invert:
        v = 255 - v
    return np.where(v == 255, 255, 0).astype(np.uint8)


def demo_sizes(W: int, H: int, Wm: int, Hm: int, res: int):
    """((w', h') of img_resized, (w, h) after the mask's first NEAREST step); ValueError where demo.py would fail."""
    w1, h1 = resized_size(W, H, res)
    wa, ha = resized_size(Wm, Hm, 512)
    wb, hb = resized_size(wa, ha, res)
    if min(w1, h1, wa, ha, wb, hb) < 1:
        raise ValueError("a resized side is 0: photo %dx%d, mask %dx%d at %d" % (W, H, Wm, Hm, res))
    if (wb, hb) != (w1, h1):
        raise ValueError("mask resizes to %dx%d, photo to %dx%d" % (wb, hb, w1, h1))
    return (w1, h1), (wa, ha)


def demo_pre(img: np.ndarray, mask: np.ndarray, invert: bool, res: int):
    """(img_resized u8 [h',w',3], mask_resized u8 [h',w'] 0/255, x f32 [4, res, res])."""
    H, W = img.shape[:2]
    (w1, h1), (wa, ha) = demo_sizes(W, H, mask.shape[1], mask.shape[0], res)
    rs = pil_bicubic(img, w1, h1) if (w1, h1) != (W, H) else img
    m = pil_nearest(pil_nearest(mask_known(mask, invert), wa, ha), w1, h1)
    sq = pil_bicubic(rs, res, res)
    mq = (pil_nearest(m, res, res) // 255).astype(np.float32)[None]
    v = np.transpose(sq, (2, 0, 1)).astype(np.float32) * np.float32(2) / np.float32(255) - np.float32(1)
    x = np.concatenate([mq - np.float32(0.5), v * mq], axis=0).astype(np.float32)
    return rs, m, x


def demo_post(y: np.ndarray, img_resized: np.ndarray, mask_resized: np.ndarray) -> np.ndarray:
    """y f32 [3, res, res] -> the composed uint8 [h', w', 3] demo.py saves."""
    t = np.clip(y.astype(np.float32) * np.float32(0.5) + np.float32(0.5), 0, 1) * np.float32(255)
    r = np.transpose(t.astype(np.uint8), (1, 2, 0))
    h1, w1 = img_resized.shape[:2]
    r = cv_cubic(np.ascontiguousarray(r), w1, h1)
    m = (mask_resized // 255)[..., None]
    return img_resized * m + r * (1 - m)

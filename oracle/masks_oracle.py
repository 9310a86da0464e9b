"""CPU oracle of the evaluation protocol's free-form masks (`RandomMask(s)` of scripts/generate_masks.py, which
scripts/evaluate_fid_lpips.py's `InferenceDataset` also calls), stated with numpy alone.

One result of `RandomMask(s)` is the first *attempt* whose hole count lies in (0, s^2).  An attempt's draws do not depend
on any earlier result, so the legacy numpy stream is a fixed sequence of attempts:

* rectangles: `randint(10)` of side up to s // 2, then `randint(5)` of side up to s; each is w, h, x, y (4 draws) and
  clears rows [max(y, 0), min(y + h, s)) x columns [max(x, 0), min(x + w, s));
* brush tries (`randint(20)`), each: the vertex count, two angle bounds, one angle per vertex, the first vertex, one
  normal radius per further vertex, the width, then two `random()` draws whose flips are thrown away.  The try draws a
  polyline of that width (the union of its two-point wide lines) and a disc of radius width // 2 at every vertex;
* two `random()` draws flip the brush layer (rows, then columns); the rectangles are never flipped;
* the mask is 255 where no rectangle and no brush pixel covers it, else 0.

`plan_attempt` makes those draws on a `np.random.RandomState`; `raster` paints an attempt with integer and float32
arithmetic that states Pillow's wide-line polygon rule and ellipse stamps (`quad`, `polygon_row_spans`, `DISC_HALF`);
`raster_pillow` paints it with Pillow's ImageDraw where that is installed.  The CUDA planner and rasterizer
(mi-gan_b200/csrc/masks.cu) implement the same statements.
"""
from __future__ import annotations

import hashlib
import math
from typing import List, NamedTuple, Tuple

import numpy as np

f32 = np.float32

# Half-width of Pillow's ellipse((x - r, y - r, x + r, y + r)) on row y + dy: DISC_HALF[r - 6][|dy|], for r = 6..23.
DISC_HALF = [
    [6, 6, 6, 5, 4, 3, 2],
    [7, 7, 7, 6, 6, 5, 4, 2],
    [8, 8, 8, 7, 7, 6, 5, 4, 2],
    [9, 9, 9, 8, 8, 7, 7, 6, 4, 2],
    [10, 10, 10, 10, 9, 9, 8, 7, 6, 5, 3],
    [11, 11, 11, 11, 10, 10, 9, 8, 8, 6, 5, 3],
    [12, 12, 12, 12, 11, 11, 10, 10, 9, 8, 7, 5, 3],
    [13, 13, 13, 13, 12, 12, 12, 11, 10, 9, 8, 7, 6, 3],
    [14, 14, 14, 14, 13, 13, 13, 12, 11, 11, 10, 9, 7, 6, 3],
    [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3],
    [16, 16, 16, 16, 15, 15, 15, 14, 14, 13, 12, 12, 11, 9, 8, 6, 3],
    [17, 17, 17, 17, 17, 16, 16, 15, 15, 14, 14, 13, 12, 11, 10, 8, 6, 4],
    [18, 18, 18, 18, 18, 17, 17, 17, 16, 16, 15, 14, 13, 12, 11, 10, 9, 7, 4],
    [19, 19, 19, 19, 19, 18, 18, 18, 17, 17, 16, 15, 15, 14, 13, 12, 10, 9, 7, 4],
    [20, 20, 20, 20, 20, 19, 19, 19, 18, 18, 17, 17, 16, 15, 14, 13, 12, 11, 9, 7, 4],
    [21, 21, 21, 21, 21, 20, 20, 20, 19, 19, 18, 18, 17, 16, 16, 15, 14, 12, 11, 9, 7, 4],
    [22, 22, 22, 22, 22, 21, 21, 21, 20, 20, 20, 19, 18, 18, 17, 16, 15, 14, 13, 11, 10, 7, 4],
    [23, 23, 23, 23, 23, 22, 22, 22, 22, 21, 21, 20, 20, 19, 18, 17, 17, 16, 14, 13, 12, 10, 8, 4],
]
DISC_R_MIN, DISC_R_MAX = 6, 23


class Attempt(NamedTuple):
    rects: List[Tuple[int, int, int, int]]              # (y0, y1, x0, x1), clipped to the canvas; may be empty
    segments: List[Tuple[int, int, int, int, int]]      # (x0, y0, x1, y1, width)
    discs: List[Tuple[int, int, int]]                   # (x, y, r)
    flip_rows: bool
    flip_cols: bool


def plan_attempt(rs: np.random.RandomState, s: int) -> Attempt:
    """The draws of one attempt of RandomMask(s) (hole_range [0, 1]) on `rs`, in the reference's order."""
    rects = []
    for tries, size in ((10, s // 2), (5, s)):
        for _ in range(rs.randint(tries)):
            w, h = rs.randint(size), rs.randint(size)
            x, y = rs.randint(-(w // 2), s - w + w // 2), rs.randint(-(h // 2), s - h + h // 2)
            rects.append((max(y, 0), min(y + h, s), max(x, 0), min(x + w, s)))
    mean, spread = 2 * math.pi / 5, 2 * math.pi / 15
    radius = math.sqrt(s * s + s * s) / 8
    segments, discs = [], []
    for _ in range(rs.randint(20)):
        nv = rs.randint(4, 18)
        lo = mean - rs.uniform(0, spread)
        hi = mean + rs.uniform(0, spread)
        angles = [2 * math.pi - rs.uniform(lo, hi) if i % 2 == 0 else rs.uniform(lo, hi) for i in range(nv)]
        pts = [(int(rs.randint(0, s)), int(rs.randint(0, s)))]
        for i in range(nv):
            r = np.clip(rs.normal(loc=radius, scale=radius // 2), 0, 2 * radius)
            x = np.clip(pts[-1][0] + r * math.cos(angles[i]), 0, s)
            y = np.clip(pts[-1][1] + r * math.sin(angles[i]), 0, s)
            pts.append((int(x), int(y)))
        width = int(rs.uniform(12, 48))
        segments += [(pts[i][0], pts[i][1], pts[i + 1][0], pts[i + 1][1], width) for i in range(nv)]
        discs += [(x, y, width // 2) for x, y in pts]
        rs.random_sample()                               # the try's two discarded flips
        rs.random_sample()
    flip_rows = rs.random_sample() > 0.5
    flip_cols = rs.random_sample() > 0.5
    return Attempt(rects, segments, discs, bool(flip_rows), bool(flip_cols))


# ---- Pillow's wide line: a quad filled by its polygon scanline rule ------------------------------------------------

def _ru_d(f: float) -> int:                              # round half up / down of a double
    return int(math.floor(f + 0.5)) if f >= 0 else -int(math.floor(abs(f) + 0.5))


def _rd_d(f: float) -> int:
    return int(math.ceil(f - 0.5)) if f >= 0 else -int(math.ceil(abs(f) - 0.5))


def _ru_f(f) -> int:                                     # the same of a float32: + 0.5 rounded to float32 when f >= 0
    return int(math.floor(f32(f) + f32(0.5))) if f >= 0 else -int(math.floor(abs(float(f)) + 0.5))


def _rd_f(f) -> int:
    return int(math.ceil(f32(f) - f32(0.5))) if f >= 0 else -int(math.ceil(abs(float(f)) - 0.5))


def quad(x0: int, y0: int, x1: int, y1: int, width: int):
    """The four vertices of Pillow's wide line from (x0, y0) to (x1, y1); None for a zero-length line (one pixel)."""
    dx, dy = x1 - x0, y1 - y0
    if dx == 0 and dy == 0:
        return None
    big = math.hypot(dx, dy)
    small = (width - 1) / 2.0
    rmax, rmin = _ru_d(small) / big, _rd_d(small) / big
    dxmin, dxmax, dymin, dymax = _rd_d(rmin * dy), _rd_d(rmax * dy), _rd_d(rmin * dx), _rd_d(rmax * dx)
    return [(x0 - dxmin, y0 + dymax), (x1 - dxmin, y1 + dymax), (x1 + dxmax, y1 - dymin), (x0 + dxmax, y0 - dymin)]


class _Edge(NamedTuple):
    x0: int
    y0: int
    xmin: int
    xmax: int
    ymin: int
    ymax: int
    dx: np.float32


def _edges(v):
    out = []
    for i in range(len(v)):
        (xa, ya), (xb, yb) = v[i], v[(i + 1) % len(v)]
        dx = f32(0) if ya == yb else f32(f32(xb - xa) / f32(yb - ya))
        out.append(_Edge(xa, ya, min(xa, xb), max(xa, xb), min(ya, yb), max(ya, yb), dx))
    return out


def _edge_x(e: _Edge, y: int):
    return f32(f32(f32(y - e.y0) * e.dx) + f32(e.x0))


def polygon_row_spans(v, s: int):
    """{row: [(a, b), ...]} inclusive column spans (before clipping) Pillow's polygon fill paints for vertices `v` on a
    canvas of s x s."""
    edges = _edges(v)
    rows = {}
    ymin = min([s - 1] + [e.ymin for e in edges])
    ymax = max([0] + [e.ymax for e in edges])
    table = []
    for e in edges:
        if e.ymin == e.ymax:                             # horizontal: drawn as a line, not scanned
            rows.setdefault(e.ymin, []).append((e.xmin, e.xmax))
        else:
            table.append(e)
    ymin, ymax = max(ymin, 0), min(ymax, s)
    for y in range(ymin, ymax + 1):
        xx = [f32(0)] * (2 * len(table))
        j = 0
        for i, e in enumerate(table):
            if not (e.ymin <= y <= e.ymax):
                continue
            xx[j] = _edge_x(e, y)
            j += 1
            if y == e.ymax and y < ymax:                 # an edge's last row: listed twice
                xx[j] = xx[j - 1]
                j += 1
            elif e.dx != 0 and j % 2 == 1 and math.floor(xx[j - 1]) == xx[j - 1]:
                for k in range(i):                       # a corner with an earlier edge of the same slope sign
                    o = table[k]
                    if (e.dx > 0 and o.dx <= 0) or (e.dx < 0 and o.dx >= 0):
                        continue
                    if xx[j - 1] == _edge_x(o, y):
                        off = -1 if y == ymax else 1
                        a, b = _edge_x(e, y + off), _edge_x(o, y + off)
                        if y == e.ymax:
                            xx[k] = f32(max(a, b) + 1) if e.dx > 0 else f32(min(a, b) - 1)
                        else:
                            xx[k] = f32(min(a, b)) if e.dx > 0 else f32(max(a, b) + 1)
                        break
        xs = sorted(xx[:j])
        for i in range(1, j, 2):
            rows.setdefault(y, []).append((_ru_f(xs[i - 1]), _rd_f(xs[i])))
    return rows


def _paint_spans(layer: np.ndarray, rows) -> None:
    s = layer.shape[0]
    for y, spans in rows.items():
        if 0 <= y < s:
            for a, b in spans:
                a, b = max(a, 0), min(b, s - 1)
                if a <= b:
                    layer[y, a:b + 1] = 1


def segment_layer(x0, y0, x1, y1, width, s: int) -> np.ndarray:
    """uint8 [s, s]: 1 where Pillow's two-point wide line paints."""
    layer = np.zeros((s, s), np.uint8)
    v = quad(x0, y0, x1, y1, width)
    if v is None:
        _paint_spans(layer, {y0: [(x0, x0)]})
    else:
        _paint_spans(layer, polygon_row_spans(v, s))
    return layer


def disc_spans(x: int, y: int, r: int):
    t = DISC_HALF[r - DISC_R_MIN]
    return {y + dy: [(x - t[abs(dy)], x + t[abs(dy)])] for dy in range(-r, r + 1)}


def brush_layer(a: Attempt, s: int) -> np.ndarray:
    """The attempt's brush layer, un-flipped: 1 where a segment or disc paints."""
    layer = np.zeros((s, s), np.uint8)
    for x0, y0, x1, y1, w in a.segments:
        layer |= segment_layer(x0, y0, x1, y1, w, s)
    for x, y, r in a.discs:
        _paint_spans(layer, disc_spans(x, y, r))
    return layer


def compose(a: Attempt, brush: np.ndarray) -> np.ndarray:
    s = brush.shape[0]
    known = np.ones((s, s), bool)
    for y0, y1, x0, x1 in a.rects:
        known[y0:y1, x0:x1] = False
    if a.flip_rows:
        brush = brush[::-1]
    if a.flip_cols:
        brush = brush[:, ::-1]
    return np.where(known & (brush == 0), 255, 0).astype(np.uint8)


def raster(a: Attempt, s: int) -> np.ndarray:
    """uint8 [s, s] of one attempt: 255 known, 0 hole."""
    return compose(a, brush_layer(a, s))


def raster_pillow(a: Attempt, s: int) -> np.ndarray:
    """The same attempt painted by Pillow's ImageDraw (a cross-check of `raster`; needs Pillow)."""
    from PIL import Image, ImageDraw
    img = Image.new("L", (s, s), 0)
    draw = ImageDraw.Draw(img)
    for x0, y0, x1, y1, w in a.segments:
        draw.line([(x0, y0), (x1, y1)], fill=1, width=w)
    for x, y, r in a.discs:
        draw.ellipse((x - r, y - r, x + r, y + r), fill=1)
    return compose(a, np.asarray(img, np.uint8))


def accepted(m: np.ndarray) -> bool:
    holes = int((m == 0).sum())
    return 0 < holes < m.size


def random_masks(s: int, n: int, seed: int = 0, rs: np.random.RandomState = None, pillow: bool = False):
    """The next n results of RandomMask(s) on `rs` (a fresh np.random.seed(seed) stream when None): (uint8 [n, s, s],
    attempts used)."""
    rs = np.random.RandomState(seed) if rs is None else rs
    paint = raster_pillow if pillow else raster
    out, attempts = [], 0
    while len(out) < n:
        m = paint(plan_attempt(rs, s), s)
        attempts += 1
        if accepted(m):
            out.append(m)
    return np.stack(out) if out else np.zeros((0, s, s), np.uint8), attempts


def digest(m: np.ndarray) -> bytes:
    """8-byte digest of one mask's bytes (row-major uint8)."""
    return hashlib.blake2b(np.ascontiguousarray(m, np.uint8).tobytes(), digest_size=8).digest()

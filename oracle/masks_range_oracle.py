"""CPU oracle of `RandomMask(s, hole_range)` (scripts/generate_masks.py) for any hole_range, stated with numpy alone.

RandomMask(s, [lo, hi]) differs from RandomMask(s) (oracle/masks_oracle.py, hole_range [0, 1]) in two places:

* its tries: with coef = min(lo + hi, 1.0) in float64, `randint(int(10 * coef))` and `randint(int(5 * coef))`
  rectangles and `randint(int(20 * coef))` brush tries, in place of 10, 5 and 20 (so [0, 1] draws the same);
* its acceptance: hole_ratio = 1 - np.mean(mask) in float64, rejected when hole_ratio <= lo or hole_ratio >= hi.

Everything else (the draws of one rectangle or brush try, the flips, the raster) is masks_oracle's.
"""
from __future__ import annotations

import math
from typing import Sequence, Tuple

import numpy as np

from . import masks_oracle as M


def tries(hole_range: Sequence[float]) -> Tuple[int, int, int]:
    coef = min(hole_range[0] + hole_range[1], 1.0)
    return int(10 * coef), int(5 * coef), int(20 * coef)


def plan_attempt(rs: np.random.RandomState, s: int, hole_range: Sequence[float] = (0, 1)) -> M.Attempt:
    """The draws of one attempt of RandomMask(s, hole_range) on `rs`, in the reference's order."""
    n_small, n_large, n_brush = tries(hole_range)
    rects = []
    for n, size in ((n_small, s // 2), (n_large, s)):
        for _ in range(rs.randint(n)):
            w, h = rs.randint(size), rs.randint(size)
            x, y = rs.randint(-(w // 2), s - w + w // 2), rs.randint(-(h // 2), s - h + h // 2)
            rects.append((max(y, 0), min(y + h, s), max(x, 0), min(x + w, s)))
    mean, spread = 2 * math.pi / 5, 2 * math.pi / 15
    radius = math.sqrt(s * s + s * s) / 8
    segments, discs = [], []
    for _ in range(rs.randint(n_brush)):
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
    return M.Attempt(rects, segments, discs, bool(flip_rows), bool(flip_cols))


def hole_ratio(holes: int, s: int) -> float:
    """1 - np.mean(mask) of a mask with `holes` hole pixels: 1 - fl(known / s^2) in float64."""
    return 1 - float(np.mean(np.arange(s * s) >= holes))


def accepted(m: np.ndarray, hole_range: Sequence[float] = (0, 1)) -> bool:
    ratio = 1 - np.mean(m == 255)
    return not (ratio <= hole_range[0] or ratio >= hole_range[1])


def random_masks(s: int, n: int, hole_range: Sequence[float], seed: int = 0, rs: np.random.RandomState = None):
    """The next n results of RandomMask(s, hole_range) on `rs` (np.random.seed(seed) when None): (uint8 [n, s, s],
    attempts used)."""
    rs = np.random.RandomState(seed) if rs is None else rs
    out, attempts = [], 0
    while len(out) < n:
        m = M.raster(plan_attempt(rs, s, hole_range), s)
        attempts += 1
        if accepted(m, hole_range):
            out.append(m)
    return np.stack(out) if out else np.zeros((0, s, s), np.uint8), attempts

"""CPU oracle of the hole-window request path (mi-gan_b200/csrc/holewin.cu, migan_b200.HoleWindowPipeline).  TEST
INFRASTRUCTURE ONLY (same rules as oracle/migan_oracle.py).

With q = R / 4, for a photo uint8 [H,W,3] and a mask of the same H x W:

1. cells: the photo split into q x q cells from the origin (the last row / column may be partial); a cell is a hole cell
   when it holds a pixel that fullres_oracle.known_mask does not mark known.
2. windows: on each axis of side n, the cell span [c0, c1] with a margin of m cells gives
   a = max(0, (c0 - m) q), b = min(n, (c1 + 1 + m) q), L = min(n, max(R, q ceil((b - a) / q))),
   s = min(max(a - (L - (b - a)) // 2, 0), n - L) and the window [s, s + L).  The hole cells are visited in row-major order;
   each starts as its own span, and while its window overlaps (positive area) a listed window, the first such window is
   removed and the spans are united; the result is appended.  Reported sorted by (y0, x0).
3. result: the photo with every window replaced by the full-resolution path (oracle/fullres_oracle.py) on its crop.
"""
import numpy as np

from . import fullres_oracle as F


def cells(mask: np.ndarray, invert: bool, R: int) -> np.ndarray:
    """uint8 [ceil(H/q), ceil(W/q)]: 1 for a hole cell."""
    q = R // 4
    hole = F.known_mask(mask, invert) != 255
    H, W = hole.shape
    gh, gw = -(-H // q), -(-W // q)
    padded = np.zeros((gh * q, gw * q), bool)
    padded[:H, :W] = hole
    return padded.reshape(gh, q, gw, q).any(axis=(1, 3)).astype(np.uint8)


def _axis(c0: int, c1: int, n: int, R: int, m: int):
    q = R // 4
    a = max(0, (c0 - m) * q)
    b = min(n, (c1 + 1 + m) * q)
    L = min(n, max(R, q * -(-(b - a) // q)))
    s = min(max(a - (L - (b - a)) // 2, 0), n - L)
    return s, L


def windows(cell_grid: np.ndarray, H: int, W: int, R: int, margin: int = 1):
    """[(y0, x0, h, w)] of one photo from its cells."""
    def window(box):
        r0, r1, c0, c1 = box
        (y0, h), (x0, w) = _axis(r0, r1, H, R, margin), _axis(c0, c1, W, R, margin)
        return y0, x0, h, w

    def overlaps(a, b):
        return a[0] < b[0] + b[2] and b[0] < a[0] + a[2] and a[1] < b[1] + b[3] and b[1] < a[1] + a[3]

    listed = []                                   # [(box, window)]
    for cy, cx in zip(*np.nonzero(cell_grid)):    # row-major
        box = (int(cy), int(cy), int(cx), int(cx))
        while True:
            hit = next((k for k, (_, w) in enumerate(listed) if overlaps(window(box), w)), None)
            if hit is None:
                break
            other = listed.pop(hit)[0]
            box = (min(box[0], other[0]), max(box[1], other[1]), min(box[2], other[2]), max(box[3], other[3]))
        listed.append((box, window(box)))
    return sorted(w for _, w in listed)


def max_windows(H: int, W: int, R: int) -> int:
    return (H // min(R, H)) * (W // min(R, W))


def crop(a: np.ndarray, win):
    y0, x0, h, w = win
    return np.ascontiguousarray(a[y0:y0 + h, x0:x0 + w])


def compose(img: np.ndarray, mask: np.ndarray, wins, window_result) -> np.ndarray:
    """The photo with window k replaced by window_result(k, crop of the photo, crop of the mask)."""
    out = img.copy()
    for k, win in enumerate(wins):
        y0, x0, h, w = win
        out[y0:y0 + h, x0:x0 + w] = window_result(k, crop(img, win), crop(mask, win))
    return out

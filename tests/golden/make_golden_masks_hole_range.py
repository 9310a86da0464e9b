"""Fixture of RandomMask(s, hole_range) (scripts/generate_masks.py) for hole ranges other than [0, 1]:
tests/golden/masks_hole_range.npz.

    python tests/golden/make_golden_masks_hole_range.py --reference /path/to/MI-GAN checkout

Needs numpy, Pillow and a checkout of the reference: its own `RandomMask(s, hole_range)` draws every mask here after
np.random.seed(0), and each call of its `RandomBrush` is counted as one attempt (make_golden_masks.load_reference).
`ranges` float64 [k, 2] lists the hole ranges; for range i and size s:

  r{i}_{s}           s = 32: packbits of the masks (1 = known), uint8 [n, ceil(s * s / 8)]
  r{i}_{s}_digest    s = 256, 512: 8-byte blake2b digests (oracle/masks_oracle.py `digest`), uint8 [n, 8]
  r{i}_{s}_holes     the masks' hole counts, int64 [n]
  r{i}_{s}_attempts  attempts the list consumed
  r{i}_{s}_state     np.random.get_state()[1] after the list: key uint32 [624]
  r{i}_{s}_rest      the rest of that state: pos, has_gauss, gauss (float64 [3])

The ranges have coef = min(lo + hi, 1) below 1 ([0, 0.2], [0.1, 0.2], [0.2, 0.4]) and equal to 1 ([0.5, 0.6], [0.8, 1]).
`versions` records the numpy and Pillow versions that drew them.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "masks_hole_range.npz")
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

RANGES = [(0.0, 0.2), (0.1, 0.2), (0.2, 0.4), (0.5, 0.6), (0.8, 1.0)]
COUNTS = {32: 40, 256: 24, 512: 12}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference (holds scripts/generate_masks.py)")
    args = ap.parse_args()
    import PIL

    from make_golden_masks import load_reference
    from oracle import masks_oracle as M
    mod = load_reference(args.reference)
    out = {"versions": np.array(["numpy " + np.__version__, "Pillow " + PIL.__version__]),
           "ranges": np.array(RANGES, np.float64)}
    for i, hole_range in enumerate(RANGES):
        for s, n in COUNTS.items():
            np.random.seed(0)
            mod.attempts = 0
            masks = np.stack([mod.RandomMask(s, list(hole_range)) for _ in range(n)])
            st = np.random.get_state()
            assert set(np.unique(masks)) <= {0, 255}
            key = "r%d_%d" % (i, s)
            if s == 32:
                out[key] = np.packbits((masks == 255).reshape(n, -1), axis=1)
            else:
                out[key + "_digest"] = np.frombuffer(b"".join(M.digest(m) for m in masks), np.uint8).reshape(n, 8)
            out[key + "_holes"] = (masks == 0).reshape(n, -1).sum(1).astype(np.int64)
            out[key + "_attempts"] = np.int64(mod.attempts)
            out[key + "_state"] = st[1].astype(np.uint32)
            out[key + "_rest"] = np.array([st[2], st[3], st[4]], np.float64)
            print("hole_range %s s %d: %d masks, %d attempts" % (list(hole_range), s, n, mod.attempts))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

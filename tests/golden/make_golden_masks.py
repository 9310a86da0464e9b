"""Fixture of the evaluation protocol's free-form masks (RandomMask of scripts/generate_masks.py): tests/golden/masks.npz.

    python tests/golden/make_golden_masks.py --reference /path/to/MI-GAN checkout

Needs numpy, Pillow and a checkout of the reference: its own `RandomMask` draws every mask here after `np.random.seed`,
and each call of its `RandomBrush` is counted as one attempt.  Contents, for each (seed, s) list:

  m{seed}_{s}          packbits of the masks (1 = known), uint8 [n, ceil(s * s / 8)]
  m{seed}_{s}_attempts attempts the list consumed
  m{seed}_{s}_state    np.random.get_state()[1] after the list: key uint32 [624]
  m{seed}_{s}_rest     the rest of that state: pos, has_gauss, gauss (float64 [3])

and `digest0_512` / `digest0_256`: 8-byte blake2b digests (oracle/masks_oracle.py `digest`) of the first 2000 masks at 512
and 1000 at 256 for seed 0, with their attempts and final states (`..._attempts`, `..._state`, `..._rest`).  `versions` records the
numpy and Pillow versions that drew them.
"""
from __future__ import annotations

import argparse
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "masks.npz")
sys.path.insert(0, ROOT)

LISTS = [(0, 32, 200), (0, 64, 100), (0, 256, 24), (0, 512, 12), (7, 128, 40)]
DIGESTS = [(512, 2000), (256, 1000)]


def load_reference(path: str):
    spec = importlib.util.spec_from_file_location("ref_generate_masks", os.path.join(path, "scripts", "generate_masks.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    brush = mod.RandomBrush
    mod.attempts = 0

    def counted(*args, **kw):
        mod.attempts += 1
        return brush(*args, **kw)
    mod.RandomBrush = counted          # RandomMask looks the name up at call time: one call per attempt
    return mod


def draw(mod, seed: int, s: int, n: int):
    np.random.seed(seed)
    mod.attempts = 0
    masks = np.stack([mod.RandomMask(s, [0, 1]) for _ in range(n)])
    st = np.random.get_state()
    return masks, mod.attempts, st[1].astype(np.uint32), np.array([st[2], st[3], st[4]], np.float64)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference (holds scripts/generate_masks.py)")
    args = ap.parse_args()
    import PIL

    from oracle import masks_oracle as M
    mod = load_reference(args.reference)
    out = {"versions": np.array(["numpy " + np.__version__, "Pillow " + PIL.__version__])}
    for seed, s, n in LISTS:
        masks, att, key, rest = draw(mod, seed, s, n)
        assert set(np.unique(masks)) <= {0, 255}
        out["m%d_%d" % (seed, s)] = np.packbits((masks == 255).reshape(n, -1), axis=1)
        out["m%d_%d_attempts" % (seed, s)] = np.int64(att)
        out["m%d_%d_state" % (seed, s)] = key
        out["m%d_%d_rest" % (seed, s)] = rest
        print("seed %d s %d: %d masks, %d attempts" % (seed, s, n, att))
    for s, n in DIGESTS:
        masks, att, key, rest = draw(mod, 0, s, n)
        out["digest0_%d" % s] = np.frombuffer(b"".join(M.digest(m) for m in masks), np.uint8).reshape(n, 8)
        out["digest0_%d_attempts" % s] = np.int64(att)
        out["digest0_%d_state" % s] = key
        out["digest0_%d_rest" % s] = rest
        print("digests s %d: %d masks, %d attempts" % (s, n, att))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

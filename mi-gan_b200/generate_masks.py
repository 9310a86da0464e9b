"""scripts/generate_masks.py on the GPU: the same command line and the same files.

    python -m migan_b200.generate_masks --images-dir DIR --output-dir OUT --resolution 512 [--hole-range LO HI]

Every `*.jpg`, `*.jpeg` and `*.png` under DIR (recursive, lowercase suffixes, as the reference globs them) is listed in
sorted order, and path k gets the k-th result of RandomMask(resolution, hole_range) after np.random.seed(0) (hole_range
`--hole-range LO HI`, by default [0, 1] as the reference script calls it), saved as
OUT/<stem>.png through `Image.fromarray(mask).convert("L").save`.  The masks come from `RandomMaskStream` in batches;
PNG encoding runs on a host thread pool.
"""
from __future__ import annotations

import argparse
import os
from concurrent.futures import ThreadPoolExecutor
from glob import glob
from pathlib import Path
from typing import List, Optional

BATCH = 256


def image_paths(images_dir) -> List[str]:
    paths = []
    for ext in (".jpg", ".jpeg", ".png"):
        paths += glob(os.path.join(images_dir, "**", "*" + ext), recursive=True)
    return sorted(paths)


def generate(images_dir, output_dir, resolution: int, device: str = "cuda", hole_range=(0.0, 1.0)) -> int:
    """Write one mask per image path; returns the number written."""
    from PIL import Image

    from .masks import RandomMaskStream, check_hole_range

    check_hole_range(hole_range, "--hole-range")
    output_dir = Path(output_dir)
    output_dir.mkdir(exist_ok=True, parents=True)
    paths = image_paths(images_dir)
    stream = RandomMaskStream(resolution, seed=0, device=device, hole_range=hole_range)

    def save(mask, path):
        Image.fromarray(mask).convert("L").save(output_dir / ("%s.png" % Path(path).stem))

    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
        pending = []
        for b0 in range(0, len(paths), BATCH):
            batch = paths[b0:b0 + BATCH]
            masks = stream.next(len(batch)).cpu().numpy()
            for f in pending:
                f.result()
            pending = [pool.submit(save, m, p) for m, p in zip(masks, batch)]
        for f in pending:
            f.result()
    return len(paths)


def main(argv: Optional[List[str]] = None) -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--images-dir", type=Path, help="Path to original images.", required=True)
    parser.add_argument("--output-dir", type=Path, help="Masks output directory.", required=True)
    parser.add_argument("--resolution", type=int, help="Mask resolution.", required=True)
    parser.add_argument("--hole-range", type=float, nargs=2, default=(0.0, 1.0), metavar=("LO", "HI"),
                        help="RandomMask's hole_range: keep masks whose hole ratio lies strictly between LO and HI.")
    args = parser.parse_args(argv)
    generate(args.images_dir, args.output_dir, args.resolution, hole_range=tuple(args.hole_range))


if __name__ == "__main__":
    main()

"""scripts/evaluate_fid_lpips.py's protocol over another inpainting method's result files, on the GPU: the evaluation
command with a directory of results in place of the generator, on one GPU or all the GPUs of a box.

    python -m migan_b200.score_results --resolution 512 --real-dir DIR --results-dir RESULTS [--mask-dir MASKS]
    torchrun --standalone --nproc_per_node=8 -m migan_b200.score_results --resolution 512 ...

For real photo p with stem s (the sorted top-level listing of `evaluate_fid_lpips`), the method's result is
`<results-dir>/<s>.png` -- the `<stem>.png` rule of the masks, and the name `python -m migan_b200.demo` writes.  Extra
files in the results directory are ignored.  The result is decoded with `Image.open(r).convert("RGB")`, goes through PIL
BICUBIC to R x R when it is not that size, exactly as the photo does, and takes the place of the model output in
:244-249: composed = masks * imgs + (1 - masks) * result, then (v * 0.5 + 0.5).clamp(0, 1) of both.  The composite always
runs, as in the script; a result the method already composited under the same mask comes out unchanged.  Masks come
from `--mask-dir` (`<stem>.png`, 255 = known) or, without it, from the generated stream with seed 0, as in
`evaluate_fid_lpips`.

It prints `evaluate_fid_lpips`'s lines (`FID:`, `LPIPS: `, with `--ssim` `SSIM:`, with `--psnr` `PSNR:`, and with `--ids`
`P-IDS:` and `U-IDS:`, then with `--hole-bins` one `HOLE` line per bin), writes its `--per-image` CSV, and has its chunking, sharding, ordered merge and statistics files: `--save-real-stats` writes the same statistics the evaluation command
writes for the same real directory, R and batch size, and `--real-stats` reads either's.

Before any GPU work one planning pass reads the header (size and mode; no pixels) of every photo, result and mask and
raises one `demo_command.PlanError` naming every missing result, missing mask and unreadable file.
"""
from __future__ import annotations

import argparse
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, Optional, Sequence

import torch

from . import evaluate_fid_lpips as E
from .demo_command import PlanError, _header

RESOLUTIONS = (256, 512)


def list_results(images: Sequence[Path], results_dir) -> List[Path]:
    """`<results_dir>/<stem>.png` of every image, whether it exists or not (a.b.jpg -> a.b.png)."""
    return E.stem_pngs(images, results_dir)


def check_files(images: Sequence[Path], results: Sequence[Path], masks: Optional[Sequence[Path]],
                num_workers: int = 2) -> None:
    """Read the header of every photo, result and mask; raise one `PlanError` naming every missing result, missing mask
    and unreadable file."""

    def look(k: int) -> List[str]:
        problems = []
        files = [("photo", images[k]), ("result", results[k])] + ([("mask", masks[k])] if masks is not None else [])
        for what, path in files:
            if what != "photo" and not path.is_file():
                problems.append("photo %s: no %s %s" % (images[k].name, what, path))
                continue
            try:
                _header(path)
            except Exception as e:  # noqa: BLE001 -- any unreadable file is reported with the others
                problems.append("%s %s: cannot be read (%s)" % (what, path, e))
        return problems

    with ThreadPoolExecutor(max_workers=max(1, int(num_workers))) as pool:
        problems = [p for ps in pool.map(look, range(len(images))) for p in ps]
    if problems:
        raise PlanError(problems)


def score(real_dir, results_dir, mask_dir=None, *, resolution: int, device="cuda", batch_size: int = E.BATCH_SIZE,
          num_workers: int = 2, real_stats=None, save_real_stats_to=None, inception_weights=None, lpips_weights=None,
          ids: bool = False, ssim: bool = False, psnr: bool = False, per_image: bool = False,
          hole_bins: Optional[Sequence[float]] = None,
          hole_range: Sequence[float] = E.FULL_RANGE) -> Optional[E.EvalResult]:
    """FID and LPIPS of the result files in `results_dir` against the photos of `real_dir`, as the command prints them
    (`evaluate_fid_lpips.evaluate`'s `EvalResult`).  `resolution`: R, 256 or 512.  The other arguments are `evaluate`'s,
    `ssim`, `psnr`, `per_image`, `hole_bins` and `hole_range` among them.

    The argument checks and the planning pass (`PlanError`) come before any device is touched.  In an initialised
    process group rank 0 returns the result; the other ranks return None."""
    E.check_stats_args(real_stats, save_real_stats_to, ids)
    E.check_hole_args(hole_bins, hole_range, mask_dir)
    if resolution not in RESOLUTIONS:
        raise ValueError("--resolution must be one of %s, got %r" % (", ".join(map(str, RESOLUTIONS)), resolution))
    if torch.device(device).type != "cuda":
        raise RuntimeError("score_results runs on a CUDA device (there is no CPU path); got %s" % device)
    images = E.list_images(real_dir)
    results = list_results(images, results_dir)
    check_files(images, results, None if mask_dir is None else E.stem_pngs(images, mask_dir), num_workers)
    if real_stats is not None and not isinstance(real_stats, tuple):
        real_stats = E.load_real_stats(real_stats)
    setup = E.EvalSetup(None, None, real_dir, mask_dir, device=device, batch_size=batch_size, num_workers=num_workers,
                        real_features=real_stats is None, inception_weights=inception_weights,
                        lpips_weights=lpips_weights, results=results, res=resolution, ssim=ssim, psnr=psnr,
                        per_image=per_image, hole_bins=hole_bins, hole_range=hole_range)
    return E.run_setup(setup, real_stats, save_real_stats_to, ids)


def get_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m migan_b200.score_results")
    parser.add_argument("--resolution", type=int, choices=RESOLUTIONS, required=True,
                        help="R: the protocol's image size.")
    parser.add_argument("--real-dir", type=Path, required=True, help="Real dataset directory path.")
    parser.add_argument("--results-dir", type=Path, required=True,
                        help="The method's results: <stem>.png for every real photo.")
    parser.add_argument("--mask-dir", type=Path, default=None, help="Pre-generated mask directory path.")
    parser.add_argument("--device", type=str, default="cuda", help="Device to use (CUDA only).")
    parser.add_argument("--batch-size", type=int, default=E.BATCH_SIZE, help="Images per chunk (the unit of work).")
    parser.add_argument("--num-workers", type=int, default=2, help="Host decode threads.")
    parser.add_argument("--save-real-stats", type=Path, default=None, help="Write the real images' mu and sigma (.npz).")
    parser.add_argument("--real-stats", type=Path, default=None, help="Score against stored real mu and sigma (.npz).")
    parser.add_argument("--inception-weights", type=Path, default=None, help="FID Inception state_dict file.")
    parser.add_argument("--lpips-weights", type=Path, default=None, help="LPIPS (alex) state_dict file.")
    parser.add_argument("--ids", action="store_true", help="Also print P-IDS and U-IDS (Co-Mod-GAN's Inception "
                        "discriminative scores).")
    E.add_per_image_args(parser)
    return parser.parse_args(argv)


def main(argv=None) -> None:
    args = get_args(argv)
    E.check_stats_args(args.real_stats, args.save_real_stats, args.ids)
    E.check_per_image_path(args.per_image)
    hole_bins, hole_range = E.check_hole_flags(args)
    res = E.run_command(args.device, lambda device: score(
        args.real_dir, args.results_dir, args.mask_dir, resolution=args.resolution, device=device,
        batch_size=args.batch_size, num_workers=args.num_workers, real_stats=args.real_stats,
        save_real_stats_to=args.save_real_stats, inception_weights=args.inception_weights,
        lpips_weights=args.lpips_weights, ids=args.ids, ssim=args.ssim, psnr=args.psnr,
        per_image=args.per_image is not None, hole_bins=hole_bins, hole_range=hole_range), "score_results")
    E.finish_command(res, args)


if __name__ == "__main__":
    main()

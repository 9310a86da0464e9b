"""Fixture of the SSIM and PSNR evaluators: tests/golden/metrics.npz.

    python tests/golden/make_golden_metrics.py --reference /path/to/MI-GAN checkout

Needs numpy, torch and a checkout of the reference: its own `compute_ssim` (lib/evaluator/eva_ssim.py) and
`psnr_evaluator.add_batch` (lib/evaluator/eva_psnr.py) compute every value here, on the CPU.  The evaluators' base class
reaches for torch.distributed; the script stands in a world of one rank and an identity `sync_`, so no process group
is started.  Contents:

  taps{ws}                      the reference's 1-D Gaussian taps, float32 [ws], ws = 1..31
  x_{case}, y_{case}            the inputs, float32 [n, C, H, W]
  ssim_{case}_w{ws}_mean        compute_ssim(x, y, ws, size_average=True), float32 scalar
  ssim_{case}_w{ws}_img         compute_ssim(x, y, ws, size_average=False), float32 [n]
  psnr_{case}_{mode}_r{range}   add_batch's per-image PSNR of (x * range, y * range) (float32 products), case hole,
                                unrelated or same (x_hole against itself), mode none / div2k2 / bench2 / bench4
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "metrics.npz")
sys.path.insert(0, ROOT)

SSIM_WINDOWS = {"hole": (11, 8, 7, 1), "gray": (11, 8, 7, 1), "bright": (11, 8), "unrelated": (11, 7), "tiny": (11, 8)}
PSNR_MODES = {"none": (None, 2), "div2k2": ("div2k", 2), "bench2": ("benchmark", 2), "bench4": ("benchmark", 4)}


def inputs():
    from oracle import metrics_oracle as M
    a = M.images(2, 3, 40, 37, seed=1)
    cases = {
        "hole": (a, M.composed(a, seed=2)),
        "gray": (M.images(2, 1, 40, 37, seed=3), M.composed(M.images(2, 3, 40, 37, seed=3), seed=4)[:, :1].contiguous()),
        "bright": (M.bright(2, 3, 33, 29, seed=5), M.bright(2, 3, 33, 29, seed=6)),
        "unrelated": (M.images(2, 3, 40, 37, seed=7), M.images(2, 3, 40, 37, seed=8)),
        "tiny": (M.images(1, 3, 7, 5, seed=9), M.images(1, 3, 7, 5, seed=10)),
    }
    return cases


def load_reference(path: str):
    sys.path.insert(0, path)
    from lib.evaluator import eva_base, eva_psnr, eva_ssim
    eva_base.dist.get_world_size = lambda: 1
    eva_base.dist.get_rank = lambda: 0
    eva_base.base_evaluator.sync_ = lambda self, d, r: d
    return eva_ssim, eva_psnr


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference (holds lib/evaluator/)")
    args = ap.parse_args()
    eva_ssim, eva_psnr = load_reference(args.reference)
    out = {"versions": np.array(["numpy " + np.__version__, "torch " + torch.__version__])}
    for ws in range(1, 32):
        out["taps%d" % ws] = eva_ssim.gaussian(ws, 1.5).numpy()
    cases = inputs()
    for name, (x, y) in cases.items():
        out["x_" + name], out["y_" + name] = x.numpy(), y.numpy()
        for ws in SSIM_WINDOWS[name]:
            out["ssim_%s_w%d_mean" % (name, ws)] = eva_ssim.compute_ssim(x, y, window_size=ws, size_average=True).numpy()
            out["ssim_%s_w%d_img" % (name, ws)] = eva_ssim.compute_ssim(x, y, window_size=ws, size_average=False).numpy()
    for name in ("hole", "unrelated", "same"):
        x, y = cases["hole"] if name == "same" else cases[name]
        if name == "same":
            y = x.clone()
        for rgb_range in (1, 255):
            xs, ys = (x * rgb_range).numpy(), (y * rgb_range).numpy()
            for mode, (for_dataset, scale) in PSNR_MODES.items():
                ev = eva_psnr.psnr_evaluator(for_dataset=for_dataset, scale=scale, rgb_range=rgb_range)
                with np.errstate(divide="ignore"):
                    ev.add_batch(xs, ys, fn=["img%d" % i for i in range(len(xs))])
                out["psnr_%s_%s_r%d" % (name, mode, rgb_range)] = np.asarray(ev.data_psnr)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

"""Fixture of the demo request path (scripts/demo.py:26-66, :120-143) at small resolutions: tests/golden/demo.npz.

    python tests/golden/make_golden_demo.py [--reference /path/to/MI-GAN checkout]

Needs numpy, torch, Pillow and OpenCV.  With a checkout of the reference, its own `resize`, `read_mask` and `preprocess`
(scripts/demo.py) produce img_resized, mask_resized and x; without one, a transcription of those three functions does.
The generator is replaced by a seeded y, and the post-processing is demo.py:135-140 verbatim.  OpenCV runs twice: with
`cv2.setUseOptimized(False)` (the scalar path, which the GPU path reproduces bit for bit: `out`) and with its default
optimised path (`out_default`, which follows the host CPU's SIMD dispatch).  The fraction of values in which the two differ
is stored as `default_mismatch`.

Cases: photos below, at and above R on each axis, a 1 x k and a k x 1 strip, a photo and mask whose mask goes through both
NEAREST steps (R = 32), masks in L, LA, RGB and RGBA, with and without invert.
"""
from __future__ import annotations

import argparse
import importlib.util
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "demo.npz")

# (R, photo W, photo H, mask mode, invert)
CASES = [
    (32, 20, 12, "L", False),        # below R on both axes
    (32, 32, 32, "RGB", False),      # at R
    (32, 48, 30, "RGBA", True),      # above R in width
    (32, 25, 70, "LA", False),       # above R in height
    (32, 1, 20, "L", True),          # 1 x k strip
    (32, 20, 1, "RGB", False),       # k x 1 strip
    (32, 700, 300, "RGBA", False),   # mask through both NEAREST steps: 700x300 -> 512x219 -> 32x13
    (32, 300, 640, "L", True),       # 300x640 -> 240x512 -> 15x32
    (64, 64, 40, "LA", True),
    (64, 100, 64, "RGB", True),
    (64, 37, 90, "L", False),
    (64, 64, 64, "RGBA", False),
]
MODES = {"L": 1, "LA": 2, "RGB": 3, "RGBA": 4}


def case_inputs(i: int):
    """Seeded photo u8 [H,W,3], mask u8 [H,W] or [H,W,C] and y f32 [3,R,R] of case i."""
    R, W, H, mode, _ = CASES[i]
    rng = np.random.default_rng(1000 + i)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    C = MODES[mode]
    m = np.full((H, W, C), 255, np.uint8)
    for _ in range(3):                                   # rectangles of holes and of near-known values
        y0, x0 = rng.integers(0, H), rng.integers(0, W)
        y1, x1 = min(H, y0 + rng.integers(1, max(2, H // 2))), min(W, x0 + rng.integers(1, max(2, W // 2)))
        m[y0:y1, x0:x1] = rng.choice(np.array([0, 17, 254], np.uint8), size=C)
    m = np.where(rng.random((H, W, 1)) < 0.1, rng.integers(0, 256, (H, W, C), dtype=np.uint8), m)
    if mode == "L":
        m = m[..., 0]
    y = (rng.standard_normal((3, R, R)) * 0.7).astype(np.float32)
    return img, np.ascontiguousarray(m), y


def _transcribed():
    """demo.py's `resize`, `read_mask` and `preprocess`, transcribed (used when no reference checkout is given)."""
    import torch
    from PIL import Image

    def resize(image, max_size, interpolation=Image.BICUBIC):
        w, h = image.size
        if w > max_size or h > max_size:
            resize_ratio = max_size / w if w > h else max_size / h
            image = image.resize((int(w * resize_ratio), int(h * resize_ratio)), interpolation)
        return image

    def read_mask(mask_path, invert=False):
        mask = Image.open(mask_path)
        mask = resize(mask, max_size=512, interpolation=Image.NEAREST)
        mask = np.array(mask)
        if len(mask.shape) == 3:
            if mask.shape[2] == 4:
                _r, _g, _b, _a = np.rollaxis(mask, axis=-1)
                mask = np.dstack([_a, _a, _a])
            elif mask.shape[2] == 2:
                _l, _a = np.rollaxis(mask, axis=-1)
                mask = np.dstack([_a, _a, _a])
            elif mask.shape[2] == 3:
                _r, _g, _b = np.rollaxis(mask, axis=-1)
                mask = np.dstack([_r, _r, _r])
        else:
            mask = np.dstack([mask, mask, mask])
        if invert:
            mask = 255 - mask
        mask[mask < 255] = 0
        return Image.fromarray(mask).convert("L")

    def preprocess(img, mask, resolution):
        img = img.resize((resolution, resolution), Image.BICUBIC)
        mask = mask.resize((resolution, resolution), Image.NEAREST)
        img = np.array(img)
        mask = np.array(mask)[:, :, np.newaxis] // 255
        img = torch.Tensor(img).float() * 2 / 255 - 1
        mask = torch.Tensor(mask).float()
        img = img.permute(2, 0, 1).unsqueeze(0)
        mask = mask.permute(2, 0, 1).unsqueeze(0)
        return torch.cat([mask - 0.5, img * mask], dim=1)

    return resize, read_mask, preprocess


def _reference(root: str):
    """The reference's own functions from scripts/demo.py (importing it needs its `lib` package on the path)."""
    sys.path.insert(0, root)
    spec = importlib.util.spec_from_file_location("ref_demo", os.path.join(root, "scripts", "demo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.resize, mod.read_mask, mod.preprocess


def main():
    import cv2
    import torch
    from PIL import Image

    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None, help="checkout of the reference (scripts/demo.py)")
    args = ap.parse_args()
    resize, read_mask, preprocess = _reference(args.reference) if args.reference else _transcribed()
    data = {"source": np.array("reference scripts/demo.py" if args.reference else "transcription of scripts/demo.py")}
    diff = total = 0
    with tempfile.TemporaryDirectory() as tmp:
        for i, (R, W, H, mode, invert) in enumerate(CASES):
            img, mask, y = case_inputs(i)
            path = os.path.join(tmp, "mask%d.png" % i)
            Image.fromarray(mask, mode).save(path)
            assert np.array_equal(np.array(Image.open(path)), mask)
            img_resized = resize(Image.fromarray(img), max_size=R)
            mask_r = read_mask(path, invert=invert)
            mask_resized = resize(mask_r, max_size=R, interpolation=Image.NEAREST)
            x = preprocess(img_resized, mask_resized, R)
            result = (torch.from_numpy(y) * 0.5 + 0.5).clamp(0, 1) * 255
            result = result.to(torch.uint8).permute(1, 2, 0).numpy()
            outs = []
            for optimized in (False, True):
                cv2.setUseOptimized(optimized)
                r = cv2.resize(result, dsize=img_resized.size, interpolation=cv2.INTER_CUBIC)
                m = np.array(mask_resized)[:, :, np.newaxis] // 255
                outs.append(np.array(img_resized) * m + r * (1 - m))
            cv2.setUseOptimized(True)
            diff += int((outs[0] != outs[1]).sum()); total += outs[0].size
            data.update({"%d_img_resized" % i: np.array(img_resized), "%d_mask_resized" % i: np.array(mask_resized),
                         "%d_x" % i: x[0].numpy(), "%d_out" % i: outs[0], "%d_out_default" % i: outs[1]})
    data["default_mismatch"] = np.array(diff / total)
    np.savez_compressed(OUT, **data)
    print("%s: %d cases, %d bytes, OpenCV default path differs in %d of %d values" % (OUT, len(CASES), os.path.getsize(OUT), diff, total))


def load_fixture():
    return np.load(OUT)


if __name__ == "__main__":
    main()

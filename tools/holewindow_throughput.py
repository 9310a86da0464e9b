"""Throughput of hole-window inpainting (`HoleWindowPipeline`) against whole-photo inpainting (`FullResPipeline`) on
cuda:0, migan-512, on phone and camera photos with local holes:

    3024 x 4032 with one small hole          2160 x 3840 with two distant holes     1080 x 1920 with one hole
    1536 x 2048 with one hole over most of it (a whole-photo window)
    6000 x 8000 with two small holes (48 Mpx: too large for one forward, so `FullResPipeline` refuses it)

Forms, alternating over `--repeats` repeats (p50 [min, max]), on the first four photos (the mix both pipelines accept):

1. fullres   `FullResPipeline.forward_batch` on numpy photos (waits)
2. holewin   `HoleWindowPipeline.forward_batch` on numpy photos (waits)
3. async     `HoleWindowPipeline.forward_batch(..., wait=False)` on pinned tensors, then one `wait()`
4. holewin+  form 2 on all five photos

Reported per form: requests/s, generator Mpx (the padded extents the generator runs at) against photo Mpx, kernel
launches, and for `async` the host enqueue time (until `forward_batch(wait=False)` returns).  The card's name and power
limit are read in the same run.  Before timing, each window of the hole-window result is checked to be byte for byte
`FullResPipeline` on that window's crop.

    python tools/holewindow_throughput.py [--repeats 5] [--out tools/out/holewindow_throughput.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from migan_b200 import FullResPipeline, HoleWindowPipeline, synthetic  # noqa: E402

R = 512
# (H, W, holes as (y, x, h, w))
MIX = [
    (3024, 4032, [(1400, 1800, 300, 400)]),
    (2160, 3840, [(150, 200, 120, 160), (1850, 3500, 150, 200)]),
    (1080, 1920, [(500, 900, 150, 200)]),
    (1536, 2048, [(60, 80, 1400, 1880)]),
    (6000, 8000, [(1000, 1200, 200, 260), (5000, 6500, 240, 300)]),
]
COMMON = 4                      # the first photos both pipelines accept


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def fixture(rng, H, W, holes):
    """A photo and a mask (255 = known) with elliptic holes inside the given boxes."""
    img = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
    mask = np.full((H, W), 255, np.uint8)
    for y, x, h, w in holes:
        yy, xx = np.ogrid[:h, :w]
        inside = ((yy - h / 2) / (h / 2)) ** 2 + ((xx - w / 2) / (w / 2)) ** 2 <= 1
        mask[y:y + h, x:x + w][inside] = 0
    return img, mask


def extent_of(pipe, h, w):
    eng = pipe.model._engine(torch.device("cuda:0"))
    Hp, Wp, mx = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert eng.lib.migan_fullres_extent(eng.handle, h, w, ctypes.byref(Hp), ctypes.byref(Wp), ctypes.byref(mx)) == 0
    return Hp.value * Wp.value


def stat(v):
    return {"p50": statistics.median(v), "min": min(v), "max": max(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    A = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    hw = HoleWindowPipeline(synthetic.export_style_state_dict(R, seed=1), R, device=dev)
    full = FullResPipeline(hw.model, R, device=dev)
    rng = np.random.RandomState(0)
    photos = [fixture(rng, H, W, holes) for H, W, holes in MIX]
    imgs, masks = [p[0] for p in photos], [p[1] for p in photos]
    pinned = [torch.from_numpy(i).pin_memory() for i in imgs[:COMMON]]
    pinned_m = [torch.from_numpy(m).pin_memory() for m in masks[:COMMON]]
    res = {"card": card(), "resolution": R, "mix": [(H, W, len(h)) for H, W, h in MIX]}

    # the windows of the hole-window result are FullResPipeline's on the window crops
    outs = hw.forward_batch(imgs, masks)
    windows = hw.last_windows
    same = True
    for img, mask, out, wins in zip(imgs, masks, outs, windows):
        for y0, x0, h, w in wins:
            crop = (np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w]), np.ascontiguousarray(mask[y0:y0 + h, x0:x0 + w]))
            same &= bool(np.array_equal(out[y0:y0 + h, x0:x0 + w], full(*crop)))
    res["windows"] = windows
    res["windows_equal_fullres_on_crops"] = same
    try:
        full.forward_batch(imgs[COMMON:], masks[COMMON:])
        res["fullres_large_photo"] = "accepted"
    except ValueError as e:
        res["fullres_large_photo"] = "refused: %s" % e

    photo_px = [H * W for H, W, _ in MIX]
    gen_full = [extent_of(full, H, W) for H, W, _ in MIX[:COMMON]]
    gen_hw = [sum(extent_of(hw, h, w) for _, _, h, w in wins) for wins in windows]

    def fullres():
        full.forward_batch(imgs[:COMMON], masks[:COMMON])
        return full.last_launches, None

    def holewin():
        hw.forward_batch(imgs[:COMMON], masks[:COMMON])
        return hw.last_launches, None

    def run_async():
        t0 = time.perf_counter()
        hw.forward_batch(pinned, pinned_m, wait=False)
        t1 = time.perf_counter()
        launches = hw.last_launches
        hw.wait()
        return launches, (t1 - t0) * 1e3

    def holewin_all():
        hw.forward_batch(imgs, masks)
        return hw.last_launches, None

    forms = {"fullres": (fullres, COMMON), "holewin": (holewin, COMMON), "async": (run_async, COMMON),
             "holewin+": (holewin_all, len(MIX))}
    first = {}
    for name, (fn, _) in forms.items():      # warm-up: every shape, plan and workspace
        fn()
        first[name] = fn()[0]
    times = {k: [] for k in forms}
    enq = []
    for _ in range(A.repeats):
        for name, (fn, _) in forms.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            _, e = fn()
            torch.cuda.synchronize(dev)
            times[name].append(time.perf_counter() - t0)
            if e is not None:
                enq.append(e)
    out = {}
    for name, (_, n) in forms.items():
        t = statistics.median(times[name])
        gen = sum(gen_full) if name == "fullres" else sum(gen_hw[:n])
        out[name] = {"s": stat(times[name]), "requests_per_s": stat([n / s for s in times[name]]), "photo_mpix": sum(photo_px[:n]) / 1e6,
                     "generator_mpix": gen / 1e6, "launches": first[name]}
    out["async"]["enqueue_ms"] = stat(enq)
    res["forms"] = out
    print(json.dumps(res))
    if A.out:
        os.makedirs(os.path.dirname(os.path.abspath(A.out)), exist_ok=True)
        with open(A.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

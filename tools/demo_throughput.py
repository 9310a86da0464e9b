"""Requests/s of the reference demo's request path (scripts/demo.py:120-143) on cuda:0, resolution 512, for 32 decoded
photos: the 20 photo sizes and mask modes of the reference's places2_512_object set, six 1080 x 1920 and six 2160 x 3840
photos (seeded pixels, rectangular holes).  Three forms:

* (a) host: demo.py's PIL / OpenCV steps on the host around `migan_b200.Generator` at batch 1, x and y crossing PCIe as
  fp32 (what `python -m migan_b200.dropin scripts.demo` runs).  Skipped with a message without Pillow / OpenCV.
* (b) `DemoPipeline.forward_batch` on the numpy photos, waiting.
* (c) `DemoPipeline.forward_batch(..., wait=False)` on pinned CPU tensors, then one `wait()`.

Each form is warmed up, then the forms are timed alternately over the repeats, each repeat ending when every result is on
the host; p50 and range are reported.  (b) and (c) must give identical bytes; the bytes of (a) differ from them only where
OpenCV's default (optimised) cubic path differs from its scalar path, by at most 1, and that fraction is reported.  Records
the card name and power limit of the same run, and the kernel launches per pass.  Measurement tooling (seeded random
weights, no oracle).

    python tools/demo_throughput.py [--repeats 10] [--res 512] [--out tools/out/demo_throughput_512.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402,F401
from migan_b200 import synthetic  # noqa: E402
from migan_b200.demo import DemoPipeline, resized_size  # noqa: E402

# (W, H, mask channels) of examples/places2_512_object/{images,masks}/1..20.png
PLACES = [(512, 343, 3), (512, 380, 3), (512, 357, 3), (512, 340, 3), (512, 384, 3), (512, 384, 1), (512, 384, 1),
          (374, 512, 1), (384, 512, 1), (383, 512, 3), (512, 340, 3), (512, 332, 3), (512, 383, 3), (512, 340, 3),
          (401, 512, 3), (512, 384, 3), (512, 384, 3), (512, 340, 3), (512, 512, 3), (512, 512, 3)]
LARGE = [(1920, 1080, 3), (1080, 1920, 1), (1920, 1080, 4), (3840, 2160, 3), (2160, 3840, 1), (3840, 2160, 2)] * 2


def traffic(seed=0):
    rng = np.random.default_rng(seed)
    reqs = []
    for W, H, C in PLACES + LARGE:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        m = np.full((H, W, C), 255, np.uint8)
        hh, hw = int(rng.integers(H // 10, H // 3)), int(rng.integers(W // 10, W // 3))
        y0, x0 = int(rng.integers(0, H - hh)), int(rng.integers(0, W - hw))
        m[y0:y0 + hh, x0:x0 + hw] = 0
        reqs.append((img, np.ascontiguousarray(m[..., 0] if C == 1 else m)))
    return reqs


def host_demo(model, res, img, mask):
    """demo.py:125-140 on decoded arrays (read_mask on the mask array instead of its file)."""
    import cv2
    from PIL import Image

    def resize(image, max_size, interpolation=Image.BICUBIC):
        w, h = image.size
        if w > max_size or h > max_size:
            r = max_size / w if w > h else max_size / h
            image = image.resize((int(w * r), int(h * r)), interpolation)
        return image

    img_resized = resize(Image.fromarray(img), res)
    m = np.array(resize(Image.fromarray(mask), 512, Image.NEAREST))
    if m.ndim == 3:
        m = m[..., {4: 3, 2: 1, 3: 0}[m.shape[2]]]
    m = np.dstack([m, m, m])
    m[m < 255] = 0
    mask_resized = resize(Image.fromarray(m).convert("L"), res, Image.NEAREST)
    sq = np.array(img_resized.resize((res, res), Image.BICUBIC))
    mq = np.array(mask_resized.resize((res, res), Image.NEAREST))[:, :, None] // 255
    t = torch.Tensor(sq).float() * 2 / 255 - 1
    mt = torch.Tensor(mq).float()
    x = torch.cat([mt.permute(2, 0, 1)[None] - 0.5, t.permute(2, 0, 1)[None] * mt.permute(2, 0, 1)[None]], dim=1)
    with torch.no_grad():
        y = model(x.to("cuda"))[0]
    y = (y * 0.5 + 0.5).clamp(0, 1) * 255
    y = y.to(torch.uint8).permute(1, 2, 0).cpu().numpy()
    y = cv2.resize(y, dsize=img_resized.size, interpolation=cv2.INTER_CUBIC)
    mr = np.array(mask_resized)[:, :, None] // 255
    return np.array(img_resized) * mr + y * (1 - mr)


def rates(ts, requests):
    rate = [requests / t for t in ts]
    return {"requests_per_s_p50": statistics.median(rate), "requests_per_s_min": min(rate), "requests_per_s_max": max(rate),
            "ms_p50": statistics.median(ts) * 1e3}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None, help="JSON output (default tools/out/demo_throughput_<res>.json)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    pipe = DemoPipeline(synthetic.export_style_state_dict(args.res, seed=1), args.res, device=dev)
    reqs = traffic()
    imgs = [i for i, _ in reqs]
    masks = [m for _, m in reqs]
    pinned = [torch.from_numpy(i).pin_memory() for i in imgs]
    pinned_masks = [torch.from_numpy(m).pin_memory() for m in masks]

    try:
        import cv2  # noqa: F401
        import PIL  # noqa: F401
        have_host = True
    except ImportError:
        have_host = False
        print("form (a) skipped: Pillow and OpenCV are not installed here", file=sys.stderr)

    def host():
        return [host_demo(pipe.model, args.res, i, m) for i, m in reqs]

    def batched():
        return pipe.forward_batch(imgs, masks)

    def asynchronous():
        outs = pipe.forward_batch(pinned, pinned_masks, wait=False)
        pipe.wait()
        return outs

    forms = [("host", host)] if have_host else []
    forms += [("batched_wait", batched), ("batched_async", asynchronous)]
    results = {name: f() for name, f in forms}                       # warm-up, and the bytes of each form
    torch.cuda.synchronize()
    b = results["batched_wait"]
    identical = all(np.array_equal(x, y.numpy()) for x, y in zip(b, results["batched_async"]))
    out = {"card": card(), "resolution": args.res, "requests": len(reqs), "repeats": args.repeats,
           "photos_wh": [[i.shape[1], i.shape[0]] for i in imgs],
           "results_wh": [list(resized_size(i.shape[1], i.shape[0], args.res)) for i in imgs],
           "launches_per_pass": pipe.last_launches, "generator_launches_per_pass": pipe.model.last_launch_count(dev),
           "outputs_identical_b_c": identical}
    if have_host:
        diff = total = worst = 0
        for x, y in zip(results["host"], b):
            d = np.abs(x.astype(int) - y.astype(int))
            diff += int((d != 0).sum()); total += d.size; worst = max(worst, int(d.max()))
        out["host_vs_gpu_differing_fraction"] = diff / total
        out["host_vs_gpu_max_abs"] = worst
    del results
    times = {name: [] for name, _ in forms}
    for _ in range(args.repeats):
        for name, f in forms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    for name, ts in times.items():
        out[name] = rates(ts, len(reqs))
    if have_host:
        for name in ("batched_wait", "batched_async"):
            out["speedup_%s_over_host_p50" % name] = out[name]["requests_per_s_p50"] / out["host"]["requests_per_s_p50"]
    print(json.dumps(out, indent=1), flush=True)
    path = args.out or "tools/out/demo_throughput_%d.json" % args.res
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    if not identical:
        sys.exit("forms (b) and (c) gave different outputs")


if __name__ == "__main__":
    main()

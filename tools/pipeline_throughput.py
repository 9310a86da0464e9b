"""Requests/s of `MIGAN_Pipeline` on cuda:0 for a seeded traffic mix (photos of 512x512, 720x1280, 1080x1920 and 2160x3840
with rectangular holes; resolution 512, padding 128), in two forms:

* device-resident, 32 requests: one `pipe(image_i, mask_i)` per request (sequential) against one `forward_batch` of all of
  them (batched);
* host-resident, `--host-passes` passes of 32 requests whose images and masks are pinned CPU tensors (how decoded photos
  arrive): `forward_batch` pass by pass, each call waiting for its results (host sync), against `forward_batch(...,
  wait=False)` for every pass followed by one `wait()` (host async).

Each pair is warmed up, then timed alternately over the repeats, each repeat ending when every result is in place; p50 and
range are reported.  The two forms of a pair must give identical images.  Records the card name and power limit of the same
run.  Measurement tooling (seeded random weights, no oracle).

    python tools/pipeline_throughput.py [--repeats 10] [--res 512] [--host-passes 4]
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
from migan_b200.pipeline import MIGAN_Pipeline  # noqa: E402

SIZES = ((512, 512), (720, 1280), (1080, 1920), (2160, 3840))


def traffic(n, dev, seed=0):
    rng = np.random.RandomState(seed)
    reqs = []
    for i in range(n):
        H, W = SIZES[rng.randint(len(SIZES))]
        image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8)).to(dev)
        mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8, device=dev)
        hh, hw = int(rng.randint(H // 10, H // 3)), int(rng.randint(W // 10, W // 3))
        y0, x0 = int(rng.randint(0, H - hh)), int(rng.randint(0, W - hw))
        mask[:, :, y0:y0 + hh, x0:x0 + hw] = 0
        reqs.append((image, mask))
    return reqs


def rates(ts, requests):
    rate = [requests / t for t in ts]
    return {"requests_per_s_p50": statistics.median(rate), "requests_per_s_min": min(rate), "requests_per_s_max": max(rate),
            "ms_p50": statistics.median(ts) * 1e3}


def host_resident(pipe, passes, repeats, dev):
    """Pinned CPU requests in passes of 32: synchronous calls pass by pass against wait=False calls and one wait()."""
    src = [(im.cpu(), m.cpu()) for im, m in traffic(32 * passes, dev, seed=1)]
    images = [im.pin_memory() for im, _ in src]
    masks = [m.pin_memory() for _, m in src]

    def restore():                                                  # host copies, outside the timed window
        for im, (s, _) in zip(images, src):
            im.copy_(s)

    def sync():
        for c in range(0, len(images), 32):
            pipe.forward_batch(images[c:c + 32], masks[c:c + 32])

    def asynchronous():
        for c in range(0, len(images), 32):
            pipe.forward_batch(images[c:c + 32], masks[c:c + 32], wait=False)
        pipe.wait()

    restore(); sync()
    a = [im.clone() for im in images]
    restore(); asynchronous()
    identical = all(torch.equal(x, y) for x, y in zip(a, images))
    del a
    times = {"host_sync": [], "host_async": []}
    for _ in range(repeats):
        for name, f in (("host_sync", sync), ("host_async", asynchronous)):
            restore()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    out = {"requests": len(images), "passes": passes, "outputs_identical": identical}
    for name, ts in times.items():
        out[name] = rates(ts, len(images))
    out["speedup_p50"] = out["host_async"]["requests_per_s_p50"] / out["host_sync"]["requests_per_s_p50"]
    return out


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
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--host-passes", type=int, default=4, help="passes of 32 pinned CPU requests (0: skip the host-resident form)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    pipe = MIGAN_Pipeline(synthetic.export_style_state_dict(args.res, seed=1), args.res, padding=128, device=dev)
    reqs = traffic(args.requests, dev)
    fresh = lambda: [im.clone() for im, _ in reqs]                  # noqa: E731
    masks = [m for _, m in reqs]

    def sequential(images):
        for im, m in zip(images, masks):
            pipe(im, m)

    def batched(images):
        pipe.forward_batch(images, masks)

    a, b = fresh(), fresh()
    sequential(a)
    batched(b)
    torch.cuda.synchronize()
    identical = all(torch.equal(x, y) for x, y in zip(a, b))
    del a, b
    for f in (sequential, batched):                                 # warm-up
        f(fresh())
    torch.cuda.synchronize()
    times = {"sequential": [], "batched": []}
    for _ in range(args.repeats):
        for name, f in (("sequential", sequential), ("batched", batched)):
            images = fresh()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f(images)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            del images
    out = {"card": card(), "resolution": args.res, "padding": 128, "requests": args.requests, "repeats": args.repeats,
           "sizes": [list(im.shape[2:]) for im, _ in reqs], "outputs_identical": identical}
    for name, ts in times.items():
        out[name] = rates(ts, args.requests)
    out["speedup_p50"] = out["batched"]["requests_per_s_p50"] / out["sequential"]["requests_per_s_p50"]
    if args.host_passes > 0:
        out["host_resident"] = host_resident(pipe, args.host_passes, args.repeats, dev)
        identical = identical and out["host_resident"]["outputs_identical"]
    print(json.dumps(out, indent=1), flush=True)
    os.makedirs("tools/out", exist_ok=True)
    with open("tools/out/pipeline_throughput_%d.json" % args.res, "w") as f:
        json.dump(out, f, indent=1)
    if not identical:
        sys.exit("the two forms of a pair gave different outputs")


if __name__ == "__main__":
    main()

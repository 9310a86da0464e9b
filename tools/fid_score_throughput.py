"""End-to-end images/s of `python -m migan_b200.fid_score`'s feature loop on cuda:0, over a seeded folder of mixed-size
JPEGs (phone and camera sizes plus some at 256^2 and 512^2; seeded noise, not photos), with `fid_throughput`'s seeded
Inception weights:

* the command's loop: `fid_score.folder_features` (host decode pool, packed uint8 upload, `InceptionV3.features_u8`
  on mixed-size batches), with the host time spent waiting for decoded photos;
* the pytorch_fid-style loop that `dropin` gives: decode and `ToTensor` on the host pool, batches of one size (the
  listing grouped by size), float32 upload, `fid.InceptionV3` forward;
* the device time of the uint8 input stage next to the rest of the forward (torch.profiler, a run of its own, one
  batch of `--batch-size` photos).

Both loops run in the same call, alternating, `--steps` timed passes over the folder each after one warm-up pass.
Records the card name and its power limit, read in the same run.

    python tools/fid_score_throughput.py [--steps 3] [--batch-size 50] [--out tools/out/fid_score_throughput.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image
from torchvision.transforms.functional import to_tensor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from migan_b200 import fid, fid_score  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from fid_throughput import card, seeded_weights  # noqa: E402

# (width, height, count): camera 12 MP landscape, phone 12 MP portrait, phone 1080p, 512^2, 256^2
SIZES = [(4000, 3000, 12), (3024, 4032, 12), (1920, 1080, 32), (512, 512, 40), (256, 256, 64)]
DEV = "cuda:0"


def make_folder(root, seed=0):
    rng = np.random.default_rng(seed)
    k = 0
    for w, h, count in SIZES:
        base = rng.integers(0, 256, size=(h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)
        for _ in range(count):
            img = Image.fromarray(np.roll(base, k, axis=1)).resize((w, h), Image.BILINEAR)
            img.save(os.path.join(root, "%04d.jpg" % ((k * 7919) % 1000)), quality=90)
            k += 1
    return fid_score.plan_folder(root)


def pytorch_fid_loop(files, net, batch_size, workers):
    """pytorch_fid's loop with one size per batch: host ToTensor, float32 upload, the float forward."""
    def load(f):
        return to_tensor(E.decode_photo(f))

    by_size = defaultdict(list)
    with ThreadPoolExecutor(workers) as pool:
        for f, hw in zip(files, pool.map(lambda f: Image.open(f).size, files)):
            by_size[hw].append(f)
        out = []
        for group in by_size.values():
            for a in range(0, len(group), batch_size):
                x = torch.stack(list(pool.map(load, group[a:a + batch_size])))
                out.append(net(x.to(DEV))[0])
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch-size", type=int, default=50)
    ap.add_argument("--workers", type=int, default=min(8, len(os.sched_getaffinity(0))))
    ap.add_argument("--out", default=os.path.join(HERE, "out", "fid_score_throughput.json"))
    args = ap.parse_args()
    net = fid.InceptionV3(weights=seeded_weights(DEV))
    res = {"card": card(), "host_cores": len(os.sched_getaffinity(0)), "workers": args.workers,
           "batch_size": args.batch_size, "sizes": SIZES}
    with tempfile.TemporaryDirectory() as root:
        t = time.perf_counter()
        files = make_folder(root)
        res["images"] = len(files)
        res["folder_seconds"] = time.perf_counter() - t

        def ours():
            got = fid_score.folder_features(files, net, args.batch_size, DEV, args.workers)
            torch.cuda.synchronize()
            return got

        times = {"fid_score": [], "pytorch_fid_style": []}
        waits = []
        ours()
        pytorch_fid_loop(files, net, args.batch_size, args.workers)
        for _ in range(args.steps):
            t = time.perf_counter()
            waits.append(ours().decode_wait_s)
            times["fid_score"].append(time.perf_counter() - t)
            t = time.perf_counter()
            pytorch_fid_loop(files, net, args.batch_size, args.workers)
            times["pytorch_fid_style"].append(time.perf_counter() - t)
        for k, v in times.items():
            res[k] = {"seconds_p50": float(np.median(v)), "images_per_s": len(files) / float(np.median(v)),
                      "seconds": v}
        res["fid_score"]["decode_wait_s"] = waits

        photos = [E.decode_photo(f) for f in files[:args.batch_size]]
        net.features_u8(photos)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            net.features_u8(photos)
            torch.cuda.synchronize()
        dev = defaultdict(float)
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            name = e.name.lower()
            kind = ("input stage" if "resizeu8k" in name else "h2d copy" if "memcpy" in name
                    else "rest of forward")
            dev[kind] += e.time_range.elapsed_us() / 1e3
        res["profile_ms_one_batch"] = dict(dev)
    print(json.dumps(res))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

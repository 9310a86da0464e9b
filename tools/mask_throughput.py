"""Rate of the evaluation protocol's free-form masks: `RandomMaskStream` on cuda:0 at s = 256 and 512, seed 0.

Reported per size: GPU masks/s of `next(256)` (p50 [min, max] over `--repeats` calls, each ending in the stream's own
synchronisation), the library's host planner time per attempt (the part of a call that runs on one host core), and the
share of the stream's attempts accepted.  The card's name and power limit are read in the same run.  The masks
themselves are checked against the reference's in tests/test_masks_gpu.py.

    python tools/mask_throughput.py [--repeats 10] [--out tools/out/mask_throughput.json]
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
import torch  # noqa: E402

from migan_b200 import RandomMaskStream, _abi  # noqa: E402

BATCH = 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def planner_us_per_attempt(s: int, attempts: int = 256) -> float:
    lib = _abi.load()
    st = _abi.NpRandom()
    _abi.check(lib.migan_np_seed(ctypes.byref(st), 0))
    recs = (_abi.MaskRecord * attempts)()
    t = time.perf_counter()
    _abi.check(lib.migan_mask_plan(ctypes.byref(st), s, attempts, recs, None))
    return (time.perf_counter() - t) / attempts * 1e6


def gpu_rate(s: int, repeats: int):
    stream = RandomMaskStream(s, seed=0)
    out = torch.empty((BATCH, s, s), dtype=torch.uint8, device="cuda")
    stream.next(BATCH, out=out)                     # warm-up at the timed shape
    rates = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        stream.next(BATCH, out=out)
        torch.cuda.synchronize()
        rates.append(BATCH / (time.perf_counter() - t))
    return rates, stream.attempts, stream._accepted


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mask_throughput measures on a GPU"
    res = {"card": card(), "batch": BATCH, "sizes": {}}
    for s in (256, 512):
        rates, att, acc = gpu_rate(s, args.repeats)
        row = {"gpu_masks_per_s_p50": statistics.median(rates), "gpu_masks_per_s_min": min(rates),
               "gpu_masks_per_s_max": max(rates),
               "planner_us_per_attempt": planner_us_per_attempt(s), "accepted_share": acc / att}
        res["sizes"][str(s)] = row
        print("s=%d: GPU %.0f masks/s [%.0f, %.0f]; planner %.1f us/attempt; %.4f of attempts accepted"
              % (s, row["gpu_masks_per_s_p50"], row["gpu_masks_per_s_min"], row["gpu_masks_per_s_max"],
                 row["planner_us_per_attempt"], row["accepted_share"]))
    print("card:", res["card"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Rate of the evaluation protocol's free-form masks: `RandomMaskStream` on cuda:0 at s = 256 and 512, seed 0.

Reported per size and hole range (`--hole-range LO HI`, repeatable; [0, 1] always runs first): GPU masks/s of `next(256)` (p50 [min, max] over `--repeats` calls, each ending in the stream's own
synchronisation), the library's host planner time per attempt (the part of a call that runs on one host core), and the
share of the stream's attempts accepted with its inverse, the attempts per accepted mask.  The ranges run in turn,
--repeats rounds of one call each, so each range's p50 and range come from calls alternating with the others'.  The card's name and power limit are read in the same run.  The masks
themselves are checked against the reference's in tests/test_masks_gpu.py.

    python tools/mask_throughput.py [--repeats 10] [--hole-range 0.1 0.2 --hole-range 0.5 0.6] [--out FILE]
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


def gpu_rates(s: int, repeats: int, ranges):
    """masks/s of next(BATCH) per hole range, the ranges alternating call by call; and each stream."""
    streams = [RandomMaskStream(s, seed=0, hole_range=r) for r in ranges]
    out = torch.empty((BATCH, s, s), dtype=torch.uint8, device="cuda")
    for stream in streams:
        stream.next(BATCH, out=out)                 # warm-up at the timed shape
    rates = [[] for _ in ranges]
    for _ in range(repeats):
        for k, stream in enumerate(streams):
            torch.cuda.synchronize()
            t = time.perf_counter()
            stream.next(BATCH, out=out)
            torch.cuda.synchronize()
            rates[k].append(BATCH / (time.perf_counter() - t))
    return rates, streams


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--hole-range", type=float, nargs=2, action="append", default=[], metavar=("LO", "HI"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mask_throughput measures on a GPU"
    ranges = [(0.0, 1.0)] + [tuple(r) for r in args.hole_range]
    res = {"card": card(), "batch": BATCH, "sizes": {}}
    for s in (256, 512):
        rates, streams = gpu_rates(s, args.repeats, ranges)
        for r, rate, stream in zip(ranges, rates, streams):
            row = {"gpu_masks_per_s_p50": statistics.median(rate), "gpu_masks_per_s_min": min(rate),
                   "gpu_masks_per_s_max": max(rate), "accepted_share": stream._accepted / stream.attempts,
                   "attempts_per_mask": stream.attempts / stream._accepted}
            if r == (0.0, 1.0):
                row["planner_us_per_attempt"] = planner_us_per_attempt(s)
            res["sizes"]["%d %s" % (s, list(r))] = row
            print("s=%d hole_range %s: GPU %.0f masks/s [%.0f, %.0f]; %.2f attempts per mask"
                  % (s, list(r), row["gpu_masks_per_s_p50"], row["gpu_masks_per_s_min"], row["gpu_masks_per_s_max"],
                     row["attempts_per_mask"]))
    print("card:", res["card"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

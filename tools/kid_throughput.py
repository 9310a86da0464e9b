"""Time of KID (`kid.kernel_inception_distance`) on cuda:0 at d = 2048, S = 100 subsets of m = 1,000, on seeded
non-negative features shaped like pool3 features (|N(0, 1)| * 0.4 plus a per-column offset; not Inception features):

* the GPU call at N = 10,000 and 36,500 rows per side: p50 [min, max] of timed calls after a warm-up (the call returns
  with the result on the host, so it ends in a synchronise);
* the device time of one call (torch.profiler, a run of its own): the tile kernel and the rest, and the achieved fp64
  rate from the shapes, 2 d m^2 x 2 per subset (X X^T and Y Y^T counted as their symmetric halves, X Y^T in full);
* the same contract in numpy float64 on the host cores of the same run (the same draws, `(x @ y.T / d + 1) ** 3`
  sums), timed once;
* `--kid`'s added time in the evaluation command: `Merge.result()` at 10,000 images with and without kept features for
  KID, on seeded features in place of the network's (the chunk loop is the same either way).

Records the card name, its power limit and the host core count of the same run.

    python tools/kid_throughput.py [--steps 5] [--warmup 1] [--out tools/out/kid_throughput.json]
"""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from migan_b200 import kid  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from fid_throughput import card  # noqa: E402

D, S, M = 2048, 100, 1000


def features(n, d, seed, shift=0.0):
    rng = np.random.RandomState(seed)
    return (np.abs(rng.standard_normal((n, d))) * 0.4 + shift * rng.standard_normal(d) ** 2).astype(np.float32)


def numpy_kid(real, fake):
    """KID of the contract on the host in numpy float64, for the time a CPU implementation takes."""
    real, fake = real.astype(np.float64), fake.astype(np.float64)
    fi, ri = kid.draw_subsets(len(real), len(fake), S, M)
    terms = []
    for a, b in zip(fi, ri):
        x, y = fake[a], real[b]
        kxx, kyy, kxy = ((p @ q.T / D + 1.0) ** 3 for p, q in ((x, x), (y, y), (x, y)))
        terms.append((kxx.sum() - np.trace(kxx), kyy.sum() - np.trace(kyy), kxy.sum()))
    return kid.finish(np.array(terms), M)[0]


def stats(out):
    return {"p50_s": float(np.median(out)), "min_s": min(out), "max_s": max(out), "calls": len(out)}


def fmt(r):
    return "%.4g s [%.4g, %.4g]" % (r["p50_s"], r["min_s"], r["max_s"])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return stats(out)


def profile(fn):
    """Device time (ms) of one call: the tile kernel, and everything else."""
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            per["tile kernel" if "kid_tile" in e.key else "other"] += t / 1e3
    return dict(per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", type=str, default="10000,36500")
    ap.add_argument("--out", type=str, default=os.path.join(HERE, "out", "kid_throughput.json"))
    args = ap.parse_args()
    rec = {"card": card(), "host_cores": os.cpu_count(), "d": D, "subsets": S, "m": M, "runs": []}
    print("card:", rec["card"], "host cores:", rec["host_cores"])
    flops = 2.0 * D * M * M * 2 * S
    for n in [int(v) for v in args.sizes.split(",")]:
        real, fake = features(n, D, 21), features(n, D, 22, 0.05)
        r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
        res = kid.kernel_inception_distance(r, f)
        t = timed(lambda: kid.kernel_inception_distance(r, f), args.steps, args.warmup)
        dev = profile(lambda: kid.kernel_inception_distance(r, f))
        t0 = time.perf_counter()
        want = numpy_kid(real, fake)
        numpy_s = time.perf_counter() - t0
        tile_s = dev.get("tile kernel", 0.0) / 1e3
        run = {"n": n, "gpu": t, "device_ms": dev, "tflops_tile_kernel": flops / tile_s / 1e12 if tile_s else None,
               "tflops_call_p50": flops / t["p50_s"] / 1e12, "kid": res.kid, "std": res.std,
               "numpy_kid": want, "numpy_s": numpy_s}
        rec["runs"].append(run)
        print("N=%d: GPU call %s (%.1f TFLOP/s fp64 over the call), KID %r std %r (numpy %r)"
              % (n, fmt(t), run["tflops_call_p50"], res.kid, res.std, want))
        print("    device ms (one call): " + ", ".join("%s %.2f" % kv for kv in sorted(dev.items()))
              + (", tile kernel %.1f TFLOP/s fp64" % run["tflops_tile_kernel"] if tile_s else ""))
        print("    numpy float64 on the host: %.2f s" % numpy_s)
        del r, f
    # --kid in the evaluation command: Merge.result() with and without the kept features, N = 10,000 images.
    n = 10000
    real, fake = features(n, D, 23), features(n, D, 24, 0.05)
    r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
    chunks = E.chunk_bounds(n, E.BATCH_SIZE)

    def tail(with_kid):
        m = E.Merge(n, "cuda", True, kid=with_kid)
        for j, (a, b) in enumerate(chunks):
            m.add(E.ChunkResult(j, a, r[a:b], f[a:b], torch.zeros(b - a, device="cuda")))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.result()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    tail(True)
    plain = stats([tail(False) for _ in range(args.steps)])
    with_kid = stats([tail(True) for _ in range(args.steps)])
    rec["evaluate_tail"] = {"n": n, "without_kid": plain, "with_kid": with_kid}
    print("evaluation tail at N=%d: Merge.result() %s, with --kid %s" % (n, fmt(plain), fmt(with_kid)))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(rec, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()

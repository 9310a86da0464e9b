"""Time of precision, recall, density and coverage (`prdc.precision_recall_density_coverage`, k = 3) on cuda:0 at
d = 2048, on seeded non-negative features shaped like pool3 features (|N(0, 1)| * 0.4 plus a per-column offset; not
Inception features):

* the GPU call at N = M = 10,000 and 36,500: p50 [min, max] of timed calls after a warm-up (the call returns with the
  result on the host, so it ends in a synchronise);
* the device time of each pass of one call (torch.profiler, a run of its own): the tile kernel's five launches in
  their order (norms and radii of the real rows, norms and radii of the fake rows, the cross pass) and the rest, and
  the fp64 rate of each counted from its tile shapes (every 64 x 64 tile over ceil(d / 64) panels of 64, padding
  included);
* the same contract in numpy float64 on the host cores of the same run, timed once: distances through the Gram
  expansion on BLAS in chunks of 1,024 rows (the fast host route; the oracle's direct sums are slower still);
* `--prdc`'s added time in the evaluation command: `Merge.result()` at 10,000 images with and without it, on seeded
  features in place of the network's (the chunk loop is the same either way).

Records the card name, its power limit and the host core count of the same run.

    python tools/prdc_throughput.py [--steps 5] [--warmup 1] [--out tools/out/prdc_throughput.json]
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
from migan_b200 import prdc  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from fid_throughput import card  # noqa: E402

D, K, TILE = 2048, 3, 64
PASSES = ("norms real", "radii real", "norms fake", "radii fake", "cross")


def features(n, d, seed, shift=0.0):
    rng = np.random.RandomState(seed)
    return (np.abs(rng.standard_normal((n, d))) * 0.4 + shift * rng.standard_normal(d) ** 2).astype(np.float32)


def numpy_prdc(real, fake, k=K, chunk=1024):
    """The contract's four counts on the host in numpy float64 (Gram route), for the time a CPU implementation takes."""
    real, fake = real.astype(np.float64), fake.astype(np.float64)
    nr, nf = (real * real).sum(1), (fake * fake).sum(1)

    def blocks(a, na, b, nb):
        for s in range(0, len(a), chunk):
            yield s, np.maximum(na[s:s + chunk, None] + nb[None, :] - 2.0 * (a[s:s + chunk] @ b.T), 0.0)

    def radii(x, nx):
        out = np.empty(len(x))
        for s, Dm in blocks(x, nx, x, nx):
            out[s:s + len(Dm)] = np.partition(Dm, k, axis=1)[:, k]
        return out

    r, s_ = radii(real, nr), radii(fake, nf)
    counts = np.zeros(4, dtype=np.int64)
    cov, rec = np.zeros(len(real), bool), np.zeros(len(real), bool)
    for j, Dm in blocks(fake, nf, real, nr):
        near = Dm <= r[None, :]
        c = near.sum(1)
        counts[0] += (c > 0).sum()
        counts[2] += c.sum()
        cov |= near.any(0)
        rec |= (Dm <= s_[j:j + len(Dm), None]).any(0)
    counts[1], counts[3] = rec.sum(), cov.sum()
    return prdc.finish(counts, k, len(real), len(fake))


def pass_flops(n_real, n_fake, d=D):
    """fp64 operations of each pass's tile products, padding included."""
    t = lambda n: (n + TILE - 1) // TILE  # noqa: E731
    per_tile = 2.0 * TILE * TILE * t(d) * TILE
    return dict(zip(PASSES, (t(n_real) * per_tile, t(n_real) ** 2 * per_tile, t(n_fake) * per_tile,
                             t(n_fake) ** 2 * per_tile, t(n_fake) * t(n_real) * per_tile)))


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
    """Device time (ms) of one call: each launch of the tile kernel in order, and everything else."""
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    passes, other = [], defaultdict(float)
    for e in sorted(prof.events(), key=lambda e: e.time_range.start):
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t <= 0 or e.device_type.name != "CUDA":
            continue
        if "prdc_pass_kernel" in e.name:
            passes.append(t / 1e3)
        else:
            other["other"] += t / 1e3
    if len(passes) != len(PASSES):
        raise RuntimeError("expected %d tile-kernel launches, profiled %d" % (len(PASSES), len(passes)))
    return dict(zip(PASSES, passes)), other["other"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", type=str, default="10000,36500")
    ap.add_argument("--out", type=str, default=os.path.join(HERE, "out", "prdc_throughput.json"))
    args = ap.parse_args()
    rec = {"card": card(), "host_cores": os.cpu_count(), "d": D, "k": K, "runs": []}
    print("card:", rec["card"], "host cores:", rec["host_cores"])
    for n in [int(v) for v in args.sizes.split(",")]:
        real, fake = features(n, D, 21), features(n, D, 22, 0.02)
        r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
        res = prdc.precision_recall_density_coverage(r, f)
        t = timed(lambda: prdc.precision_recall_density_coverage(r, f), args.steps, args.warmup)
        dev, other_ms = profile(lambda: prdc.precision_recall_density_coverage(r, f))
        flops = pass_flops(n, n)
        rates = {p: flops[p] / (dev[p] / 1e3) / 1e12 for p in PASSES}
        t0 = time.perf_counter()
        want = numpy_prdc(real, fake)
        numpy_s = time.perf_counter() - t0
        run = {"n": n, "gpu": t, "device_ms": dev, "other_device_ms": other_ms, "tflops": rates,
               "tflops_call_p50": sum(flops.values()) / t["p50_s"] / 1e12, "result": res._asdict(),
               "numpy_result": want._asdict(), "numpy_s": numpy_s}
        rec["runs"].append(run)
        print("N=M=%d: GPU call %s (%.1f TFLOP/s fp64 over the call), %s (numpy %s)"
              % (n, fmt(t), run["tflops_call_p50"], tuple(res[:4]), tuple(want[:4])))
        print("    device ms (one call): " + ", ".join("%s %.2f (%.1f TFLOP/s)" % (p, dev[p], rates[p])
                                                       for p in PASSES) + ", other %.2f" % other_ms)
        print("    numpy float64 on the host: %.2f s" % numpy_s)
        del r, f
    # --prdc in the evaluation command: Merge.result() with and without it, N = 10,000 images.
    n = 10000
    real, fake = features(n, D, 23), features(n, D, 24, 0.02)
    r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
    chunks = E.chunk_bounds(n, E.BATCH_SIZE)

    def tail(with_prdc):
        m = E.Merge(n, "cuda", True, prdc=with_prdc)
        for j, (a, b) in enumerate(chunks):
            m.add(E.ChunkResult(j, a, r[a:b], f[a:b], torch.zeros(b - a, device="cuda")))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.result()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    tail(True)
    plain = stats([tail(False) for _ in range(args.steps)])
    with_prdc = stats([tail(True) for _ in range(args.steps)])
    rec["evaluate_tail"] = {"n": n, "without_prdc": plain, "with_prdc": with_prdc}
    print("evaluation tail at N=%d: Merge.result() %s, with --prdc %s" % (n, fmt(plain), fmt(with_prdc)))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(rec, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()

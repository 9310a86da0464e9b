"""Time of the Fréchet distance at d = 2048 on cuda:0, against a cuSOLVER and two host routes, on seeded feature
statistics (ReLU'd correlated Gaussian features, N = 5000 rows each):

* this library's fid_frechet_distance (fp64 block Jacobi on the device; the call is synchronous) and the public
  fid.frechet_distance on CUDA tensors (adds the finiteness and symmetry checks);
* torch.linalg.eigh / eigvalsh in float64 on the same card (cuSOLVER), the same eigenvalue route;
* the numpy eigh route on the host cores;
* fid.calculate_frechet_distance (scipy.linalg.sqrtm) on the host cores;
* the sweeps of both eigensolves, the per-kernel device time of one call (torch.profiler, a run of its own) and the
  update kernel's achieved fp64 TFLOP/s counted from its tile shapes;
* the evaluation tail at FFHQ size: two FeatureStatistics of 10,000 rows each, then mean_cov() + scipy, or
  FeatureStatistics.frechet_distance.

Each route: warm-up calls, then timed calls, p50 [min, max] of host-clock times around synchronous calls.  Records the
card name, its power limit and the host core count of the same run.

    python tools/frechet_throughput.py [--steps 10] [--host-steps 10] [--scipy-steps 3] [--out tools/out/frechet_throughput.json]
"""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from migan_b200 import fid  # noqa: E402
from fid_throughput import card  # noqa: E402

D, N_ROWS, G = 2048, 5000, 64


def times(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return {"p50_s": float(np.median(out)), "min_s": min(out), "max_s": max(out), "calls": steps, "warmup": warmup}


def fmt(r):
    return "%.4g s [%.4g, %.4g]" % (r["p50_s"], r["min_s"], r["max_s"])


def feature_stats(N, d, seed, rank=64):
    """(mu, sigma) of N rows of relu(z L + noise + b) with z in `rank` latent dimensions (float64, seeded)."""
    rng = np.random.default_rng(seed)
    mix = rng.standard_normal((rank, d)) / np.sqrt(rank)
    noise = 0.3 * rng.standard_normal((N, d))
    f = np.maximum(rng.standard_normal((N, rank)) @ mix + noise + 0.2 * rng.standard_normal(d)[None, :], 0.0)
    return f.mean(axis=0), np.cov(f, rowvar=False)


def numpy_trace_sqrt(s1, s2):
    d, v = np.linalg.eigh(s1)
    sd = np.sqrt(np.maximum(d, 0.0))
    m = (v.T @ s2 @ v) * sd[:, None] * sd[None, :]
    return float(np.sqrt(np.maximum(np.linalg.eigvalsh((m + m.T) / 2), 0.0)).sum())


def cusolver_trace_sqrt(s1, s2):
    d, v = torch.linalg.eigh(s1)
    sd = d.clamp_min(0).sqrt()
    m = (v.T @ s2 @ v) * sd[:, None] * sd[None, :]
    return torch.linalg.eigvalsh((m + m.T) / 2).clamp_min(0).sqrt().sum()


def update_flop(sweeps, n=D):
    """fp64 FLOP of the update kernels of one call: per round, J_k^T X J_l on the (g + 1) g / 2 tiles of A and X J_l on
    the (N / 64) g tiles of V (first solve only), 2 * 64^3 each product."""
    N = (n + G - 1) // G * G
    g = N // G
    rounds = 2 * g - 1
    prod = 2 * G ** 3
    a = g * (g + 1) // 2 * 2 * prod
    v = (N // G) * g * prod
    return sweeps[0] * rounds * (a + v) + sweeps[1] * rounds * a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-steps", type=int, default=10)
    ap.add_argument("--scipy-steps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "host_cores": os.cpu_count(), "d": D, "rows": N_ROWS}
    print("card: %s, host cores: %d" % (res["card"], res["host_cores"]))

    mu1, s1 = feature_stats(N_ROWS, D, seed=10)
    mu2, s2 = feature_stats(N_ROWS, D, seed=11)
    t = [torch.from_numpy(x).to(dev) for x in (mu1, s1, mu2, s2)]
    terms = fid._frechet(*t)
    res["sweeps"] = list(terms.sweeps)
    res["fid"] = terms.fid

    routes = {}
    routes["library call"] = times(lambda: fid._frechet(*t), args.steps, args.warmup)
    routes["fid.frechet_distance (CUDA tensors)"] = times(lambda: fid.frechet_distance(*t), args.steps, args.warmup)
    routes["cuSOLVER eigh + eigvalsh (torch, fp64)"] = times(lambda: cusolver_trace_sqrt(t[1], t[3]).item(), args.steps,
                                                             args.warmup)
    routes["numpy eigh route (host)"] = times(lambda: numpy_trace_sqrt(s1, s2), args.host_steps, min(args.warmup, 1))
    routes["scipy sqrtm (host)"] = times(lambda: fid.calculate_frechet_distance(mu1, s1, mu2, s2), args.scipy_steps, 1)
    res["routes"] = routes
    for k, r in routes.items():
        print("%-42s %s" % (k, fmt(r)))

    want_ts = numpy_trace_sqrt(s1, s2)
    cus = float(cusolver_trace_sqrt(t[1], t[3]))
    res["trace_sqrt"] = {"library": terms.trace_sqrt, "numpy_eigh": want_ts, "cusolver": cus}
    print("tr sqrt: library %.15g  numpy eigh %.15g  cuSOLVER %.15g" % (terms.trace_sqrt, want_ts, cus))

    # per-kernel device time of one call
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fid._frechet(*t)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name
            for key in ("frechet_pair_kernel", "frechet_update_kernel", "frechet_gemm_kernel"):
                if key in name:
                    name = key
            if "ck_items_kernel" in name:
                name = "item kernels"
            per[name][0] += e.device_time_total / 1e3
            per[name][1] += 1
    res["kernels_ms"] = {k: {"ms": v[0], "launches": v[1]} for k, v in per.items()}
    for k, v in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print("  %-28s %9.2f ms  %6d launches" % (k, v[0], v[1]))
    upd = per.get("frechet_update_kernel", [0.0, 0])[0]
    if upd > 0:
        flop = update_flop(terms.sweeps)
        res["update_tflops"] = flop / (upd / 1e3) / 1e12
        print("update kernel: %.1f GFLOP in %.1f ms = %.2f TFLOP/s fp64" % (flop / 1e9, upd, res["update_tflops"]))

    # the evaluation tail at FFHQ size: 10,000 feature rows per side
    rng = np.random.default_rng(7)
    mix = torch.from_numpy(rng.standard_normal((64, D)) / 8).float().to(dev)
    stats = []
    for side in range(2):
        st = fid.FeatureStatistics(D, device=dev)
        gen = torch.Generator(device=dev).manual_seed(side)
        for _ in range(20):
            z = torch.randn(500, 64, device=dev, generator=gen)
            st.add(torch.relu(z @ mix + 0.3 * torch.randn(500, D, device=dev, generator=gen)))
        stats.append(st)
    tail = {
        "FeatureStatistics.frechet_distance": times(lambda: stats[0].frechet_distance(stats[1]), 3, 1),
        "mean_cov() + scipy": times(lambda: fid.calculate_frechet_distance(*stats[0].mean_cov(), *stats[1].mean_cov()),
                                    1, 0),
    }
    res["ffhq_tail"] = tail
    for k, r in tail.items():
        print("tail, 10,000 rows: %-36s %s" % (k, fmt(r)))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

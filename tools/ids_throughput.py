"""Time of P-IDS / U-IDS (`ids.inception_discriminative_scores`) on cuda:0 at d = 2048, on seeded gamma-distributed
features ("overlap": the fake columns scaled by up to 1.02, "separable": by up to 1.3; not Inception features):

* the GPU solve at N = 10,000 and 36,500 pairs: p50 [min, max] of timed calls after warm-up (the call is synchronous),
  its Newton iterations and stop rule;
* per-kernel device time of one call (torch.profiler, a run of its own), grouped into Gram, Cholesky (diagonal, panel,
  trailing), substitution, margins, line search and the rest;
* sklearn's LinearSVC(dual=False).fit on the host cores of the same run, when sklearn is importable ("not measured"
  otherwise; --sklearn-max-n caps the sizes it is timed at);
* `--ids`'s added time in the evaluation command: `Merge.result()` with and without kept features, on seeded features
  in place of the network's (the chunk loop is the same either way).

Records the card name, its power limit and the host core count of the same run.

    python tools/ids_throughput.py [--steps 5] [--warmup 1] [--out tools/out/ids_throughput.json]
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
from migan_b200 import fid, ids  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from fid_throughput import card  # noqa: E402

D = 2048
PHASES = [("gram", "ids_gram"), ("cholesky", "ids_diag"), ("cholesky", "ids_panel"), ("cholesky", "ids_trail"),
          ("substitution", "ids_solve"), ("line search", "ids_line"), ("line search", "StepK"),
          ("margins", "MarginPartK"), ("margins", "MarginK"), ("gradient", "GradPartK"), ("gradient", "GradK")]


def features(n, d, kind, seed=0):
    """Seeded (real, fake) [n, d] float32 gamma features; the fake columns are scaled by up to 1 + shift."""
    rng = np.random.default_rng(seed)
    shift = {"overlap": 0.02, "separable": 0.3}[kind]
    real = rng.gamma(2.0, 0.25, (n, d))
    fake = rng.gamma(2.0, 0.25, (n, d)) * (1.0 + shift * rng.random(d))
    return real.astype(np.float32), fake.astype(np.float32)


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


def phase_of(name):
    for phase, key in PHASES:
        if key in name:
            return phase
    return "other"


def profile(fn):
    """Device time per phase (ms) of one call."""
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0 and ("ids" in e.key or "ck_items" in e.key):
            per[phase_of(e.key)] += t / 1e3
    return dict(per)


def sklearn_fit(real, fake):
    try:
        from sklearn.svm import LinearSVC
    except ImportError:
        return None
    X = np.concatenate([real, fake]).astype(np.float64)
    y = [1] * len(real) + [0] * len(fake)
    t = time.perf_counter()
    svm = LinearSVC(dual=False).fit(X, y)
    return {"seconds": time.perf_counter() - t, "n_iter": int(svm.n_iter_)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", type=str, default="10000,36500")
    ap.add_argument("--kinds", type=str, default="overlap,separable")
    ap.add_argument("--sklearn-max-n", type=int, default=10000)
    ap.add_argument("--sklearn-kinds", type=str, default="overlap")
    ap.add_argument("--out", type=str, default=os.path.join(HERE, "out", "ids_throughput.json"))
    args = ap.parse_args()
    rec = {"card": card(), "host_cores": os.cpu_count(), "d": D, "runs": []}
    print("card:", rec["card"])
    for n in [int(v) for v in args.sizes.split(",")]:
        for kind in args.kinds.split(","):
            real, fake = features(n, D, kind, seed=11)
            r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
            res = ids.inception_discriminative_scores(r, f)
            t = timed(lambda: ids.inception_discriminative_scores(r, f), args.steps, args.warmup)
            phases = profile(lambda: ids.inception_discriminative_scores(r, f))
            sk = sklearn_fit(real, fake) if n <= args.sklearn_max_n and kind in args.sklearn_kinds.split(",") else None
            run = {"n": n, "kind": kind, "gpu": t, "iterations": res.iterations, "stop_rule": res.stop_rule,
                   "p_ids": res.p_ids, "u_ids": res.u_ids, "phases_ms": phases,
                   "sklearn": sk if sk is not None else "not measured"}
            rec["runs"].append(run)
            print("N=%d %s: GPU %s, %d iterations (%s), P %.4f U %.4f" % (n, kind, fmt(t), res.iterations,
                                                                        res.stop_rule, res.p_ids, res.u_ids))
            print("    device ms per phase (one call): " + ", ".join("%s %.1f" % kv for kv in sorted(phases.items())))
            print("    sklearn LinearSVC(dual=False).fit: " + ("%.2f s, %d iterations" % (sk["seconds"], sk["n_iter"])
                                                              if sk else "not measured"))
            del r, f
    # --ids in the evaluation command: Merge.result() with and without the kept features, N = 10,000 images.
    n = 10000
    real, fake = features(n, D, "overlap", seed=12)
    r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
    chunks = E.chunk_bounds(n, E.BATCH_SIZE)

    def merged(keep):
        m = E.Merge(n, "cuda", True, keep_features=keep)
        for j, (a, b) in enumerate(chunks):
            m.add(E.ChunkResult(j, a, r[a:b], f[a:b], torch.zeros(b - a, device="cuda")))
        return m

    def tail(keep):
        m = merged(keep)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.result()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    tail(True)
    plain = stats([tail(False) for _ in range(args.steps)])
    with_ids = stats([tail(True) for _ in range(args.steps)])
    rec["evaluate_tail"] = {"n": n, "without_ids": plain, "with_ids": with_ids}
    print("evaluation tail at N=%d: Merge.result() %s, with --ids %s" % (n, fmt(plain), fmt(with_ids)))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(rec, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()

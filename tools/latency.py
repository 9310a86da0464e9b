"""Small-batch latency of Generator.forward on cuda:0: p50 / p90 of (launch + wait) per call, CUDA-graph replay vs the plain
launch sequence, device-resident input; plus the host-buffer call at batch 1.
    python tools/latency.py --res 512 --out tools/out/latency.json
Measurement tooling (scripts/demo.py:125-142 is the batch-1 caller this path serves)."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import synthetic  # noqa: E402


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(q * len(v)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = migan_b200.Generator(a.res, path="tc")
    g.load_state_dict(synthetic.export_style_state_dict(a.res, seed=1))
    g = g.to(dev).eval()
    rows = []
    for n in (1, 2, 4, 8):
        x = synthetic.synthetic_input(a.res, n, seed=3, masks="free_form").to(dev)
        for mode, gmax in (("graph", 8), ("plain", 0)):
            g.graph_max_batch = gmax
            for _ in range(10):
                g(x)
            torch.cuda.synchronize()
            lat = []
            for _ in range(a.iters):
                t0 = time.perf_counter()
                g(x)
                torch.cuda.synchronize()
                lat.append((time.perf_counter() - t0) * 1e3)
            # device time alone (events), back to back
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(50):
                g(x)
            e1.record()
            torch.cuda.synchronize()
            rows.append({"n": n, "mode": mode, "p50_ms": statistics.median(lat), "p90_ms": pct(lat, 0.9),
                         "back_to_back_ms": e0.elapsed_time(e1) / 50, "img_per_s_back_to_back": n / (e0.elapsed_time(e1) / 50) * 1e3,
                         "launches": g.last_launch_count()})
            print(rows[-1], flush=True)
    # host-buffer call, batch 1 (pinned in / out, H2D + forward + D2H + wait)
    g.graph_max_batch = 8
    xh = synthetic.synthetic_input(a.res, 1, seed=3, masks="free_form").pin_memory()
    yh = torch.empty(1, 3, a.res, a.res).pin_memory()
    for _ in range(5):
        g.forward_host(xh, out=yh)
    lat = []
    for _ in range(a.iters):
        t0 = time.perf_counter()
        g.forward_host(xh, out=yh)
        lat.append((time.perf_counter() - t0) * 1e3)
    rows.append({"n": 1, "mode": "forward_host", "p50_ms": statistics.median(lat), "p90_ms": pct(lat, 0.9)})
    print(rows[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"res": a.res, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()

"""Megapixels/s and per-kernel times of the fully convolutional forward (`Generator.forward_fc`) on cuda:0, migan-512,
next to the fixed-resolution `forward` at 512 x 512:

* `forward` and `forward_fc` at 512 x 512, n = 32
* `forward_fc` at 640 x 896 n = 8, 1024 x 1536 n = 4 and 2048 x 2048 n = 2

Each configuration is warmed up, then timed with CUDA events over `--steps` calls per repeat, the configurations
alternating over `--repeats` repeats (p50 and range reported).  A separate profiled pass per configuration brackets every
launch with events (`set_profiling` / `profile_steps`) and reports the time per kernel kind and its share of the step.
Records the card name and power limit of the same run.  Measurement tooling (seeded random weights, no oracle).

    python tools/fullconv_throughput.py [--steps 10] [--repeats 5] [--path tc] [--out tools/out/fullconv_throughput.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from collections import defaultdict

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import synthetic  # noqa: E402

CONFIGS = [("forward", 32, 512, 512), ("forward_fc", 32, 512, 512), ("forward_fc", 8, 640, 896),
           ("forward_fc", 4, 1024, 1536), ("forward_fc", 2, 2048, 2048)]


def seeded_input(n, H, W, seed):
    """x = cat([mask - 0.5, img * mask]) with 8 x 8 blocky holes, as the generator's callers build it."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(n, 3, H, W, generator=g) * 2 - 1
    mask = F.interpolate((torch.rand(n, 1, H // 8, W // 8, generator=g) > 0.4).float(), size=(H, W), mode="nearest")
    return torch.cat([mask - 0.5, img * mask], dim=1)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--path", default="tc")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    g = migan_b200.Generator(512, path=a.path)
    g.load_state_dict(synthetic.export_style_state_dict(512, seed=1))
    g = g.to(dev).eval()
    inputs = {}
    for kind, n, H, W in CONFIGS:
        inputs[(n, H, W)] = seeded_input(n, H, W, seed=n).to(dev)

    def call(kind, n, H, W):
        x = inputs[(n, H, W)]
        return g(x) if kind == "forward" else g.forward_fc(x)

    for cfg in CONFIGS:                      # warm-up: plans, tensor maps, workspaces
        for _ in range(3):
            call(*cfg)
    torch.cuda.synchronize()
    times = defaultdict(list)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.repeats):
        for cfg in CONFIGS:
            call(*cfg)
            e0.record()
            for _ in range(a.steps):
                call(*cfg)
            e1.record()
            torch.cuda.synchronize()
            times[cfg].append(e0.elapsed_time(e1) / a.steps)
    rows = []
    name = card()
    print("card: %s   path: %s   steps %d x repeats %d" % (name, a.path, a.steps, a.repeats))
    for cfg in CONFIGS:
        kind, n, H, W = cfg
        mp = n * H * W / 1e6
        ts = times[cfg]
        rate = [mp / (t / 1e3) for t in ts]
        call(*cfg)
        launches = g.last_launch_count()
        g.set_profiling(True)
        call(*cfg)
        torch.cuda.synchronize()
        by_kind = defaultdict(float)
        for label, ms, _, _ in g.profile_steps():
            by_kind[label.rsplit(".", 1)[-1]] += ms
        g.set_profiling(False)
        total = sum(by_kind.values())
        row = {"call": kind, "n": n, "H": H, "W": W, "ms_p50": statistics.median(ts), "ms_min": min(ts), "ms_max": max(ts),
               "mpix_per_s_p50": statistics.median(rate), "mpix_per_s_min": min(rate), "mpix_per_s_max": max(rate),
               "launches": launches, "kernel_ms": dict(by_kind), "sum_of_kernels_ms": total}
        rows.append(row)
        print("%-10s n=%-2d %4dx%-4d  %8.3f ms [%.3f-%.3f]  %7.1f Mpix/s [%.1f-%.1f]  launches %d" % (
            kind, n, H, W, row["ms_p50"], row["ms_min"], row["ms_max"], row["mpix_per_s_p50"], row["mpix_per_s_min"],
            row["mpix_per_s_max"], launches))
        print("           per kernel (profiled pass, share of the sum): " + "  ".join(
            "%s %.3f ms %.1f%%" % (k, v, 100 * v / total) for k, v in sorted(by_kind.items(), key=lambda kv: -kv[1])))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"card": name, "path": a.path, "steps": a.steps, "repeats": a.repeats, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()

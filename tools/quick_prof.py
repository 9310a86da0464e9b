"""Quick A/B of kernel variants: per-kernel and per-layer CUDA-event times of the generator forward (no oracle, no e2e).
    python tools/quick_prof.py --res 512 --n 32 --tag base
To compare two variants, run it on each revision with its own --tag.
Prints one summary line + the launches above --min-ms.  Profiling tooling."""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--path", default="tc")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--tag", default="")
    ap.add_argument("--min-ms", type=float, default=0.25)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.manual_seed(0)
    g = migan_b200.Generator(a.res, path=a.path).to("cuda:0").eval()
    x = torch.randn(a.n, 4, a.res, a.res, device="cuda:0")
    for _ in range(3):
        g(x)
    torch.cuda.synchronize()
    # whole-step time without per-launch events
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        g(x)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps
    g.set_profiling(True)
    acc = defaultdict(float)
    order = []
    for _ in range(a.steps):
        g(x)
        torch.cuda.synchronize()
        for label, ms, nbytes, flops in g.profile_steps():
            if label not in acc:
                order.append((label, nbytes))
            acc[label] += ms / a.steps
    by_kernel = defaultdict(float)
    for label, _ in order:
        by_kernel[label.rsplit(".", 1)[-1]] += acc[label]
    print("[%s] R=%d N=%d step %.3f ms (%.0f img/s)  launches %d  sum-of-kernels %.3f ms | %s" % (
        a.tag, a.res, a.n, step_ms, a.n / step_ms * 1e3, g.last_launch_count(), sum(acc.values()),
        "  ".join("%s %.3f" % (k, v) for k, v in sorted(by_kernel.items(), key=lambda kv: -kv[1]))))
    for label, nbytes in order:
        if acc[label] >= a.min_ms:
            print("    %-40s %.3f ms  %6.0f GB/s" % (label, acc[label], nbytes / acc[label] / 1e6))
    if a.out:
        json.dump({"tag": a.tag, "step_ms": step_ms, "launches": [{"launch": l, "ms": acc[l], "alg_bytes": b} for l, b in order]},
                  open(a.out, "w"))


if __name__ == "__main__":
    main()

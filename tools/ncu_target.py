"""Minimal process for ncu captures: `forwards` generator forwards at (res, n) on cuda:0, nothing else.
    ncu --set full -k regex:sepconv_tc -s 32 -c 3 -o tools/out/sepconv_tc python tools/ncu_target.py --res 512 --n 32
Profiling tooling (no oracle import: weights are seeded random, outputs are not checked here)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--path", default="tc")
    ap.add_argument("--forwards", type=int, default=2)
    a = ap.parse_args()
    torch.manual_seed(0)
    g = migan_b200.Generator(a.res, path=a.path).to("cuda:0").eval()
    x = torch.randn(a.n, 4, a.res, a.res, device="cuda:0")
    for _ in range(a.forwards):
        y = g(x)
    torch.cuda.synchronize()
    print("ncu_target: R=%d N=%d launches/forward=%d |y|max=%.3f" % (a.res, a.n, g.last_launch_count(), float(y.abs().max())))


if __name__ == "__main__":
    main()

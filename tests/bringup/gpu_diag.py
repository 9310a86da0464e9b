"""GPU bring-up diagnostics: per-stage error vs the oracle and a quick timing.
    python tests/bringup/gpu_diag.py --path simt --res 64 --n 2
Test/debug tooling (imports the oracle as the checker)."""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import migan_b200  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--path", default="simt")
    ap.add_argument("--res", type=int, default=64)
    ap.add_argument("--n", type=int, default=2)
    ap.add_argument("--taps", type=int, default=1)
    ap.add_argument("--time", type=int, default=0, help="time a forward at this batch size (no oracle)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = O.make_state_dict(a.res, seed=1)
    g = migan_b200.Generator(a.res, path=a.path)
    g.load_state_dict(sd)
    g = g.to(dev).eval()
    x = O.make_input(a.res, a.n, seed=5)
    taps = {}
    want = O.generator_forward(sd, x, a.res, taps=taps)
    xd = x.to(dev)
    try:
        y = g(xd)
        torch.cuda.synchronize()
    except Exception as e:  # a trapped pipeline wait leaves a host-mapped record naming the barrier
        from migan_b200 import _abi
        print("[diag] FAILED: %s" % str(e).splitlines()[-1])
        print("[diag] tensor-core pipeline timeout record: 0x%x" % (_abi.load().migan_debug_tc_timeout(0) & 0xFFFFFFFF), flush=True)
        sys.exit(3)
    d = (y.cpu() - want).abs()
    print("[diag] path=%s R=%d N=%d launches=%d  FINAL max-abs=%.3e mean-abs=%.3e |y|max=%.3f"
          % (a.path, a.res, a.n, g.last_launch_count(), float(d.max()), float(d.mean()), float(want.abs().max())), flush=True)
    if a.taps:
        for name, shape in g.tap_names():
            _, got = g.forward_with_tap(xd, name, shape)
            if name.endswith("out_skip"):
                w = taps[name[:-5]] + taps["feat%d" % shape[1]]
            else:
                w = taps[name]
            e = (got.cpu() - w).abs()
            flag = "" if float(e.max()) < 2e-4 * max(1.0, float(w.abs().max())) else "   <<<<<< MISMATCH"
            print("[diag]   %-40s %-16s max-abs=%.3e  |ref|max=%.3e%s" % (name, tuple(shape), float(e.max()), float(w.abs().max()), flag), flush=True)
    if a.time:
        xb = O.make_input(a.res, a.time, seed=6).to(dev)
        for _ in range(3):
            g(xb)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        iters = 10
        for _ in range(iters):
            g(xb)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / iters
        print("[diag] timing path=%s R=%d N=%d: %.3f ms/forward  %.1f img/s" % (a.path, a.res, a.time, dt * 1e3, a.time / dt), flush=True)


if __name__ == "__main__":
    main()

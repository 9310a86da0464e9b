"""Throughput of full-resolution inpainting (`FullResPipeline`) on cuda:0, migan-512, on a mixed traffic of photo sizes:
2 x 720 x 1280, 2 x 1080 x 1920, 2160 x 3840, 3024 x 4032, 300 x 400 and 480 x 360, with free-form holes
(`synthetic.free_form_mask`).  Three forms of the same work, alternating over `--repeats` repeats (p50 [min, max]):

1. loop    the caller's loop without this pipeline: numpy reflect pad, `.cuda()`, `forward_fc_u8` per photo, `.cpu()`
2. batch   `forward_batch(imgs, masks)` on numpy photos (waits)
3. async   `forward_batch(..., wait=False)` on pinned tensors, then one `wait()`

Reported per form: requests/s, photo and padded Mpix/s, kernel launches, host enqueue time per pass (the time until
`forward_batch(wait=False)` returns); plus the padded-pixel share of the mix (from the shapes) and the card name and power
limit read in the same run.

`--enqueue-only` times only the host enqueue of `migan_forward_hw` alternating between 1152 x 1920 and 768 x 1280 on one
workspace (what a per-shape plan cache saves).  It uses only interfaces older than this pipeline, so
`--package-root <tree>` runs it against another checkout's built package for a comparison in the same session.

    python tools/fullres_throughput.py [--repeats 5] [--out tools/out/fullres_throughput.json]
    python tools/fullres_throughput.py --enqueue-only [--package-root DIR]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time


def _args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--enqueue-only", action="store_true")
    ap.add_argument("--enqueue-calls", type=int, default=200)
    ap.add_argument("--package-root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None)
    return ap.parse_args()


A = _args()
sys.path.insert(0, os.path.abspath(A.package_root))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import migan_b200  # noqa: E402
from migan_b200 import _abi, synthetic  # noqa: E402

R = 512
MIX = [(720, 1280), (720, 1280), (1080, 1920), (1080, 1920), (2160, 3840), (3024, 4032), (300, 400), (480, 360)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def extent(g, dev, H, W):
    """The padded extent of an H x W photo, from the library (migan_fullres_extent)."""
    eng = g._engine(dev)
    Hp, Wp, mx = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _abi.check(eng.lib.migan_fullres_extent(eng.handle, H, W, ctypes.byref(Hp), ctypes.byref(Wp), ctypes.byref(mx)))
    return Hp.value, Wp.value


def host_pad(img, known, Hp, Wp):
    """What a caller does without the pipeline: reflect-pad the photo and its known-mask on the host."""
    H, W = known.shape
    return (np.pad(img, ((0, Hp - H), (0, Wp - W), (0, 0)), mode="reflect"),
            np.pad(known, ((0, Hp - H), (0, Wp - W)), mode="reflect"))


def stat(v):
    return {"p50": statistics.median(v), "min": min(v), "max": max(v)}


def enqueue_alternating(g, dev, calls):
    """Host time per migan_forward_hw enqueue, alternating between two extents on one workspace (n = 1)."""
    eng = g._engine(dev)
    lib = eng.lib
    shapes = [(1152, 1920), (768, 1280)]
    need = max(lib.migan_workspace_bytes_hw(eng.handle, 1, H, W) for H, W in shapes)
    raw = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
    ws = raw[(-raw.data_ptr()) % 1024:][:need]
    xs = [torch.zeros(1, 4, H, W, device=dev) for H, W in shapes]
    ys = [torch.empty(1, 3, H, W, device=dev) for H, W in shapes]
    stream = torch.cuda.current_stream(dev).cuda_stream
    path = _abi.path_id(g.path)
    times = []
    for i in range(calls + 4):
        k = i % 2
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        _abi.check(lib.migan_forward_hw(eng.handle, xs[k].data_ptr(), ys[k].data_ptr(), 1, *shapes[k], ws.data_ptr(),
                                        ws.numel(), path, stream))
        t1 = time.perf_counter()
        if i >= 4:                       # the first calls of each extent build its plan in either version
            times.append((t1 - t0) * 1e3)
    torch.cuda.synchronize(dev)
    return {"shapes": shapes, "enqueue_ms": stat(times)}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    sd = synthetic.export_style_state_dict(R, seed=1)
    res = {"card": card(), "resolution": R}
    if A.enqueue_only:
        g = migan_b200.Generator(R)
        g.load_state_dict(sd)
        g = g.to(dev).eval()
        res["package_root"] = os.path.abspath(A.package_root)
        res["forward_hw_alternating"] = enqueue_alternating(g, dev, A.enqueue_calls)
        print(json.dumps(res))
        return
    from migan_b200.fullres import FullResPipeline

    pipe = FullResPipeline(sd, R, device=dev)
    g = pipe.model
    rng = np.random.RandomState(0)
    imgs, masks = [], []
    for H, W in MIX:
        imgs.append(rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8))
        s = max(H, W)
        m = synthetic.free_form_mask(s, rng, hole_range=(0.1, 0.4))[:H, :W]
        masks.append((m * 255).astype(np.uint8))
    pinned = [torch.from_numpy(i).pin_memory() for i in imgs]
    photo_px = sum(H * W for H, W in MIX)
    exts = [extent(g, dev, H, W) for H, W in MIX]
    padded_px = sum(Hp * Wp for Hp, Wp in exts)
    res.update({"mix": MIX, "photo_mpix": photo_px / 1e6, "padded_mpix": padded_px / 1e6,
                "padded_share": (padded_px - photo_px) / padded_px})

    def loop():
        launches = 0
        out = []
        for img, m, ext in zip(imgs, masks, exts):
            H, W = m.shape
            pi, pm = host_pad(img, m, *ext)
            o = g.forward_fc_u8(torch.from_numpy(pi[None]).cuda(dev), torch.from_numpy(pm[None]).cuda(dev))
            launches += 2 + g.last_launch_count()
            out.append(o[0, :H, :W].cpu())
        return launches, None

    def batch():
        pipe.forward_batch(imgs, masks)
        return pipe.last_launches, None

    def run_async():
        t0 = time.perf_counter()
        pipe.forward_batch(pinned, masks, wait=False)
        t1 = time.perf_counter()
        pipe.wait()
        return pipe.last_launches, (t1 - t0) * 1e3

    forms = {"loop": loop, "batch": batch, "async": run_async}
    first = {}
    for name, fn in forms.items():      # warm-up: every shape, plan and workspace
        fn()
        first[name] = fn()
    ref = pipe.forward_batch(imgs, masks)
    loop_out = []
    for img, m, ext in zip(imgs, masks, exts):
        H, W = m.shape
        pi, pm = host_pad(img, m, *ext)
        loop_out.append(g.forward_fc_u8(torch.from_numpy(pi[None]).cuda(dev), torch.from_numpy(pm[None]).cuda(dev))[0, :H, :W].cpu().numpy())
    res["batch_equals_loop"] = all(np.array_equal(a, b) for a, b in zip(ref, loop_out))
    times = {k: [] for k in forms}
    enq = []
    for _ in range(A.repeats):
        for name, fn in forms.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            _, e = fn()
            torch.cuda.synchronize(dev)
            times[name].append(time.perf_counter() - t0)
            if e is not None:
                enq.append(e)
    out = {}
    for name in forms:
        t = statistics.median(times[name])
        out[name] = {"s": stat(times[name]), "requests_per_s": len(MIX) / t, "photo_mpix_per_s": photo_px / 1e6 / t,
                     "padded_mpix_per_s": padded_px / 1e6 / t, "launches": first[name][0]}
    out["async"]["enqueue_ms_per_pass"] = stat(enq)
    res["forms"] = out
    res["forward_hw_alternating"] = enqueue_alternating(g, dev, A.enqueue_calls)
    print(json.dumps(res))
    if A.out:
        os.makedirs(os.path.dirname(os.path.abspath(A.out)), exist_ok=True)
        with open(A.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

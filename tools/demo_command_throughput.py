"""Images/s of `python -m migan_b200.demo` on cuda:0 at migan-512, on a seeded photo directory written to a temporary
directory: `--n` JPEG photos (default 1,024) of mixed sizes from 480 x 360 to 4032 x 3024, with PNG masks of their own
size (modes L and RGBA).  Three forms, timed alternately over `--repeats`, p50 and range:

* command: `demo_command.demo(...)` in this process, from the weight file to the last PNG written (interpreter start
  excluded; the plan, the header pass and the weight upload included);
* loop: `run_rank` alone on a loaded `DemoSetup` (the chunk loop: decode, GPU passes, readback, PNG encode);
* host: scripts/demo.py restated (PIL decode, PIL and OpenCV resizes on the CPU, read_mask, preprocess) around the same
  H100 generator at batch 1, saving each PNG, on the first `--host-n` photos only (it is slow).

The loop also reports the share of its wall time the host spent waiting for decoded chunks, for a chunk's GPU results
and for PNG encodes.  The card name and power limit are read in the same run.  Only one GPU is used: rates at W > 1 are
not measured here.  Measurement tooling (seeded random weights, no oracle).

    python tools/demo_command_throughput.py [--n 1024] [--repeats 3] [--num-workers 8] [--out tools/out/demo_command.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402,F401
from migan_b200 import demo_command as D  # noqa: E402
from migan_b200 import synthetic  # noqa: E402

SIZES = [(480, 360), (640, 480), (1024, 768), (1280, 720), (1920, 1080), (2048, 1536), (3024, 4032), (4032, 3024)]


def write_photo(root: Path, k: int, seed: int):
    from PIL import Image
    rng = np.random.default_rng((seed, k))
    W, H = SIZES[int(rng.integers(0, len(SIZES)))]
    low = rng.integers(0, 256, (H // 16 + 1, W // 16 + 1, 3), dtype=np.uint8)
    img = np.asarray(Image.fromarray(low).resize((W, H), Image.BILINEAR))
    img = (img ^ (rng.integers(0, 16, (H, W, 1), dtype=np.uint8))).astype(np.uint8)
    sub = root / "images" / ("d%d" % (k % 4))
    Image.fromarray(img).save(sub / ("photo_%04d.jpg" % k), quality=90)
    v = np.full((H, W), 255, np.uint8)
    hh, ww = int(rng.integers(H // 8, H // 3)), int(rng.integers(W // 8, W // 3))
    y0, x0 = int(rng.integers(0, H - hh)), int(rng.integers(0, W - ww))
    v[y0:y0 + hh, x0:x0 + ww] = 0
    m = Image.fromarray(v) if k % 2 else Image.fromarray(np.dstack([v, v, v, v]), "RGBA")
    m.save(root / "masks" / ("photo_%04d.png" % k))
    return W * H


def host_loop(model, res, items, out: Path):
    """scripts/demo.py:122-142 over files, with the generator on the GPU at batch 1."""
    import cv2
    from PIL import Image

    def resize(image, max_size, interpolation=Image.BICUBIC):
        w, h = image.size
        if w > max_size or h > max_size:
            r = max_size / w if w > h else max_size / h
            image = image.resize((int(w * r), int(h * r)), interpolation)
        return image

    def read_mask(path):
        mask = np.array(resize(Image.open(path), 512, Image.NEAREST))
        if mask.ndim == 3:
            mask = mask[..., {4: 3, 2: 1, 3: 0}[mask.shape[2]]]
        mask = np.dstack([mask, mask, mask])
        mask[mask < 255] = 0
        return Image.fromarray(mask).convert("L")

    for it in items:
        img_resized = resize(Image.open(it.photo).convert("RGB"), res)
        mask_resized = resize(read_mask(it.mask), res, Image.NEAREST)
        sq = np.array(img_resized.resize((res, res), Image.BICUBIC))
        mq = np.array(mask_resized.resize((res, res), Image.NEAREST))[:, :, None] // 255
        t = torch.Tensor(sq).float() * 2 / 255 - 1
        mt = torch.Tensor(mq).float().permute(2, 0, 1)[None]
        x = torch.cat([mt - 0.5, t.permute(2, 0, 1)[None] * mt], dim=1)
        with torch.no_grad():
            y = model(x.to("cuda"))[0]
        y = ((y * 0.5 + 0.5).clamp(0, 1) * 255).to(torch.uint8).permute(1, 2, 0).cpu().numpy()
        y = cv2.resize(y, dsize=img_resized.size, interpolation=cv2.INTER_CUBIC)
        mr = np.array(mask_resized)[:, :, None] // 255
        Image.fromarray(img_resized * mr + y * (1 - mr)).save(out / it.output)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def summary(rates):
    return {"images_per_s_p50": statistics.median(rates), "images_per_s_min": min(rates),
            "images_per_s_max": max(rates), "runs": len(rates)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--host-n", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=8)
    ap.add_argument("--out", default=None, help="JSON output (default tools/out/demo_command.json)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("demo_command_throughput needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model_name = "migan-%d" % args.res
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        for k in range(4):
            (root / "images" / ("d%d" % k)).mkdir(parents=True)
        (root / "masks").mkdir()
        t = time.perf_counter()
        with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as pool:
            pixels = sum(pool.map(lambda k: write_photo(root, k, 0), range(args.n)))
        print("wrote %d photos (%.1f Mpixel on average) in %.1f s" % (args.n, pixels / args.n / 1e6,
                                                                     time.perf_counter() - t), flush=True)
        wpath = root / "weights.pth"
        torch.save(synthetic.export_style_state_dict(args.res, seed=1), wpath)
        kw = dict(batch_size=args.batch_size, num_workers=args.num_workers, device=dev)

        def command(out):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = D.demo(model_name, wpath, root / "images", root / "masks", out, **kw)
            return time.perf_counter() - t0, st

        setup = D.DemoSetup(model_name, wpath, root / "images", root / "masks", root / "out_loop", **kw)
        host_items = setup.items[:args.host_n]
        (root / "out_host").mkdir()

        def host():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_loop(setup.model, args.res, host_items, root / "out_host")
            return time.perf_counter() - t0

        # warm-up: every form once (kernels, plans, pinned-memory cache, page cache of the files)
        command(root / "out_cmd")
        D.run_rank(setup)
        host_loop(setup.model, args.res, host_items[:4], root / "out_host")
        rates = {"command": [], "loop": [], "host": []}
        shares = []
        for r in range(args.repeats):
            s, st = command(root / "out_cmd")
            rates["command"].append(st.images / s)
            st = D.run_rank(setup)
            rates["loop"].append(st.images / st.seconds)
            shares.append({"decode": st.decode_wait_s / st.seconds, "gpu": st.gpu_wait_s / st.seconds,
                           "encode": st.encode_wait_s / st.seconds})
            rates["host"].append(len(host_items) / host())
            print("repeat %d: command %.1f, loop %.1f, host %.2f images/s; loop waits: decode %.1f %%, gpu %.1f %%, "
                  "encode %.1f %%" % (r, rates["command"][-1], rates["loop"][-1], rates["host"][-1],
                                      100 * shares[-1]["decode"], 100 * shares[-1]["gpu"], 100 * shares[-1]["encode"]),
                  flush=True)
        same = sum((root / "out_cmd" / it.output).read_bytes() == (root / "out_loop" / it.output).read_bytes()
                   for it in setup.items)
        host_same = sum((root / "out_host" / it.output).read_bytes() == (root / "out_cmd" / it.output).read_bytes()
                        for it in host_items)
    res = {
        "card": card(), "model": model_name, "photos": args.n, "mean_megapixels": pixels / args.n / 1e6,
        "batch_size": args.batch_size, "num_workers": args.num_workers, "host_photos": len(host_items),
        "command": summary(rates["command"]), "loop": summary(rates["loop"]), "host": summary(rates["host"]),
        "loop_wait_share_p50": {k: statistics.median(s[k] for s in shares) for k in ("decode", "gpu", "encode")},
        "command_files_equal_loop_files": "%d of %d" % (same, len(setup.items)),
        "host_files_byte_identical": "%d of %d (OpenCV's default cubic path may differ by 1 from the scalar path the "
                                     "pipeline reproduces)" % (host_same, len(host_items)),
        "not_measured": "more than one GPU (W > 1)",
    }
    print(json.dumps(res, indent=1))
    out = args.out or os.path.join(os.path.dirname(os.path.abspath(__file__)), "out", "demo_command.json")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

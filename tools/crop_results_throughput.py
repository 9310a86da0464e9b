"""Images/s of `python -m migan_b200.crop_results` on cuda:0 at migan-512, on a seeded photo directory written to a
temporary directory: `--n` JPEG photos (default 256) of phone and camera sizes from 640 x 480 to 4032 x 3024, with PNG
masks (mode L) of their own size holding one or two local holes.  Timed alternately over `--repeats`, p50 and range:

* command: `crop_results.crop_results(...)` in this process, from the weight file to the last PNG written (interpreter
  start excluded; the plan, the header pass and the weight upload included);
* caller loop: what a user writes without the command, on the first `--loop-n` photos: PIL decode, host `read_mask`,
  transpose to [1,3,H,W], one `MIGAN_Pipeline` call per photo, transpose back, PNG encode;
* device: CUDA-event time of one `CropPipeline.forward_batch` pass of 32 decoded photos already on the device (mask
  launch, flags, planning, pre-processing, generator, blend).

The card name and power limit are read in the same run.  Measurement tooling (seeded random weights, no oracle).

    python tools/crop_results_throughput.py [--n 256] [--loop-n 64] [--repeats 3] [--out tools/out/crop_results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402,F401
from migan_b200 import crop_results as C  # noqa: E402
from migan_b200 import demo_command as D  # noqa: E402
from migan_b200 import synthetic  # noqa: E402
from migan_b200.pipeline import CropPipeline, MIGAN_Pipeline  # noqa: E402

SIZES = [(640, 480), (1280, 720), (1920, 1080), (2048, 1536), (3024, 4032), (4032, 3024), (1080, 1920), (3264, 2448)]
RES = 512


def write_photo(images: Path, masks: Path, k: int, seed: int) -> None:
    from PIL import Image
    rng = np.random.default_rng(seed * 100003 + k)
    w, h = SIZES[k % len(SIZES)]
    low = rng.integers(0, 256, (max(2, h // 64), max(2, w // 64), 3), dtype=np.uint8)
    img = np.asarray(Image.fromarray(low).resize((w, h), Image.BILINEAR))
    Image.fromarray(img).save(images / ("p%04d.jpg" % k), quality=90)
    m = np.full((h, w), 255, np.uint8)
    for _ in range(1 + k % 2):
        hh, ww = int(rng.integers(h // 16, h // 5)), int(rng.integers(w // 16, w // 5))
        y0, x0 = int(rng.integers(0, h - hh)), int(rng.integers(0, w - ww))
        m[y0:y0 + hh, x0:x0 + ww] = 0
    Image.fromarray(m).save(masks / ("p%04d.png" % k))


def read_mask(path, invert=False):
    """create_onnx_pipeline.py:27-45, on the host."""
    from PIL import Image
    mask = np.array(Image.open(path))
    if mask.ndim == 3:
        mask = mask[:, :, {4: 3, 2: 1, 3: 0}[mask.shape[2]]]
    mask = np.dstack([mask, mask, mask])
    if invert:
        mask = 255 - mask
    mask[mask < 255] = 0
    return Image.fromarray(mask).convert("L")


def caller_loop(pipe, items, out: Path) -> None:
    from PIL import Image
    out.mkdir(parents=True, exist_ok=True)
    for it in items:
        img = Image.open(it.photo).convert("RGB")
        mask = read_mask(it.mask)
        with torch.no_grad():
            x = np.expand_dims(img, 0).transpose(0, 3, 1, 2)
            m = np.expand_dims(mask, (0, 1))
            result = pipe(torch.tensor(x), torch.tensor(m)).numpy()
        Image.fromarray(result[0].transpose(1, 2, 0)).save(out / D.output_name(it.photo))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def summary(values, key):
    return {key + "_p50": statistics.median(values), key + "_min": min(values), key + "_max": max(values),
            "runs": len(values)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--loop-n", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--num-workers", type=int, default=8)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crop_results_throughput needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"card": card(), "resolution": RES, "photos": args.n, "sizes": SIZES}
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        images, masks = root / "images", root / "masks"
        images.mkdir()
        masks.mkdir()
        for k in range(args.n):
            write_photo(images, masks, k, seed=1)
        wpath = root / "migan.pth"
        sd = synthetic.export_style_state_dict(RES, seed=1)
        torch.save(sd, wpath)
        items = D.plan_items(D.list_photos(images), masks)
        ref = MIGAN_Pipeline(sd, RES, device=dev)

        def command(out):
            t = time.perf_counter()
            C.crop_results(wpath, RES, images, masks, out, device=dev, num_workers=args.num_workers)
            torch.cuda.synchronize()
            return args.n / (time.perf_counter() - t)

        def loop(out):
            t = time.perf_counter()
            caller_loop(ref, items[:args.loop_n], out)
            torch.cuda.synchronize()
            return args.loop_n / (time.perf_counter() - t)

        command(root / "warm_cmd")
        loop(root / "warm_loop")
        same = all((root / "warm_cmd" / "sample_results" / D.output_name(it.photo)).read_bytes()
                   == (root / "warm_loop" / D.output_name(it.photo)).read_bytes() for it in items[:args.loop_n])
        rates = {"command": [], "caller_loop": []}
        for r in range(args.repeats):
            rates["command"].append(command(root / ("cmd%d" % r)))
            rates["caller_loop"].append(loop(root / ("loop%d" % r)))
        result["command"] = summary(rates["command"], "images_per_s")
        result["caller_loop"] = summary(rates["caller_loop"], "images_per_s")
        result["caller_loop"]["photos"] = args.loop_n
        result["command_files_equal_caller_loop"] = same

        # device time of one pass of 32 decoded photos on the device
        from PIL import Image
        pipe = CropPipeline(sd, RES, device=dev)
        chunk = items[:32]
        imgs = [torch.from_numpy(np.array(Image.open(it.photo).convert("RGB"))).to(dev) for it in chunk]
        ms = [torch.from_numpy(np.array(Image.open(it.mask))).to(dev) for it in chunk]
        pipe.forward_batch(imgs, ms)
        times = []
        for _ in range(max(5, 3 * args.repeats)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pipe.forward_batch(imgs, ms)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        result["device_pass_32"] = summary(times, "ms")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()

"""Cost of `--ssim --psnr --per-image` in the evaluation command's chunk loop, migan-512 on `tools/evaluate_throughput.py`'s
2,048 seeded 768 x 512 JPEG photos with their PNG masks.

* in process: `evaluate()` without and with `ssim=True, psnr=True, per_image=True`, each called once to warm up, then
  alternating, --repeats times: the chunk loop's images/s (`EvalResult.seconds`) and its share of host-decode waiting,
  reported as p50 and range; the FID and LPIPS of the two forms must be the same bits;
* device: CUDA events around the chunk's added work -- the hole fraction, `metrics.compute_ssim`,
  `metrics.compute_psnr` and the column stack on one 32-image chunk at 512 x 512 -- next to the LPIPS and Inception
  calls every chunk already makes on the same tensors, --steps launches each after warm-up.

Seeded random weights (MI-GAN from `synthetic`, Inception and LPIPS as tools/fid_throughput.py and
tools/lpips_throughput.py build them).  Records the card name and power limit of the same run.

    python tools/per_image_scores_throughput.py [--data /tmp/evaldata] [--num-workers 8] [--out tools/out/per_image.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import migan_b200  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from migan_b200 import fid, lpips, metrics, synthetic  # noqa: E402
from evaluate_throughput import N, R, write_data  # noqa: E402
from fid_throughput import card, seeded_weights as inception_weights  # noqa: E402
from lpips_throughput import seeded_weights as lpips_weights  # noqa: E402
from score_results_throughput import summary  # noqa: E402

FLAGS = dict(ssim=True, psnr=True, per_image=True)


def event_ms(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def device_costs(sd, isd, lsd, real_dir, mask_dir, steps, dev):
    """Per-chunk device ms of the added work and of the chunk's existing LPIPS and Inception calls."""
    from PIL import Image
    paths = E.list_images(real_dir)[:E.BATCH_SIZE]
    photos = [np.array(Image.open(p).convert("RGB")) for p in paths]
    masks = [np.array(Image.open(m).convert("L")) for m in E.list_masks(paths, mask_dir)]
    pipe = migan_b200.EvalPipeline(sd, R, device=dev)
    real, composed, _ = pipe.forward_batch(photos, masks, hole_fraction=True)
    x = torch.rand((len(paths), 4, R, R), device=dev)          # stands for the pass's x: channel 0 is read
    net = lpips.LPIPS(net="alex", weights=lsd).to(dev)
    inception = fid.InceptionV3(weights=isd)

    def added():
        hole = 1 - (x[:, 0] + 0.5).mean((1, 2))
        torch.stack([hole, metrics.compute_ssim(real, composed, window_size=11, size_average=False),
                     metrics.compute_psnr(composed, real, for_dataset=None)], 1)

    with torch.no_grad():
        return {"chunk": len(paths),
                "added_ms": event_ms(added, steps),
                "ssim_ms": event_ms(lambda: metrics.compute_ssim(real, composed, window_size=11, size_average=False),
                                    steps),
                "psnr_ms": event_ms(lambda: metrics.compute_psnr(composed, real, for_dataset=None), steps),
                "lpips_ms": event_ms(lambda: net(real, composed, normalize=True), steps),
                "inception_ms": event_ms(lambda: inception(torch.cat([real, composed])), steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default="/tmp/migan_evaluate_throughput")
    ap.add_argument("--num-workers", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "n": N, "R": R, "photo": "%dx%d JPEG" % (R * 3 // 2, R), "num_workers": a.num_workers,
           "repeats": a.repeats}
    print(json.dumps({"card": res["card"]}), flush=True)
    real, masks = write_data(a.data)
    sd, isd, lsd = synthetic.export_style_state_dict(R, seed=1), inception_weights(dev), lpips_weights()

    kw = dict(device=dev, num_workers=a.num_workers, inception_weights=isd, lpips_weights=lsd)
    calls = {"plain": lambda: E.evaluate("migan-512", sd, real, masks, **kw),
             "ssim_psnr_per_image": lambda: E.evaluate("migan-512", sd, real, masks, **kw, **FLAGS)}
    for call in calls.values():
        call()                                                   # warm-up: uploads, workspaces
    loops = {k: [] for k in calls}
    for rep in range(a.repeats):
        for name, call in calls.items():
            r = call()
            loops[name].append(r)
            print(json.dumps({"in_process": name, "repeat": rep, "loop_s": r.seconds, "decode_wait_s": r.decode_wait_s,
                              "fid": r.fid, "lpips": r.lpips, "ssim": r.ssim, "psnr": r.psnr}), flush=True)
    plain, flagged = loops["plain"][0], loops["ssim_psnr_per_image"][0]
    res["same_fid_lpips"] = (plain.fid, plain.lpips) == (flagged.fid, flagged.lpips)
    res["loop_images_per_s"] = {k: summary([N / r.seconds for r in v]) for k, v in loops.items()}
    res["decode_wait_share"] = {k: summary([r.decode_wait_s / r.seconds for r in v]) for k, v in loops.items()}
    p50 = res["loop_images_per_s"]
    res["loop_cost_share"] = 1 - p50["ssim_psnr_per_image"]["p50"] / p50["plain"]["p50"]
    res["device"] = device_costs(sd, isd, lsd, real, masks, a.steps, dev)
    d = res["device"]
    res["device"]["added_share_of_lpips_inception"] = d["added_ms"] / (d["lpips_ms"] + d["inception_ms"])
    print(json.dumps({k: res[k] for k in ("card", "loop_images_per_s", "loop_cost_share", "decode_wait_share",
                                          "same_fid_lpips", "device")}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Latency of one `MIGAN_Pipeline` request (any-size image + mask -> in-place result) on cuda:0: p50 over 30 requests per
image size, split into the part before the crop window is known (mask resize + hole flags + D2H) and the rest.
Measurement tooling (seeded random weights, no oracle)."""
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import synthetic  # noqa: E402
from migan_b200.pipeline import MIGAN_Pipeline  # noqa: E402


def main():
    res = int(sys.argv[1]) if len(sys.argv) > 1 else 512
    dev = torch.device("cuda", 0)
    pipe = MIGAN_Pipeline(synthetic.export_style_state_dict(res, seed=1), res, padding=128, device=dev)
    rng = np.random.RandomState(0)
    rows = []
    for (H, W) in ((512, 512), (1080, 1920), (2160, 3840)):
        image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8)).to(dev)
        mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8, device=dev)
        mask[:, :, H // 3: H // 3 + H // 4, W // 3: W // 3 + W // 4] = 0
        for _ in range(3):
            pipe(image.clone(), mask)
        torch.cuda.synchronize()
        lat, box_ms = [], []
        for _ in range(30):
            img = image.clone()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.get_masked_bbox(mask)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            pipe(img, mask)
            torch.cuda.synchronize()
            lat.append((time.perf_counter() - t2) * 1e3)
            box_ms.append((t1 - t0) * 1e3)
        rows.append({"image": [H, W], "crop_window": list(pipe.last_box), "p50_ms": statistics.median(lat), "p90_ms": sorted(lat)[26],
                     "crop_window_stage_p50_ms": statistics.median(box_ms)})
        print(rows[-1], flush=True)
    out = {"resolution": res, "padding": 128, "requests": rows}
    os.makedirs("tools/out", exist_ok=True)
    json.dump(out, open("tools/out/pipeline_latency_%d.json" % res, "w"), indent=1)


if __name__ == "__main__":
    main()

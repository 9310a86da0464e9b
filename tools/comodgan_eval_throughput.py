"""Throughput of the Co-Mod-GAN evaluation step on cuda:0 at comodgan-256 and comodgan-512, two ways:

* pipeline: `EvalPipeline` with a `comodgan.Generator` (GPU resizes and composite, seeded noise drawn on the device,
  generator chunks of `generator_batch`), then `lpips.LPIPS`, two `fid.InceptionV3` calls and two
  `FeatureStatistics.add`;
* dropin: the loop the unmodified evaluation script runs under `dropin`: PIL BICUBIC / NEAREST resizes and x on the host,
  `comodgan.Generator(x)` (z and noise planes from torch.randn), the composite on the host after a copy back, then the
  same LPIPS and Inception calls.

Images/s as p50 [min, max] over alternating repeats of both loops, n = 32 photos of 1.5R x R per step (the resize runs)
and R x R directory masks.  Seeded random weights; records the card name and power limit of the same run.

    python tools/comodgan_eval_throughput.py [--steps 3] [--repeats 5] [--out tools/out/comodgan_eval_throughput.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import comodgan, fid, lpips  # noqa: E402
from fid_throughput import card, seeded_weights as inception_weights, timed  # noqa: E402
from lpips_throughput import seeded_weights as lpips_weights  # noqa: E402

N = 32


def comodgan_weights(R, seed=1):
    """Seeded state_dict: unit-variance weights and small non-zero biases, noise strengths and w_avg."""
    g = comodgan.Generator(comodgan.Mapping(num_ws=2 * int(np.log2(R)) - 2), comodgan.Encoder(resolution=R),
                           comodgan.Synthesis(resolution=R))
    gen = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in g.state_dict().items():
        if k.endswith("resample_filter"):
            sd[k] = v
        elif k.endswith("weight") or k.endswith("noise_const"):
            sd[k] = torch.randn(v.shape, generator=gen)
        else:
            sd[k] = 0.1 * torch.randn(v.shape, generator=gen)
    return sd


def dropin_batch(model, imgs, masks, R, dev):
    """The script's batch under dropin: InferenceDataset on the host, model(x), the composite on the host."""
    from PIL import Image
    xs, ims, mks = [], [], []
    for img, mask in zip(imgs, masks):
        im = Image.fromarray(img)
        if im.size != (R, R):
            im = im.resize((R, R), Image.BICUBIC)
        mk = Image.fromarray(mask)
        if mk.size != (R, R):
            mk = mk.resize((R, R), Image.NEAREST)
        a = torch.from_numpy(np.array(im)).float().permute(2, 0, 1) * 2 / 255 - 1
        m = torch.from_numpy(np.array(mk)[None] // 255).float()
        xs.append(torch.cat([m - 0.5, a * m]))
        ims.append(a)
        mks.append(m)
    x, im, mk = torch.stack(xs), torch.stack(ims), torch.stack(mks)
    y = model(x.to(dev)).cpu()
    composed = mk * im + (1 - mk) * y
    return (im * 0.5 + 0.5).clamp(0, 1).to(dev), (composed * 0.5 + 0.5).clamp(0, 1).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "n": N}
    net = lpips.LPIPS(net="alex", weights=lpips_weights()).to(dev)
    inception = fid.InceptionV3(weights=inception_weights(dev))
    for R in (256, 512):
        model = comodgan.load(comodgan_weights(R), R).to(dev)
        pipe = migan_b200.EvalPipeline(model, R, device=dev, seed=0)
        rng = np.random.default_rng(R)
        imgs = [rng.integers(0, 256, size=(R, R * 3 // 2, 3), dtype=np.uint8) for _ in range(N)]
        masks = [np.where(rng.random((R, R)) < 0.4, 0, 255).astype(np.uint8) for _ in range(N)]
        s_r, s_c = fid.FeatureStatistics(device=dev), fid.FeatureStatistics(device=dev)

        def finish(real, composed):
            net(real, composed, normalize=True)
            s_r.add(inception(real)[0])
            s_c.add(inception(composed)[0])

        loops = {"pipeline": lambda: finish(*pipe.forward_batch(imgs, masks)),
                 "dropin": lambda: finish(*dropin_batch(model, imgs, masks, R, dev))}
        rates = {k: [] for k in loops}
        with torch.no_grad():
            for _ in range(a.repeats):
                for name, fn in loops.items():
                    rates[name].append(N / timed(fn, a.steps, warmup=1))
        row = {k: {"images_per_s_p50": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
               for k, v in rates.items()}
        row["generator_batch"] = pipe.noise.generator_batch
        row["pass_launches"] = pipe.last_launches
        res["comodgan_%d" % R] = row
        print(json.dumps({"comodgan_%d" % R: row, "card": res["card"]}), flush=True)
        del model, pipe
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

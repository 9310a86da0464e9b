"""Throughput of SSIM and PSNR on cuda:0, next to pytorch-ssim in eager PyTorch on the same card:

* SSIM (window 11) and PSNR (None, "div2k" and "benchmark") pairs/s at n = 32 from 256^2 and 512^2 inputs, the achieved
  GB/s against the bytes of the two input images, and its share of the H100 SXM data sheet's 3.35 TB/s;
* SSIM's FP64 work: the window sums' DFMA per map value computed from the tile shape, and the achieved TFLOP/s;
* pytorch-ssim's formula in eager PyTorch (five depthwise cuDNN conv2d and the element-wise map, cuDNN defaults) with
  its error against a float64 run of the same formula on the same pairs, and this kernel's error against that run;
* per-kernel times from torch.profiler (CUDA activities, a run of its own);
* the evaluation step at migan-512, n = 32: EvalPipeline + LPIPS + two InceptionV3 calls + two statistics updates +
  SSIM + PSNR, images/s.

Records the card name and power limit of the same run.

    python tools/metrics_throughput.py [--steps 20] [--out tools/out/metrics_throughput.json]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import fid, lpips, metrics, synthetic  # noqa: E402
from fid_throughput import card, images, seeded_weights as inception_weights, timed  # noqa: E402
from lpips_throughput import pairs, seeded_weights as lpips_weights  # noqa: E402

N = 32
HBM_TBS = 3.35
WS = 11
TILE = 32


def eager_ssim(x, y, ws=WS):
    """pytorch-ssim's _ssim with the reference's window, in the inputs' dtype (per-image means)."""
    g = metrics.gaussian_taps(ws).to(x)
    w2 = g.unsqueeze(1).mm(g.unsqueeze(1).t())
    c = x.shape[1]
    win = w2.expand(c, 1, ws, ws).contiguous()

    def conv(t):
        return F.conv2d(t, win, padding=ws // 2, groups=c)

    mu1, mu2 = conv(x), conv(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(x * x) - mu1_sq, conv(y * y) - mu2_sq, conv(x * y) - mu1_mu2
    m = ((2 * mu1_mu2 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1_sq + mu2_sq + 0.01 ** 2) * (s1 + s2 + 0.03 ** 2))
    return m.mean(1).mean(1).mean(1)


def dfma_per_value(ws=WS):
    """Window-sum DFMA per map value: the horizontal pass over (TILE + ws - 1) rows and the vertical pass, 5 moments."""
    return 5 * ws * (TILE + (TILE + ws - 1)) / TILE


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "n": N}
    for size in (256, 512):
        x, y = (t.to(dev) for t in pairs(N, size, seed=size))
        nbytes = 2 * x.numel() * 4
        with torch.no_grad():
            want = eager_ssim(x.double(), y.double())
        row = {}
        t = timed(lambda: metrics.compute_ssim(x, y, size_average=False), a.steps)
        got = metrics.compute_ssim(x, y, size_average=False)
        values = x.numel()   # one map value per input pixel at an odd window
        row["ssim"] = {"pairs_per_s": N / t, "ms": t * 1e3, "GB_per_s": nbytes / t / 1e9,
                       "share_of_hbm": nbytes / t / 1e12 / HBM_TBS, "dfma_per_value": dfma_per_value(),
                       "fp64_tflops": 2 * values * dfma_per_value() / t / 1e12,
                       "err_vs_fp64": float((got.double() - want).abs().max())}
        with torch.no_grad():
            te = timed(lambda: eager_ssim(x, y), a.steps)
            ge = eager_ssim(x, y)
        row["ssim_torch_eager"] = {"pairs_per_s": N / te, "ms": te * 1e3, "err_vs_fp64": float((ge.double() - want).abs().max())}
        for label, (fd, sc) in (("psnr_none", (None, 2)), ("psnr_div2k", ("div2k", 2)), ("psnr_benchmark", ("benchmark", 2))):
            tp = timed(lambda: metrics.compute_psnr(x, y, fd, sc), a.steps)
            row[label] = {"pairs_per_s": N / tp, "ms": tp * 1e3, "GB_per_s": nbytes / tp / 1e9,
                          "share_of_hbm": nbytes / tp / 1e12 / HBM_TBS}
        res["metrics_%d" % size] = row
        print(json.dumps({"metrics_%d" % size: row}), flush=True)
    # per-kernel times at 512^2, n = 32
    x, y = (t.to(dev) for t in pairs(N, 512, seed=1))
    metrics.compute_ssim(x, y)
    metrics.compute_psnr(x, y)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            metrics.compute_ssim(x, y)
            metrics.compute_psnr(x, y, "benchmark", 2)
        torch.cuda.synchronize()
    per_k = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "metrics_" in e.name:
            name = e.name.split("metrics_", 1)[1].split("(")[0]
            per_k[name][0] += 1
            per_k[name][1] += e.device_time_total / 1e3
    res["per_kernel_ms_512_n32"] = {k: {"launches": v[0], "ms_each": v[1] / v[0]} for k, v in per_k.items()}
    print(json.dumps({"per_kernel_ms_512_n32": res["per_kernel_ms_512_n32"]}), flush=True)
    # the evaluation step at migan-512, n = 32
    pipe = migan_b200.EvalPipeline(synthetic.export_style_state_dict(512, seed=1), resolution=512, device=dev, seed=0)
    inception = fid.InceptionV3(weights=inception_weights(dev))
    net = lpips.LPIPS(net="alex", weights=lpips_weights()).to(dev)
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, size=(512, 512, 3), dtype=np.uint8) for _ in range(N)]
    s_r, s_c = fid.FeatureStatistics(device=dev), fid.FeatureStatistics(device=dev)
    values = []

    def step(with_metrics):
        real, composed = pipe.forward_batch(imgs)
        values.append(net(real, composed, normalize=True))
        s_r.add(inception(real)[0])
        s_c.add(inception(composed)[0])
        if with_metrics:
            values.append(metrics.compute_ssim(real, composed, size_average=False))
            values.append(metrics.compute_psnr(real, composed, None))

    for label, wm in (("eval_step_migan512_n32", True), ("eval_step_without_ssim_psnr", False)):
        t = timed(lambda: step(wm), max(3, a.steps // 4))
        res[label] = {"images_per_s": N / t, "ms": t * 1e3}
        values.clear()
    print(json.dumps({k: res[k] for k in ("eval_step_migan512_n32", "eval_step_without_ssim_psnr", "card")}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Throughput of the LPIPS distance and of the whole evaluation step on cuda:0, next to AlexNet-LPIPS in eager PyTorch on
the same card:

* LPIPS pairs/s at n = 32 from 256^2 and 512^2 inputs, and achieved TFLOP/s against the convolution MACs of both images
  of a pair, computed from the shapes (the three TF32 passes are not counted as extra work);
* torchvision AlexNet features[:12] with lpips 0.1's head in eager PyTorch, with cuDNN defaults (TF32 allowed, as the
  evaluation script runs today) and with TF32 off, each with its error against a float64 run on the same pairs;
* per-kernel times of one forward (torch.profiler, CUDA activities, a run of its own);
* the evaluation step at migan-512, n = 32: EvalPipeline + LPIPS + two InceptionV3 calls + two statistics updates,
  images/s.

Seeded random weights (He-scaled convolutions, bias 0.1 randn, lin{k} uniform in [0, 4 / C)); the eager network and its
float64 run are built here because tools/ do not import the test oracle.  Records the card name and power limit of the
same run.

    python tools/lpips_throughput.py [--steps 10] [--out tools/out/lpips_throughput.json]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch
import torch.nn.functional as F
from torchvision.models import alexnet

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import fid, lpips, synthetic  # noqa: E402
from fid_throughput import card, images, seeded_weights as inception_weights, timed  # noqa: E402

TAPS = (1, 4, 7, 9, 11)
N = 32


def seeded_weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    feats = alexnet(weights=None).features[:12]
    sd = {"scaling_layer.shift": torch.tensor(lpips.SHIFT).view(1, 3, 1, 1),
          "scaling_layer.scale": torch.tensor(lpips.SCALE).view(1, 3, 1, 1)}
    for ours, tv in lpips.TORCHVISION_KEYS.items():
        conv = feats[int(tv.split(".")[1])]
        sd[ours + ".weight"] = (torch.randn(conv.weight.shape, generator=g, dtype=torch.float64)
                                * (2.0 / conv.weight[0].numel()) ** 0.5).float()
        sd[ours + ".bias"] = (0.1 * torch.randn(conv.bias.shape, generator=g, dtype=torch.float64)).float()
    for k, c in enumerate(lpips.CHANNELS):
        sd["lin%d.model.1.weight" % k] = (torch.rand((1, c, 1, 1), generator=g, dtype=torch.float64) * 4 / c).float()
    return sd


class EagerLPIPS(torch.nn.Module):
    """lpips 0.1's LPIPS(net="alex") arithmetic on torchvision's AlexNet features[:12], in eager PyTorch."""

    def __init__(self, sd):
        super().__init__()
        self.features = alexnet(weights=None).features[:12]
        self.features.load_state_dict({tv.split(".")[1] + "." + leaf: sd[ours + "." + leaf]
                                       for ours, tv in lpips.TORCHVISION_KEYS.items() for leaf in ("weight", "bias")})
        self.register_buffer("shift", sd["scaling_layer.shift"].clone())
        self.register_buffer("scale", sd["scaling_layer.scale"].clone())
        for k in range(5):
            self.register_buffer("lin%d" % k, sd["lin%d.model.1.weight" % k].clone())

    def taps(self, x):
        out = []
        for i, layer in enumerate(self.features):
            x = layer(x)
            if i in TAPS:
                out.append(x.clone())
        return out

    def forward(self, a, b, normalize=True):
        if normalize:
            a, b = 2 * a - 1, 2 * b - 1
        fa, fb = self.taps((a - self.shift) / self.scale), self.taps((b - self.shift) / self.scale)
        per = []
        for k, (u, v) in enumerate(zip(fa, fb)):
            nu = u / (u.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            nv = v / (v.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            per.append(F.conv2d((nu - nv) ** 2, getattr(self, "lin%d" % k)).mean((2, 3)).view(-1))
        per = torch.stack(per)
        return per, per.sum(0)


def macs_per_image(h, w):
    """Multiply-adds of the five convolutions of features[:12] on one h x w image."""
    total, c = 0, 3
    for layer in ((11, 4, 2, 64), "pool", (5, 1, 2, 192), "pool", (3, 1, 1, 384), (3, 1, 1, 256), (3, 1, 1, 256)):
        if layer == "pool":
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
            continue
        k, s, p, cout = layer
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        total += h * w * cout * c * k * k
        c = cout
    return total


def pairs(n, size, seed):
    a = images(n, size, size, seed)
    b = a.clone()
    q = size // 4
    b[:, :, q:2 * q, size // 3:size // 3 + q] = images(n, size, size, seed + 1)[:, :, q:2 * q, size // 3:size // 3 + q]
    return a, b


def rel_err(per, tot, want_per, want):
    return {"per_layer": float(((per.double() - want_per).abs() / want_per).max()),
            "total": float(((tot.double() - want).abs() / want).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "n": N}
    sd = seeded_weights()
    net = lpips.LPIPS(net="alex", weights=sd).to(dev)
    ref = EagerLPIPS(sd).to(dev).eval()
    ref64 = EagerLPIPS(sd).double().to(dev).eval()
    for size in (256, 512):
        x0, x1 = (t.to(dev) for t in pairs(N, size, seed=size))
        with torch.no_grad():
            want_per, want = ref64(x0.double(), x1.double())
        gmac = 2 * macs_per_image(size, size) / 1e9   # both images of a pair
        t = timed(lambda: net(x0, x1, normalize=True), a.steps)
        val, per = net(x0, x1, retPerLayer=True, normalize=True)
        row = {"pairs_per_s": N / t, "ms": t * 1e3, "gmac_per_pair": gmac, "tflops": N * 2 * gmac * 1e9 / t / 1e12,
               "err_vs_fp64": rel_err(torch.stack([p.view(N) for p in per]), val.view(N), want_per, want)}
        for label, tf32 in (("torch_cudnn_default", True), ("torch_tf32_off", False)):
            old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32 and old[1]
            with torch.no_grad():
                tt = timed(lambda: ref(x0, x1), a.steps)
                p, v = ref(x0, x1)
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
            row[label] = {"pairs_per_s": N / tt, "ms": tt * 1e3, "tflops": N * 2 * gmac * 1e9 / tt / 1e12,
                          "err_vs_fp64": rel_err(p, v, want_per, want)}
        res["lpips_%d" % size] = row
        print(json.dumps({("lpips_%d" % size): row}), flush=True)
    # per-kernel times, one profiled forward at 512^2
    x0, x1 = (t.to(dev) for t in pairs(N, 512, seed=1))
    net(x0, x1, normalize=True)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        net(x0, x1, normalize=True)
        torch.cuda.synchronize()
    per_k = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            if "incep_conv" in e.name:
                name = "conv_tf32"
            elif "lpips_reduce" in e.name:
                name = "reduce"
            elif "ck_items_kernel" in e.name:
                name = e.name.split("::")[-1].split(">")[0]
            else:
                name = e.name
            per_k[name][0] += 1
            per_k[name][1] += e.device_time_total / 1e3   # ms
    res["per_kernel_ms_512_n32"] = {k: {"launches": v[0], "ms": v[1]} for k, v in sorted(per_k.items(), key=lambda kv: -kv[1][1])}
    print(json.dumps({"per_kernel_ms_512_n32": res["per_kernel_ms_512_n32"]}), flush=True)
    conv_events = [(e.device_time_total / 1e3) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA and "incep_conv" in e.name]
    res["conv_ms_512_n32_in_order"] = conv_events
    print(json.dumps({"conv_ms_512_n32_in_order": conv_events}), flush=True)
    # the evaluation step at migan-512, n = 32
    pipe = migan_b200.EvalPipeline(synthetic.export_style_state_dict(512, seed=1), resolution=512, device=dev, seed=0)
    inception = fid.InceptionV3(weights=inception_weights(dev))
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, size=(512, 512, 3), dtype=np.uint8) for _ in range(N)]
    s_r, s_c = fid.FeatureStatistics(device=dev), fid.FeatureStatistics(device=dev)
    values = []

    def step():
        real, composed = pipe.forward_batch(imgs)
        values.append(net(real, composed, normalize=True))
        s_r.add(inception(real)[0])
        s_c.add(inception(composed)[0])

    t = timed(step, max(2, a.steps // 2))
    res["eval_step_migan512_n32"] = {"images_per_s": N / t, "ms": t * 1e3}
    print(json.dumps({"eval_step_migan512_n32": res["eval_step_migan512_n32"], "card": res["card"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

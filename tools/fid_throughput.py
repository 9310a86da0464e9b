"""Throughput of the FID InceptionV3 features and of the evaluation step on cuda:0, next to torchvision's Inception3 in
eager PyTorch on the same card:

* InceptionV3 feature images/s at n = 32 from 256^2 and 512^2 inputs, and achieved TFLOP/s against 2 x 5.71 GMAC per
  image (the dense convolutions at 299 x 299; the three TF32 passes are not counted as extra work);
* per-kernel times of one forward (torch.profiler, CUDA activities, a run of its own);
* torchvision Inception3 (FID blocks, eager) with cuDNN defaults (TF32 allowed, as the evaluation script runs today) and
  with TF32 off, each with its feature error against the float64 oracle on the same images;
* the evaluation step at migan-512, n = 32: EvalPipeline + two feature calls + two statistics updates, images/s.

Seeded random weights, BatchNorm statistics calibrated on seeded images so every layer stays alive; the comparison
network and its float64 run (the "oracle" column) are torchvision's blocks with the FID pool variants, built here
because tools/ do not import the test oracle.  Records the card name and power limit of the same run.

    python tools/fid_throughput.py [--steps 10] [--out tools/out/fid_throughput.json]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import torch
import torch.nn.functional as F
from torchvision.models import inception as tvi

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import migan_b200  # noqa: E402
from migan_b200 import fid  # noqa: E402
from migan_b200 import synthetic  # noqa: E402

GMAC_PER_IMAGE = 5.71
BLOCKS = ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3", "maxpool2",
          "Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e", "Mixed_7a",
          "Mixed_7b", "Mixed_7c", "avgpool")


def _pool(x, kind):
    if kind == "max":
        return F.max_pool2d(x, 3, 1, 1)
    return F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)


class _A(tvi.InceptionA):
    def forward(self, x):
        return torch.cat([self.branch1x1(x), self.branch5x5_2(self.branch5x5_1(x)),
                          self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x))),
                          self.branch_pool(_pool(x, "avg"))], 1)


class _C(tvi.InceptionC):
    def forward(self, x):
        d = self.branch7x7dbl_1(x)
        for m in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            d = m(d)
        return torch.cat([self.branch1x1(x), self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x))), d,
                          self.branch_pool(_pool(x, "avg"))], 1)


class _E(tvi.InceptionE):
    def __init__(self, cin, kind):
        super().__init__(cin)
        self.kind = kind

    def forward(self, x):
        t = self.branch3x3_1(x)
        u = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        return torch.cat([self.branch1x1(x), self.branch3x3_2a(t), self.branch3x3_2b(t), self.branch3x3dbl_3a(u),
                          self.branch3x3dbl_3b(u), self.branch_pool(_pool(x, self.kind))], 1)


def eager_network():
    """torchvision Inception3 with the FID blocks (pytorch_fid's fid_inception_v3 structure)."""
    m = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False)
    for name, cin, pf in (("Mixed_5b", 192, 32), ("Mixed_5c", 256, 64), ("Mixed_5d", 288, 64)):
        setattr(m, name, _A(cin, pool_features=pf))
    for name, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        setattr(m, name, _C(768, channels_7x7=c7))
    m.Mixed_7b, m.Mixed_7c = _E(1280, "avg"), _E(2048, "max")
    return m.eval()


def eager_features(m, x):
    x = 2 * F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1
    for name in BLOCKS:
        x = getattr(m, name)(x)
    return x.flatten(1)


def _calibrate(bn, y):
    bn.running_mean.copy_(y.mean((0, 2, 3)))
    bn.running_var.copy_(y.var((0, 2, 3), unbiased=False))


def seeded_weights(dev, seed=0):
    """He-scaled convolutions, BN gamma in [0.5, 1.5], beta 0.1 randn, running statistics from one float64 pass."""
    g = torch.Generator().manual_seed(seed)
    m = eager_network().double().to(dev)
    for bc in (mod for mod in m.modules() if isinstance(mod, tvi.BasicConv2d)):
        w = bc.conv.weight
        with torch.no_grad():
            w.copy_(torch.randn(w.shape, generator=g, dtype=torch.float64) * (2.0 / w[0].numel()) ** 0.5)
            bc.bn.weight.copy_(0.5 + torch.rand(bc.bn.weight.shape, generator=g, dtype=torch.float64))
            bc.bn.bias.copy_(0.1 * torch.randn(bc.bn.bias.shape, generator=g, dtype=torch.float64))
        bc.conv.register_forward_hook(lambda mod, i, o, bn=bc.bn: _calibrate(bn, o))
    with torch.no_grad():
        eager_features(m, images(2, 128, 160, seed + 1).double().to(dev))
    return {k: v.float().cpu() for k, v in m.state_dict().items()}


def images(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.rand((n, 3, max(2, h // 16), max(2, w // 16)), generator=g)
    x = 0.8 * F.interpolate(low, size=(h, w), mode="bilinear", align_corners=False) + 0.2 * torch.rand((n, 3, h, w), generator=g)
    return x.clamp(0, 1)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn, steps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps / 1e3   # seconds per call


def rel_err(got, want):
    return float((got.double().cpu() - want).abs().max()) / max(float(want.abs().max()), 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "gmac_per_image": GMAC_PER_IMAGE, "n": 32}
    sd = seeded_weights(dev)
    net = fid.InceptionV3(weights=sd)
    ref = eager_network()
    ref.load_state_dict(sd)
    ref = ref.to(dev)
    oracle = eager_network()
    oracle.load_state_dict(sd)
    oracle = oracle.double().to(dev)
    for size in (256, 512):
        x = images(32, size, size, seed=size).to(dev)
        with torch.no_grad():
            want = eager_features(oracle, x[:4].double()).cpu()
        t = timed(lambda: net(x), a.steps)
        row = {"images_per_s": 32 / t, "tflops": 32 * 2 * GMAC_PER_IMAGE * 1e9 / t / 1e12,
               "err_vs_fp64": rel_err(net(x[:4])[0].view(4, 2048), want)}
        for label, tf32 in (("torch_cudnn_default", True), ("torch_tf32_off", False)):
            old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32 and old[1]
            with torch.no_grad():
                tt = timed(lambda: eager_features(ref, x), a.steps)
                e = rel_err(eager_features(ref, x[:4]), want)
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
            row[label] = {"images_per_s": 32 / tt, "tflops": 32 * 2 * GMAC_PER_IMAGE * 1e9 / tt / 1e12, "err_vs_fp64": e}
        res["features_%d" % size] = row
        print(json.dumps({("features_%d" % size): row}), flush=True)
    # per-kernel times, one profiled forward at 512^2
    x = images(32, 512, 512, seed=1).to(dev)
    net(x)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        net(x)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = "conv_tf32" if "incep_conv" in e.name else e.name.split("incep::")[-1].split(">")[0] if "incep::" in e.name else e.name
            per[name][0] += 1
            per[name][1] += e.device_time_total / 1e3   # ms
    res["per_kernel_ms_512_n32"] = {k: {"launches": v[0], "ms": v[1]} for k, v in sorted(per.items(), key=lambda kv: -kv[1][1])}
    print(json.dumps({"per_kernel_ms_512_n32": res["per_kernel_ms_512_n32"]}), flush=True)
    # the evaluation step at migan-512, n = 32
    pipe = migan_b200.EvalPipeline(synthetic.export_style_state_dict(512, seed=1), resolution=512, device=dev, seed=0)
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, size=(512, 512, 3), dtype=np.uint8) for _ in range(32)]
    s_r, s_c = fid.FeatureStatistics(device=dev), fid.FeatureStatistics(device=dev)

    def step():
        real, composed = pipe.forward_batch(imgs)
        s_r.add(net(real)[0])
        s_c.add(net(composed)[0])

    t = timed(step, max(2, a.steps // 2))
    res["eval_step_migan512_n32"] = {"images_per_s": 32 / t, "ms": t * 1e3}
    print(json.dumps({"eval_step_migan512_n32": res["eval_step_migan512_n32"], "card": res["card"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

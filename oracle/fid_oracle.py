"""CPU float64 oracle of the FID evaluation: pytorch_fid's InceptionV3([3]) features and the Frechet distance.

pytorch_fid is not a dependency of this project, so the network is restated here on torchvision's `Inception3`
(`fid_inception_v3()`): 1008 classes, no aux logits, and four block types replaced -- Mixed_5b..5d (InceptionA), 6b..6e
(InceptionC) and 7b (InceptionE) average their branch_pool with count_include_pad=False, Mixed_7c (InceptionE) max-pools
it (3 x 3, stride 1, padding 1).  Input stage: bilinear resize to 299 x 299 (align_corners=False, no antialias), 2x - 1.
Everything else is torchvision's own module.  The statistics are numpy's np.mean / np.cov(rowvar=False) and the
distance scipy's sqrtm, as evaluate_fid_lpips.py computes them through pytorch_fid.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F
from scipy import linalg
from torchvision.models import inception as tvi

SIZE = 299
DIM = 2048


def _avg_pool(x):
    return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)


class FIDInceptionA(tvi.InceptionA):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(_avg_pool(x))
        return torch.cat([b1, b5, b3, bp], 1)


class FIDInceptionC(tvi.InceptionC):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = self.branch7x7dbl_1(x)
        for m in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            bd = m(bd)
        bp = self.branch_pool(_avg_pool(x))
        return torch.cat([b1, b7, bd, bp], 1)


class FIDInceptionE(tvi.InceptionE):
    """pool="avg": Mixed_7b (FIDInceptionE_1); pool="max": Mixed_7c (FIDInceptionE_2)."""

    def __init__(self, in_channels, pool):
        super().__init__(in_channels)
        self.pool = pool

    def forward(self, x):
        b1 = self.branch1x1(x)
        t = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(t), self.branch3x3_2b(t)], 1)
        t = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(t), self.branch3x3dbl_3b(t)], 1)
        p = _avg_pool(x) if self.pool == "avg" else F.max_pool2d(x, kernel_size=3, stride=1, padding=1)
        return torch.cat([b1, b3, bd, self.branch_pool(p)], 1)


def stock_inception() -> tvi.Inception3:
    """torchvision's module at the FID configuration's shape (the key list and shapes the weight file has)."""
    return tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False)


def fid_inception() -> tvi.Inception3:
    m = stock_inception()
    m.Mixed_5b = FIDInceptionA(192, pool_features=32)
    m.Mixed_5c = FIDInceptionA(256, pool_features=64)
    m.Mixed_5d = FIDInceptionA(288, pool_features=64)
    m.Mixed_6b = FIDInceptionC(768, channels_7x7=128)
    m.Mixed_6c = FIDInceptionC(768, channels_7x7=160)
    m.Mixed_6d = FIDInceptionC(768, channels_7x7=160)
    m.Mixed_6e = FIDInceptionC(768, channels_7x7=192)
    m.Mixed_7b = FIDInceptionE(1280, "avg")
    m.Mixed_7c = FIDInceptionE(2048, "max")
    return m


def input_stage(x: torch.Tensor) -> torch.Tensor:
    x = F.interpolate(x, size=(SIZE, SIZE), mode="bilinear", align_corners=False)
    return 2 * x - 1


def blocks(m: tvi.Inception3, x: torch.Tensor) -> torch.Tensor:
    """pytorch_fid's blocks 0..3 after the input stage: [n, 2048, 1, 1]."""
    for name in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3",
                 "maxpool2", "Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d",
                 "Mixed_6e", "Mixed_7a", "Mixed_7b", "Mixed_7c", "avgpool"):
        x = getattr(m, name)(x)
    return x


def model(state_dict) -> tvi.Inception3:
    m = fid_inception()
    m.load_state_dict(state_dict)
    return m.double().eval()


@torch.no_grad()
def features(state_dict_or_model, x: torch.Tensor) -> torch.Tensor:
    """[n, 2048] float64 pool3 features of x [n, 3, H, W] in [0, 1]."""
    m = state_dict_or_model if isinstance(state_dict_or_model, torch.nn.Module) else model(state_dict_or_model)
    return blocks(m, input_stage(x.double())).flatten(1)


def seeded_state_dict(seed: int = 0, calib_images: int = 2) -> dict:
    """Weights that keep all 94 layers numerically alive: He-scaled conv weights, BN gamma in [0.5, 1.5], beta =
    0.1 randn, and running mean / variance calibrated by one pass over seeded images, so every pre-activation has about
    unit scale while running_var != 1 (the BatchNorm fold matters)."""
    g = torch.Generator().manual_seed(seed)
    m = fid_inception().double().eval()
    convs = [mod for mod in m.modules() if isinstance(mod, tvi.BasicConv2d)]
    for bc in convs:
        w = bc.conv.weight
        fan_in = w.shape[1] * w.shape[2] * w.shape[3]
        with torch.no_grad():
            w.copy_(torch.randn(w.shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5)
            bc.bn.weight.copy_(0.5 + torch.rand(bc.bn.weight.shape, generator=g, dtype=torch.float64))
            bc.bn.bias.copy_(0.1 * torch.randn(bc.bn.bias.shape, generator=g, dtype=torch.float64))
    stats = {}

    def hook(mod, inp, out):
        y = out.detach()
        mean = y.mean(dim=(0, 2, 3))
        var = y.var(dim=(0, 2, 3), unbiased=False)
        mod.running_mean.copy_(mean)
        mod.running_var.copy_(var)
        stats[mod] = True

    hooks = [bc.conv.register_forward_hook(lambda mod, i, o, bn=bc.bn: hook(bn, i, o)) for bc in convs]
    x = make_images(calib_images, 128, 160, seed=seed + 1)
    with torch.no_grad():
        blocks(m, input_stage(x.double()))   # calibrated layer by layer: each BN is set before the next layer runs
    for h in hooks:
        h.remove()
    assert len(stats) == len(convs)
    sd = m.float().state_dict()
    sd["fc.weight"] = torch.randn(sd["fc.weight"].shape, generator=g) * 0.01
    sd["fc.bias"] = torch.zeros(sd["fc.bias"].shape)
    return sd


def make_images(n: int, h: int, w: int, seed: int = 0) -> torch.Tensor:
    """Seeded float32 images in [0, 1] with spatial structure (smooth blobs plus noise)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand((n, 3, max(2, h // 16), max(2, w // 16)), generator=g)
    x = F.interpolate(low, size=(h, w), mode="bilinear", align_corners=False)
    x = 0.8 * x + 0.2 * torch.rand((n, 3, h, w), generator=g)
    return x.clamp(0, 1).float()


# ---- statistics and distance (pytorch_fid.fid_score) ----------------------------------------------------------------
def statistics(feats: np.ndarray):
    feats = np.asarray(feats, dtype=np.float64)
    return np.mean(feats, axis=0), np.cov(feats, rowvar=False)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))

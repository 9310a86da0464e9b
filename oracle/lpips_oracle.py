"""CPU float64 oracle of the LPIPS distance: lpips 0.1's `LPIPS(net="alex")` as evaluate_fid_lpips.py calls it.

lpips is not a dependency of this project, so the distance is restated here on torchvision's `alexnet().features[:12]`:
the ScalingLayer ((x - shift) / scale, after 2x - 1 with `normalize`), the five ReLU outputs (features 1, 4, 7, 9, 11),
each normalised per pixel by (its L2 norm over the channels + 1e-10), the squared difference, the 1 x 1 `lin{k}`
without bias (dropout is the identity in eval), the spatial mean, and the sum over the five layers.  The state_dict
layout is lpips 0.1's: `scaling_layer.shift` / `.scale`, `net.slice{1..5}.{0,3,6,8,10}.weight` / `.bias` (torchvision's
`features.{0,3,6,8,10}`) and `lin{0..4}.model.1.weight`.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torchvision.models import alexnet

from .fid_oracle import make_images

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CHANNELS = (64, 192, 384, 256, 256)
TAPS = (1, 4, 7, 9, 11)   # the ReLUs of features[:12] whose outputs LPIPS compares
LPIPS_TO_TORCHVISION = {"net.slice1.0": "features.0", "net.slice2.3": "features.3", "net.slice3.6": "features.6",
                        "net.slice4.8": "features.8", "net.slice5.10": "features.10"}


def alexnet_features() -> torch.nn.Sequential:
    return alexnet(weights=None).features[:12]


def seeded_state_dict(seed: int = 0) -> dict:
    """LPIPS-layout weights: He-scaled convolutions, bias 0.1 randn, lin{k} uniform in [0, 4 / C), the ScalingLayer's
    constants.  float32, as a state_dict would hold them."""
    g = torch.Generator().manual_seed(seed)
    sd = {"scaling_layer.shift": torch.tensor(SHIFT).view(1, 3, 1, 1),
          "scaling_layer.scale": torch.tensor(SCALE).view(1, 3, 1, 1)}
    feats = alexnet_features()
    for ours, tv in LPIPS_TO_TORCHVISION.items():
        conv = feats[int(tv.split(".")[1])]
        w = conv.weight
        sd[ours + ".weight"] = torch.randn(w.shape, generator=g, dtype=torch.float64).mul((2.0 / w[0].numel()) ** 0.5).float()
        sd[ours + ".bias"] = (0.1 * torch.randn(conv.bias.shape, generator=g, dtype=torch.float64)).float()
    for k, c in enumerate(CHANNELS):
        sd["lin%d.model.1.weight" % k] = (torch.rand((1, c, 1, 1), generator=g, dtype=torch.float64) * 4 / c).float()
    return sd


def model(sd: dict) -> torch.nn.Sequential:
    """torchvision's features[:12] in float64 with the LPIPS state_dict's convolutions loaded."""
    m = alexnet_features()
    m.load_state_dict({tv.split(".")[1] + "." + leaf: sd[ours + "." + leaf] for ours, tv in LPIPS_TO_TORCHVISION.items()
                       for leaf in ("weight", "bias")})
    return m.double().eval()


@torch.no_grad()
def taps(m: torch.nn.Sequential, x: torch.Tensor) -> list:
    out = []
    for i, layer in enumerate(m):
        x = layer(x)
        if i in TAPS:
            out.append(x.clone())
    return out


@torch.no_grad()
def distance(sd: dict, in0: torch.Tensor, in1: torch.Tensor, normalize: bool = False, m=None):
    """(per_layer [5, n], total [n]) float64 LPIPS of the pairs (in0[i], in1[i]), in0, in1 [n, 3, H, W], on their device
    (`m`: model(sd) on that device)."""
    m = model(sd) if m is None else m
    x0, x1 = in0.double(), in1.double()
    shift = sd["scaling_layer.shift"].to(x0)
    scale = sd["scaling_layer.scale"].to(x0)
    if normalize:
        x0, x1 = 2 * x0 - 1, 2 * x1 - 1
    f0, f1 = taps(m, (x0 - shift) / scale), taps(m, (x1 - shift) / scale)
    per = []
    for k, (a, b) in enumerate(zip(f0, f1)):
        na = a / (a.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        nb = b / (b.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        d = F.conv2d((na - nb) ** 2, sd["lin%d.model.1.weight" % k].to(x0))
        per.append(d.mean((2, 3)).view(-1))
    per = torch.stack(per)
    return per, per.sum(0)


def composed(x: torch.Tensor, seed: int = 0) -> torch.Tensor:
    """A copy of x [n, 3, H, W] with a rectangle (a quarter of each side, off-centre) replaced by other structured
    content: the 'composed' image of an inpainting evaluation."""
    n, _, h, w = x.shape
    y = x.clone()
    other = make_images(n, h, w, seed=seed)
    y0, x0 = h // 4, w // 3
    y[:, :, y0:y0 + max(1, h // 4), x0:x0 + max(1, w // 4)] = other[:, :, y0:y0 + max(1, h // 4), x0:x0 + max(1, w // 4)]
    return y

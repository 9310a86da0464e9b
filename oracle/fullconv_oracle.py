"""CPU oracle of the fully convolutional generator forward: any H x W that is a multiple of R/4 and at least R.
TEST INFRASTRUCTURE ONLY (same rules as oracle/migan_oracle.py, whose forward it reuses).

The reference README ("Quick Test") says the network is fully convolutional once `filter_const` and `noise_const` are
made dynamic.  Here they are rebuilt from the input's shape:

* every `Upsample2d.filter_const` is the zero-insertion pattern at its block's output extent,
* every `noise_const` is its r x r plane tiled over the layer's extent: noise[i, j] = noise_const[i mod r, j mod r],

where the nominal level r runs at (H r / R, W r / R).  At H = W = R this is `migan_oracle.generator_forward`.
Parity pin: tests/golden/make_golden_fullconv.py applies the same two replacements to the reference's own module tree,
runs its forward and asserts equality with `generator_forward_fc`.
"""
from collections import OrderedDict
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import migan_oracle as O


def make_input_hw(resolution: int, n: int, H: int, W: int, seed: int = 1234, *, hole: float = 0.4) -> torch.Tensor:
    """`migan_oracle.make_input` at an H x W extent: the same convention and 8 x 8 hole cells."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(n, 3, H, W, generator=g) * 2 - 1
    coarse = (torch.rand(n, 1, max(H // 8, 1), max(W // 8, 1), generator=g) > hole).float()
    mask = F.interpolate(coarse, size=(H, W), mode="nearest")
    return torch.cat([mask - 0.5, img * mask], dim=1).contiguous()


def fullconv_shape_error(resolution: int, n: int, H: int, W: int) -> Optional[str]:
    """None if an n x H x W input is accepted, else why not.  H, W >= R and multiples of R/4 (every level's extent is an
    integer and at least its side); the largest activation n*H*W*ch(R) must stay below 2^31 elements."""
    R, q = resolution, resolution // 4
    if H < R or W < R or H % q or W % q:
        return "H and W must be multiples of %d and at least %d" % (q, R)
    if n * H * W * O.channels(R) > 2 ** 31 - 1:
        return "the largest activation has more than 2^31 - 1 elements"
    return None


def zero_insertion(h: int, w: int) -> torch.Tensor:
    """Upsample2d.filter_const at an h x w output extent (migan_inference.py:83-85 at (h, w))."""
    f = torch.zeros(1, 1, h, w)
    f[:, :, ::2, ::2] = 1
    return f


def tiled_noise(noise_const: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """noise[i, j] = noise_const[i mod r, j mod r] over h x w."""
    r = noise_const.shape[-1]
    return noise_const.repeat((h + r - 1) // r, (w + r - 1) // r)[:h, :w].contiguous()


def fullconv_state_dict(sd: Dict[str, torch.Tensor], resolution: int, H: int, W: int) -> "OrderedDict[str, torch.Tensor]":
    """sd with the two size-dependent buffers rebuilt for an H x W input.  At H = W = R the values are sd's own."""
    out = OrderedDict()
    for k, v in sd.items():
        if k.endswith("filter_const"):
            r = v.shape[-1]
            v = zero_insertion(H * r // resolution, W * r // resolution)
        elif k.endswith("noise_const"):
            r = v.shape[-1]
            v = tiled_noise(v, H * r // resolution, W * r // resolution)
        out[k] = v
    return out


@torch.no_grad()
def generator_forward_fc(sd: Dict[str, torch.Tensor], x: torch.Tensor, resolution: int,
                         taps: Optional[dict] = None, dtype=torch.float32) -> torch.Tensor:
    """Fully convolutional Generator.forward: x[N,4,H,W] -> img[N,3,H,W], with the level extents, zero-insertion
    patterns and tiled noise built from x's shape.  Equals `migan_oracle.generator_forward` at H = W = R."""
    if x.dim() != 4 or x.shape[1] != 4:
        raise ValueError("expected x of shape [N,4,H,W], got %s" % (tuple(x.shape),))
    n, _, H, W = x.shape
    err = fullconv_shape_error(resolution, n, H, W)
    if err:
        raise ValueError("%d x %d is not a valid size for resolution %d: %s" % (H, W, resolution, err))
    sd = fullconv_state_dict(sd, resolution, H, W)
    if dtype != torch.float32:
        sd = {k: v.to(dtype) for k, v in sd.items()}
        x = x.to(dtype)
    x4, feats = O.encoder_forward(sd, x, resolution, taps)
    if taps is not None:
        for r, f in feats.items():
            taps["feat%d" % r] = f
    return O.synthesis_forward(sd, x4, feats, resolution, taps)


def fixture_rows(n: int, period: int = 8):
    """Rows of an output kept in a fixture: r % period in {0, 1} (both phases of every 2x resampling) and the last two
    rows (the bottom edge, where tiles are partial).  tests/golden/fullconv.npz uses period 8; tests/golden/fir.npz uses
    16, which keeps its four cases near 500 KB."""
    r = torch.arange(n)
    return r[(r % period < 2) | (r >= n - 2)]

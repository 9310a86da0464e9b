"""CPU oracle of the full-resolution request path (mi-gan_b200/csrc/fullres.cu, migan_b200.fullres).  TEST INFRASTRUCTURE
ONLY (same rules as oracle/migan_oracle.py).

For a photo uint8 [H,W,3] of any size and a mask of the same H x W ([H,W] or [H,W,C], C in 1..4):

1. known = read_mask's per-pixel steps without its resize: the channel (alpha of LA / RGBA, R of RGB, L itself), 255 - v
   if invert, then v < 255 -> 0; known where the result is 255.
2. (Hp, Wp) = (max(R, q ceil(H / q)), max(R, q ceil(W / q))), q = R / 4.
3. photo and known-mask padded on the bottom and right with np.pad(mode="reflect").
4. x = prepost_oracle.preprocess of the padded pair; after the generator, prepost_oracle.postprocess cropped to H x W.
"""
import numpy as np
import torch

from . import prepost_oracle as P


def known_mask(mask: np.ndarray, invert: bool) -> np.ndarray:
    """uint8 [H,W]: 255 where the pixel is known, 0 in the hole."""
    m = mask if mask.ndim == 2 else mask[..., {1: 0, 2: 1, 3: 0, 4: 3}[mask.shape[2]]]
    if invert:
        m = 255 - m
    return np.where(m == 255, 255, 0).astype(np.uint8)


def extent(H: int, W: int, R: int):
    q = R // 4
    return max(R, -(-H // q) * q), max(R, -(-W // q) * q)


def pad(img: np.ndarray, known: np.ndarray, Hp: int, Wp: int):
    """Photo [Hp,Wp,3] and known-mask [Hp,Wp] reflected on the bottom and right."""
    H, W = known.shape
    return (np.pad(img, ((0, Hp - H), (0, Wp - W), (0, 0)), mode="reflect"),
            np.pad(known, ((0, Hp - H), (0, Wp - W)), mode="reflect"))


def preprocess(img: np.ndarray, mask: np.ndarray, invert: bool, R: int) -> torch.Tensor:
    """x [1,4,Hp,Wp] of one request."""
    H, W = img.shape[:2]
    pi, pm = pad(img, known_mask(mask, invert), *extent(H, W, R))
    return P.preprocess(pi[None], pm[None])


def postprocess(y: torch.Tensor, img: np.ndarray, mask: np.ndarray, invert: bool) -> np.ndarray:
    """The composed uint8 [H,W,3] from y [1,3,Hp,Wp] (or [3,Hp,Wp])."""
    H, W = img.shape[:2]
    y = y.reshape(1, 3, y.shape[-2], y.shape[-1])[:, :, :H, :W]
    return P.postprocess(y, img[None], known_mask(mask, invert)[None])[0]

"""`EvalPipeline`: the evaluation batch of scripts/evaluate_fid_lpips.py around the generator, on the GPU;
`ResultsPipeline`: the same batch around another method's result images.

    pipe = EvalPipeline(state_dict_or_generator, resolution=512, seed=0)
    real, composed = pipe.forward_batch(imgs)              # generated masks: RandomMask after np.random.seed(seed)
    real, composed = pipe.forward_batch(imgs, masks)       # masks read from --mask-dir
    real, composed = ResultsPipeline(512).forward_batch(imgs, results, masks)   # results in place of the generator
    real, composed, hole = pipe.forward_batch(imgs, masks, hole_fraction=True)   # and each R x R mask's hole share

`imgs[i]` is `np.array(Image.open(p).convert("RGB"))` of any size (uint8 [H, W, 3]); `masks[i]` is
`np.array(Image.open(mask_path).convert("L"))` (uint8 [Hm, Wm]).  `real` and `composed` are CUDA float32 [n, 3, R, R]:
the script's `imgs` and `composed_imgs` after :248-249, the tensors it hands to LPIPS and InceptionV3, bit for bit:

* `InferenceDataset.__getitem__`: the photo through PIL BICUBIC to R x R when it is not that size, the mask through PIL
  NEAREST to R x R, `mask // 255`, x = cat(mask - 0.5, (v * 2 / 255 - 1) * mask);
* :244-249: y = model(x), composed = masks * imgs + (1 - masks) * y, then (v * 0.5 + 0.5).clamp(0, 1) of both.

Per pass of up to 32 images (csrc/demo_resize.cu behind include/migan_b200.h): the demo path's stages on the evaluation
layout -- tables, [PIL BICUBIC width and height passes, when a photo of the pass is not R x R], R x R + mask + x -- then
`Generator.forward` (`ResultsPipeline`: the same preprocess stage on the results, under the same masks), then one
composite launch.  Generated masks come from `RandomMaskStream` in call order, so images
fed in sorted-path order get the masks `generate_masks` writes for those paths.  There is no CPU path.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi
from .demo import GENERATOR_BATCH
from ._request_path import NoiseSeeds, _to, load_generator
from .masks import RandomMaskStream


class _EvalBatch(torch.nn.Module):
    """The evaluation batch without its fill-in: the input checks, the mask stream and the per-pass loop that every
    source of the composite's fill-in (a generator, or a method's result images) shares."""

    def __init__(self, resolution: int, device: Union[str, torch.device] = "cuda", seed: int = 0,
                 hole_range: Tuple[float, float] = (0.0, 1.0)):
        super().__init__()
        self.res = int(resolution)
        self.device_ = torch.device(device)
        if self.device_.type != "cuda":
            raise RuntimeError("migan_b200.%s runs on a CUDA device (there is no CPU path); got %s"
                               % (type(self).__name__, self.device_))
        self.masks = RandomMaskStream(self.res, seed=seed, device=self.device_, hole_range=hole_range)
        self.last_launches = []                 # kernel launches of each pass of the last call, fill-in included

    @staticmethod
    def preprocess_launches(resized: bool) -> int:
        """Launches of one `b200_eval_preprocess`: tables, [two resize passes when an image is not R x R], R x R + x."""
        return 2 + (2 if resized else 0)

    @classmethod
    def pass_launches(cls, resized: bool, generator: int) -> int:
        """Launches of one pass: the photos' preprocess, the fill-in's (`generator`: the generator's, summed over the
        pass's generator chunks, Co-Mod-GAN noise launches included; or the results' preprocess), the composite."""
        return cls.preprocess_launches(resized) + generator + 1

    def _check(self, i, img, mask, what="image"):
        img = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
        if not isinstance(img, torch.Tensor) or img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 \
                or min(img.shape[:2]) < 1:
            raise ValueError("%s: %s %d must be uint8 [H, W, 3]" % (type(self).__name__, what, i))
        if mask is not None:
            mask = torch.from_numpy(np.ascontiguousarray(mask)) if isinstance(mask, np.ndarray) else mask
            if not isinstance(mask, torch.Tensor) or mask.dtype != torch.uint8 or mask.dim() != 2 or min(mask.shape) < 1:
                raise ValueError("%s: mask %d must be uint8 [Hm, Wm] (mode L)" % (type(self).__name__, i))
        return img, mask

    @staticmethod
    def _preprocess(lib, imgs_d, masks_d, x, img, stream, keep) -> bool:
        """`b200_eval_preprocess` of one pass: x [k, 4, R, R] and img (v * 2 / 255 - 1, [k, 3, R, R]) of the photos
        `imgs_d` under `masks_d`, the scratch sized for these very requests.  True when a photo was resized."""
        k, R = len(imgs_d), x.shape[-1]
        reqs = (_abi.DemoRequest * k)()
        resized = False
        for r, im, m in zip(reqs, imgs_d, masks_d):
            r.img, r.H, r.W = im.data_ptr(), int(im.shape[0]), int(im.shape[1])
            r.mask, r.Hm, r.Wm, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), 1
            resized |= (r.H, r.W) != (R, R)
        need = int(lib.b200_eval_scratch_bytes(reqs, k, R))
        if need == 0:
            _abi.check(_abi.ERR_INVALID)
        scratch = torch.empty(need, dtype=torch.uint8, device=x.device)
        _abi.check(lib.b200_eval_preprocess(reqs, k, R, x.data_ptr(), img.data_ptr(), scratch.data_ptr(), need, stream))
        keep.append(scratch)
        return resized

    def _passes(self, imgs: Sequence, masks: Optional[Sequence], fill_in, fills: Optional[Sequence] = None,
                hole_fraction: bool = False):
        """(real, composed) of the photos `imgs`: per pass of up to PIPE_MAX_BATCH photos, the photos' preprocess, then
        `fill_in(c, k, x, fills_d, masks_d, stream, keep) -> (y, launches)` gives the fill-in y [k, 3, R, R] of photos
        c .. c+k (v * 2 / 255 - 1), then the composite.  `fills`: per-photo uint8 [H, W, 3] inputs of the fill-in,
        checked as the photos are and handed to `fill_in` on the device as `fills_d` (None without them).
        `hole_fraction`: also return CUDA float32 [n], 1 - mean of each R x R mask the composite used (x channel 0 is
        mask - 0.5), computed on the current stream."""
        imgs = list(imgs)
        n, R, dev = len(imgs), self.res, self.device_
        name = type(self).__name__
        if masks is not None and len(masks) != n:
            raise ValueError("%s.forward_batch: %d images and %d masks" % (name, n, len(masks)))
        if fills is not None and len(fills) != n:
            raise ValueError("%s.forward_batch: %d images and %d results" % (name, n, len(fills)))
        checked = [self._check(i, img, None if masks is None else masks[i]) for i, img in enumerate(imgs)]
        fills = None if fills is None else [self._check(i, f, None, "result")[0] for i, f in enumerate(fills)]
        real = torch.empty((n, 3, R, R), dtype=torch.float32, device=dev)
        composed = torch.empty((n, 3, R, R), dtype=torch.float32, device=dev)
        holes = torch.empty(n, dtype=torch.float32, device=dev) if hole_fraction else None
        out = (real, composed) if holes is None else (real, composed, holes)
        if n == 0:
            return out
        with torch.cuda.device(dev):
            imgs_d = [_to(img, dev, False) for img, _ in checked]
            fills_d = None if fills is None else [_to(f, dev, False) for f in fills]
            if masks is None:
                generated = self.masks.next(n)
                masks_d = [generated[i] for i in range(n)]
            else:
                masks_d = [_to(m, dev, False) for _, m in checked]
            lib = _abi.load()
            stream = torch.cuda.current_stream(dev).cuda_stream
            self.last_launches = []
            keep = []
            for c in range(0, n, _abi.PIPE_MAX_BATCH):
                k = min(_abi.PIPE_MAX_BATCH, n - c)
                x = torch.empty((k, 4, R, R), dtype=torch.float32, device=dev)
                resized = self._preprocess(lib, imgs_d[c:c + k], masks_d[c:c + k], x, real[c], stream, keep)
                y, fill_launches = fill_in(c, k, x, None if fills_d is None else fills_d[c:c + k], masks_d[c:c + k],
                                           stream, keep)
                _abi.check(lib.b200_eval_composite(x.data_ptr(), y.data_ptr(), k, R, real[c].data_ptr(),
                                                   composed[c].data_ptr(), stream))
                if holes is not None:
                    holes[c:c + k] = 1 - (x[:, 0] + 0.5).mean((1, 2))
                keep.append((x, y))
                self.last_launches.append(self.pass_launches(resized, fill_launches))
            torch.cuda.current_stream(dev).synchronize()   # the inputs and the pass buffers are freed on return
        return out


class EvalPipeline(_EvalBatch):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from; or a
    `migan_b200.comodgan.Generator` of the same resolution (see `comodgan.load`).  `seed`: the script's np.random.seed,
    and `hole_range` RandomMask's, for the generated masks.  Co-Mod-GAN draws its noise planes and z from seeded streams
    on the device: the k-th image processed gets seed `noise_seed * 2**32 + k` (`noise_index` = k) unless
    `forward_batch(..., seeds=...)` names them, and the generator runs in chunks of at most `generator_batch`."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda", seed: int = 0, *,
                 noise_seed: int = 0, generator_batch: int = GENERATOR_BATCH,
                 hole_range: Tuple[float, float] = (0.0, 1.0)):
        model = load_generator(self, model_or_state_dict, resolution, device, accept_comodgan=True)
        super().__init__(resolution, device, seed, hole_range)
        self.model = model
        self.noise = NoiseSeeds(self.model, noise_seed, generator_batch)

    @property
    def noise_index(self) -> int:
        """How many images have drawn their Co-Mod-GAN noise from the pipeline's counter; settable."""
        return self.noise.noise_index

    @noise_index.setter
    def noise_index(self, k: int) -> None:
        self.noise.noise_index = int(k)

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Optional[Sequence] = None, seeds=None, *,
                      hole_fraction: bool = False) -> Tuple[torch.Tensor, ...]:
        """(real, composed), CUDA float32 [n, 3, R, R] each.  masks=None takes the next n generated masks.  seeds
        (Co-Mod-GAN only, else ValueError): one 64-bit noise seed per image instead of the pipeline's counter.
        hole_fraction=True adds a third tensor, CUDA float32 [n]: the share of hole pixels in each R x R mask."""
        imgs = list(imgs)
        seeds = self.noise.take("EvalPipeline", len(imgs), seeds)

        def generate(c, k, x, fills_d, masks_d, stream, keep):
            return self.noise.run(self.model, x, None if seeds is None else seeds[c:c + k])
        return self._passes(imgs, masks, generate, hole_fraction=hole_fraction)


class ResultsPipeline(_EvalBatch):
    """The evaluation batch around another method's results: `forward_batch(imgs, results, masks)` is
    `EvalPipeline.forward_batch(imgs, masks)` with `results[i]` in place of the generator's output for photo i.

    `results[i]` is `np.array(Image.open(r).convert("RGB"))` of any size (uint8 [H, W, 3]).  It goes through the
    photo's own stage -- PIL BICUBIC to R x R when it is not that size, v * 2 / 255 - 1 -- and takes the place of
    `output_imgs` in :244-249: composed = masks * imgs + (1 - masks) * result, then (v * 0.5 + 0.5).clamp(0, 1) of both.
    The composite always runs, as in the script; a result that the method already composited under the same mask comes
    out unchanged.  `ResultsPipeline(resolution, device="cuda", seed=0, hole_range=(0.0, 1.0))`; `seed`: the script's
    np.random.seed, and `hole_range` RandomMask's, for the generated masks."""

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, results: Sequence, masks: Optional[Sequence] = None, *,
                      hole_fraction: bool = False) -> Tuple[torch.Tensor, ...]:
        """(real, composed), CUDA float32 [n, 3, R, R] each.  masks=None takes the next n generated masks.
        hole_fraction=True adds a third tensor, CUDA float32 [n]: the share of hole pixels in each R x R mask."""
        R = self.res

        def resize(c, k, x, fills_d, masks_d, stream, keep):
            # the photos' stage on the results, under the same masks: its img output is the result's v * 2 / 255 - 1
            # at R x R; its x output is not used
            y = torch.empty((k, 3, R, R), dtype=torch.float32, device=self.device_)
            x_unused = torch.empty_like(x)
            resized = self._preprocess(_abi.load(), fills_d, masks_d, x_unused, y, stream, keep)
            keep.append(x_unused)
            return y, self.preprocess_launches(resized)
        return self._passes(imgs, masks, resize, results, hole_fraction)

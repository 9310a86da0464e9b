"""`EvalPipeline`: the evaluation batch of scripts/evaluate_fid_lpips.py around the generator, on the GPU.

    pipe = EvalPipeline(state_dict_or_generator, resolution=512, seed=0)
    real, composed = pipe.forward_batch(imgs)              # generated masks: RandomMask after np.random.seed(seed)
    real, composed = pipe.forward_batch(imgs, masks)       # masks read from --mask-dir

`imgs[i]` is `np.array(Image.open(p).convert("RGB"))` of any size (uint8 [H, W, 3]); `masks[i]` is
`np.array(Image.open(mask_path).convert("L"))` (uint8 [Hm, Wm]).  `real` and `composed` are CUDA float32 [n, 3, R, R]:
the script's `imgs` and `composed_imgs` after :248-249, the tensors it hands to LPIPS and InceptionV3, bit for bit:

* `InferenceDataset.__getitem__`: the photo through PIL BICUBIC to R x R when it is not that size, the mask through PIL
  NEAREST to R x R, `mask // 255`, x = cat(mask - 0.5, (v * 2 / 255 - 1) * mask);
* :244-249: y = model(x), composed = masks * imgs + (1 - masks) * y, then (v * 0.5 + 0.5).clamp(0, 1) of both.

Per pass of up to 32 images (csrc/demo_resize.cu behind include/migan_b200.h): the demo path's stages on the evaluation
layout -- tables, [PIL BICUBIC width and height passes, when a photo of the pass is not R x R], R x R + mask + x -- then
`Generator.forward`, then one composite launch.  Generated masks come from `RandomMaskStream` in call order, so images
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


class EvalPipeline(torch.nn.Module):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from; or a
    `migan_b200.comodgan.Generator` of the same resolution (see `comodgan.load`).  `seed`: the script's np.random.seed,
    for the generated masks.  Co-Mod-GAN draws its noise planes and z from seeded streams on the device: the k-th image
    processed gets seed `noise_seed * 2**32 + k` (`noise_index` = k) unless `forward_batch(..., seeds=...)` names them,
    and the generator runs in chunks of at most `generator_batch`."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda", seed: int = 0, *,
                 noise_seed: int = 0, generator_batch: int = GENERATOR_BATCH):
        super().__init__()
        self.model = load_generator(self, model_or_state_dict, resolution, device, accept_comodgan=True)
        self.res = int(resolution)
        self.device_ = torch.device(device)
        self.masks = RandomMaskStream(self.res, seed=seed, device=self.device_)
        self.noise = NoiseSeeds(self.model, noise_seed, generator_batch)
        self.last_launches = []                 # kernel launches of each pass of the last call, generator included

    @property
    def noise_index(self) -> int:
        """How many images have drawn their Co-Mod-GAN noise from the pipeline's counter; settable."""
        return self.noise.noise_index

    @noise_index.setter
    def noise_index(self, k: int) -> None:
        self.noise.noise_index = int(k)

    @staticmethod
    def pass_launches(resized: bool, generator: int) -> int:
        """Launches of one pass: tables, [two resize passes when a photo is not R x R], R x R + x, the generator's, the
        composite.  `generator` is the sum over the pass's generator chunks (Co-Mod-GAN: noise launches included)."""
        return 2 + (2 if resized else 0) + generator + 1

    def _check(self, i, img, mask):
        img = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
        if not isinstance(img, torch.Tensor) or img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 \
                or min(img.shape[:2]) < 1:
            raise ValueError("EvalPipeline: image %d must be uint8 [H, W, 3]" % i)
        if mask is not None:
            mask = torch.from_numpy(np.ascontiguousarray(mask)) if isinstance(mask, np.ndarray) else mask
            if not isinstance(mask, torch.Tensor) or mask.dtype != torch.uint8 or mask.dim() != 2 or min(mask.shape) < 1:
                raise ValueError("EvalPipeline: mask %d must be uint8 [Hm, Wm] (mode L)" % i)
        return img, mask

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Optional[Sequence] = None, seeds=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(real, composed), CUDA float32 [n, 3, R, R] each.  masks=None takes the next n generated masks.  seeds
        (Co-Mod-GAN only, else ValueError): one 64-bit noise seed per image instead of the pipeline's counter."""
        imgs = list(imgs)
        n, R, dev = len(imgs), self.res, self.device_
        if masks is not None and len(masks) != n:
            raise ValueError("EvalPipeline.forward_batch: %d images and %d masks" % (n, len(masks)))
        seeds = self.noise.take("EvalPipeline", n, seeds)
        checked = [self._check(i, img, None if masks is None else masks[i]) for i, img in enumerate(imgs)]
        real = torch.empty((n, 3, R, R), dtype=torch.float32, device=dev)
        composed = torch.empty((n, 3, R, R), dtype=torch.float32, device=dev)
        if n == 0:
            return real, composed
        with torch.cuda.device(dev):
            imgs_d = [_to(img, dev, False) for img, _ in checked]
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
                reqs = (_abi.DemoRequest * k)()
                resized = False
                for r, img, m in zip(reqs, imgs_d[c:c + k], masks_d[c:c + k]):
                    r.img, r.H, r.W = img.data_ptr(), int(img.shape[0]), int(img.shape[1])
                    r.mask, r.Hm, r.Wm, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), 1
                    resized |= (r.H, r.W) != (R, R)
                need = int(lib.b200_eval_scratch_bytes(reqs, k, R))
                if need == 0:
                    _abi.check(_abi.ERR_INVALID)
                scratch = torch.empty(need, dtype=torch.uint8, device=dev)
                x = torch.empty((k, 4, R, R), dtype=torch.float32, device=dev)
                _abi.check(lib.b200_eval_preprocess(reqs, k, R, x.data_ptr(), real[c].data_ptr(), scratch.data_ptr(), need,
                                                    stream))
                y, gen_launches = self.noise.run(self.model, x, None if seeds is None else seeds[c:c + k])
                _abi.check(lib.b200_eval_composite(x.data_ptr(), y.data_ptr(), k, R, real[c].data_ptr(),
                                                   composed[c].data_ptr(), stream))
                keep.append((scratch, x, y))
                self.last_launches.append(self.pass_launches(resized, gen_launches))
            torch.cuda.current_stream(dev).synchronize()   # the inputs and the pass buffers are freed on return
        return real, composed

"""`DemoPipeline`: the reference demo's request path (scripts/demo.py:26-66, :120-143) at any photo size, on the GPU.

    pipe = DemoPipeline(state_dict_or_generator, resolution=512)
    composed = pipe(img, mask, invert=False)          # img uint8 [H,W,3]; mask uint8 [H,W] / [H,W,2|3|4]
    outs = pipe.forward_batch(imgs, masks)            # many photos of any sizes, one generator forward per 32
    pipe.forward_batch(imgs_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                       # ... outputs written, pipe.last_sizes set

`img` is `np.array(Image.open(p).convert("RGB"))` and `mask` is `np.array(Image.open(mask_path))` in any mode `read_mask`
handles (L, LA, RGB, RGBA; it may have its own size).  The result is byte for byte the image demo.py saves: its size is
that of `resize(img, max_size=R)`.  Per pass of up to 32 requests (kernels in csrc/demo_resize.cu behind
include/migan_b200.h, one launch per stage for every request):

    tables -> [PIL BICUBIC down-scale of the photos larger than R: width pass, height pass] -> PIL BICUBIC to R x R + the
    mask's NEAREST chain + x  ->  Generator.forward at the pass's batch size  ->  uint8 + OpenCV INTER_CUBIC width pass
    -> height pass + composite

OpenCV's cubic resize is reproduced as its scalar path computes it (`cv2.setUseOptimized(False)`); OpenCV's default
optimised path differs from it by at most 1 in a small fraction of values.  MI-GAN's output does not depend on the
batch size, so request i of a batch gets the bytes of a call with request i alone.  Co-Mod-GAN's does (one style RMS over
the batch, stylegan.py:146): its requests get the same bytes for the same `generator_batch` chunking.  There is no CPU
path.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple, Union

import torch

from . import _abi
from ._request_path import NoiseSeeds, _PhotoPipeline, _to

MASK_MAX = 512          # read_mask's first resize (demo.py:28)
# Co-Mod-GAN images per generator forward: its workspace is 9.8 GiB at 16 images of 512^2 (5.7 GiB at 256^2)
GENERATOR_BATCH = 16


def resized_size(w: int, h: int, max_size: int) -> Tuple[int, int]:
    """demo.py `resize` (:48-53): the (w, h) of an image after its down-scale to at most max_size."""
    if w > max_size or h > max_size:
        ratio = max_size / w if w > h else max_size / h
        return int(w * ratio), int(h * ratio)
    return w, h


class DemoPipeline(_PhotoPipeline):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from; or a
    `migan_b200.comodgan.Generator` of the same resolution (see `comodgan.load`).  Co-Mod-GAN draws its noise planes and
    z from seeded streams on the device: the k-th image processed gets seed `noise_seed * 2**32 + k` (`noise_index` = k)
    unless `forward_batch(..., seeds=...)` names them, and the generator runs in chunks of at most `generator_batch`."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda", *,
                 noise_seed: int = 0, generator_batch: int = GENERATOR_BATCH):
        super().__init__(model_or_state_dict, resolution, device, accept_comodgan=True)
        self.device_ = torch.device(device)
        self.noise = NoiseSeeds(self.model, noise_seed, generator_batch)
        self.last_sizes: List[Tuple[int, int]] = []       # (w', h') of every result of the last completed call(s)
        self.last_launches = 0                             # kernel launches of the last pass (MI-GAN: generator excluded)

    @property
    def noise_index(self) -> int:
        """How many images have drawn their Co-Mod-GAN noise from the pipeline's counter; settable."""
        return self.noise.noise_index

    @noise_index.setter
    def noise_index(self, k: int) -> None:
        self.noise.noise_index = int(k)

    def _set_record(self, record: list) -> None:
        self.last_sizes = record

    # -- one pass ---------------------------------------------------------------------------------------------------
    def _pass(self, imgs, masks, inverts, outs, seeds) -> None:
        """Enqueue one pass over <= 32 requests: imgs [H,W,3] / masks [Hm,Wm,C] uint8 CUDA contiguous, outs [h',w',3]
        uint8 CUDA contiguous, all on one device; seeds: the pass's Co-Mod-GAN seeds (None for MI-GAN)."""
        lib = _abi.load()
        n = len(imgs)
        dev = imgs[0].device
        stream = torch.cuda.current_stream(dev).cuda_stream
        reqs = (_abi.DemoRequest * n)()
        for r, img, m, inv, out in zip(reqs, imgs, masks, inverts, outs):
            r.img, r.H, r.W = img.data_ptr(), int(img.shape[0]), int(img.shape[1])
            r.mask, r.Hm, r.Wm, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), int(m.shape[2])
            r.invert = int(bool(inv))
            r.out, r.out_h, r.out_w = out.data_ptr(), int(out.shape[0]), int(out.shape[1])
        need = int(lib.b200_demo_scratch_bytes(reqs, n, self.res))
        if need == 0:
            _abi.check(_abi.ERR_INVALID)
        with torch.cuda.device(dev):
            # the caching allocator hands the scratch to the next pass on this stream in order
            scratch = torch.empty(need, dtype=torch.uint8, device=dev)
            x = torch.empty((n, 4, self.res, self.res), dtype=torch.float32, device=dev)
            _abi.check(lib.b200_demo_preprocess(reqs, n, self.res, x.data_ptr(), scratch.data_ptr(), need, stream))
            y, gen_launches = self.noise.run(self.model, x, seeds)
            if y.dtype != torch.float32 or tuple(y.shape) != (n, 3, self.res, self.res) or not y.is_contiguous():
                raise RuntimeError("generator output must be contiguous float32 (%d,3,%d,%d)" % (n, self.res, self.res))
            _abi.check(lib.b200_demo_postprocess(y.data_ptr(), reqs, n, self.res, scratch.data_ptr(), need, stream))
        down = any((int(r.out_w), int(r.out_h)) != (int(r.W), int(r.H)) for r in reqs)
        self.last_launches = 2 + (2 if down else 0) + 2 + (gen_launches if seeds is not None else 0)

    # -- public calls -----------------------------------------------------------------------------------------------
    def _check_mask_size(self, i, img, mask) -> None:
        """demo.py resizes the mask on its own, so it may have any size whose two resizes end at the photo's (w', h');
        ValueError where demo.py fails."""
        H, W, Hm, Wm = int(img.shape[0]), int(img.shape[1]), int(mask.shape[0]), int(mask.shape[1])
        if Hm < 1 or Wm < 1:
            raise ValueError("DemoPipeline: request %d: mask of shape %s, expected [H, W] or [H, W, 1..4]" % (i, tuple(mask.shape)))
        w1, h1 = resized_size(W, H, self.res)
        wb, hb = resized_size(*resized_size(Wm, Hm, MASK_MAX), self.res)
        if min(w1, h1, wb, hb) < 1 or min(resized_size(Wm, Hm, MASK_MAX)) < 1:
            raise ValueError("DemoPipeline: request %d: photo %dx%d or mask %dx%d resizes to a 0-pixel side at resolution %d"
                             % (i, W, H, Wm, Hm, self.res))
        if (wb, hb) != (w1, h1):
            raise ValueError("DemoPipeline: request %d: the mask resizes to %dx%d and the photo to %dx%d (w x h); demo.py "
                             "cannot compose them" % (i, wb, hb, w1, h1))

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True, seeds=None) -> list:
        """Many requests of any sizes, one pass per 32.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [Hm,Wm] or [Hm,Wm,C];
        numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns the composed images, uint8
        [h',w',3]: numpy for numpy photos, a tensor on the photo's device otherwise.  `last_sizes` holds every (w', h').

        wait=False only enqueues the work on the current stream and returns the output tensors, which hold the results
        (and `last_sizes` is set) after `wait()`.  CPU photos must then be pinned tensors (`pin_memory()`), since they are
        copied asynchronously; pageable CPU masks are staged through pinned memory.

        seeds (Co-Mod-GAN only, else ValueError): one 64-bit seed per request instead of the pipeline's counter."""
        kinds, checked, inverts = self._requests(imgs, masks, invert, wait)
        seeds = self.noise.take("DemoPipeline", len(checked), seeds)
        if not checked:
            return []
        dev = self._device()
        sizes = [resized_size(int(t.shape[1]), int(t.shape[0]), self.res) for t, _ in checked]
        nb = not wait
        imgs_d = [_to(t, dev, nb) for t, _ in checked]
        masks_d = [_to(m, dev, nb) for _, m in checked]
        outs_d = [torch.empty((h, w, 3), dtype=torch.uint8, device=dev) for w, h in sizes]
        for c in range(0, len(checked), _abi.PIPE_MAX_BATCH):
            s = slice(c, c + _abi.PIPE_MAX_BATCH)
            self._pass(imgs_d[s], masks_d[s], inverts[s], outs_d[s], None if seeds is None else seeds[s])
        return self._complete(kinds, outs_d, sizes, (imgs_d, masks_d, outs_d), torch.cuda.current_stream(dev), wait)


if __name__ == "__main__":
    # python -m migan_b200.demo: scripts/demo.py's command line (migan_b200/demo_command.py)
    from .demo_command import main
    main()

"""`MIGAN_Pipeline`: the arbitrary-resolution crop pipeline of the deployed (ONNX) form, scripts/create_onnx_pipeline.py:121-264.

Same constructor and call as the reference class:

    pipe = MIGAN_Pipeline(model_path, resolution, padding=128, device="cuda")
    result = pipe(image, mask)       # image (1,3,H,W) uint8, mask (1,1,h,w) uint8 (255 = known); image is updated in place
    results = pipe.forward_batch([image_0, image_1, ...], [mask_0, mask_1, ...])   # requests of different sizes at once
    pipe.forward_batch(images_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                         # ... images_t updated, pipe.last_boxes set

What happens per request (all on the GPU, kernels in csrc/pipeline.cu behind include/migan_b200.h):
mask -> image size (nearest) -> hole flags per column / row -> crop window (`get_masked_bbox` arithmetic, planned on the
device) -> crop resized to the model resolution (anti-aliased bilinear, bit-identical to torchvision's tensor resize on the
CPU) and turned into the generator input -> `Generator.forward` -> output mapped to [0, 255], resized to the crop, blended
into the image under the feathered mask.  There is no CPU path.

Every call, single request or many, runs in passes of up to 32 requests: one launch per stage covers every request of the
pass (hole flags, planning, weight tables, width pass, height pass; the post-processing's height pass is fused into the
blend), and the generator runs once at the pass's batch size (the captured CUDA graph when that is at most
`model.graph_max_batch`).  The planning launch turns the flags into the crop windows and the descriptors the later
launches read, so a pass is enqueued without waiting for the device; the windows come back to the host by an asynchronous
copy for `last_boxes`.  The generator's output does not depend on the batch size, so request i of a pass gets the same
bytes as a call with request i alone.

`CropPipeline` is the same pipeline on what a decoder produces, the form of the other photo pipelines:

    pipe = CropPipeline(state_dict_or_generator, resolution=512)
    out = pipe(img, mask, invert=False)       # img uint8 [H,W,3]; mask uint8 [h,w] / [h,w,1..4] of any size
    outs = pipe.forward_batch(imgs, masks)    # many photos of any sizes, one generator forward per 32

Each result is a new photo [H,W,3]: a copy of `img` with the crop window blended in, byte for byte what MIGAN_Pipeline
gives on the photo transposed to [3,H,W] and create_onnx_pipeline.py's `read_mask(mask, invert)` (:27-45).  The raw
mask becomes that plane in one launch per pass (channel, invert, 255 / 0 and the NEAREST resize to the photo's size), and
the stages address the photo in place through its pixel and channel strides.

Both classes also take a Co-Mod-GAN generator of their resolution (`comodgan.Generator`, see `comodgan.load`).  It draws
its noise from seeded streams: the k-th image processed gets seed `noise_seed * 2**32 + k` unless `forward_batch(...,
seeds=...)` names them, and it runs in chunks of at most `generator_batch` crops, whose style RMS it shares (DESIGN §8).
"""
from __future__ import annotations

import ctypes
from typing import List, Sequence, Tuple, Union

import torch

from . import _abi, ops
from ._request_path import NoiseSeeds, _Call, _PhotoPipeline, _Queued, _to
from .demo import GENERATOR_BATCH


def _crop_pass(pipe, images, masks, sizes, layout: int, seeds) -> torch.Tensor:
    """Enqueue one pass of `pipe` (MIGAN_Pipeline or CropPipeline) over <= 32 requests: images uint8 CUDA contiguous in
    `layout` (updated in place), masks [H,W] uint8 CUDA contiguous at the images' sizes `sizes` [(H, W)], all on one
    device; seeds: the pass's Co-Mod-GAN seeds (None for MI-GAN).  Nothing here waits for the device: the crop windows are
    planned on it.  Returns the pinned host buffer [n,4] int32 the windows are being copied into."""
    lib = _abi.load()
    n = len(images)
    dev = images[0].device
    stream = ops._stream(images[0])
    reqs = (_abi.PipeRequest * n)()
    for r, image, mask, (H, W) in zip(reqs, images, masks, sizes):
        r.image, r.mask, r.H, r.W = image.data_ptr(), mask.data_ptr(), H, W
    with torch.cuda.device(dev):
        flags = torch.empty(sum(r.W + r.H for r in reqs), dtype=torch.uint8, device=dev)
        _abi.check(lib.b200_hole_flags_batch(reqs, n, flags.data_ptr(), stream))
        need = int(lib.b200_pipeline_batch_scratch_bound(reqs, n, pipe.res))
        if need == 0:
            _abi.check(_abi.ERR_INVALID)
        # sized from the image sizes alone; the caching allocator hands it to the next pass on this stream in order
        scratch = torch.empty(need, dtype=torch.uint8, device=dev)
        boxes = torch.empty((n, 4), dtype=torch.int32, device=dev)
        _abi.check(lib.b200_pipeline_plan_batch_layout(reqs, n, pipe.res, int(pipe.padding), layout, flags.data_ptr(),
                                                       boxes.data_ptr(), scratch.data_ptr(), need, stream))
        x = torch.empty((n, 4, pipe.res, pipe.res), dtype=torch.float32, device=dev)
        _abi.check(lib.b200_pipeline_preprocess_planned(reqs, n, pipe.res, x.data_ptr(), scratch.data_ptr(), need, stream))
        y = pipe.model(x) if seeds is None else pipe.noise.run(pipe.model, x, seeds)[0]
        if y.dtype != torch.float32 or tuple(y.shape) != (n, 3, pipe.res, pipe.res) or not y.is_contiguous():
            raise RuntimeError("generator output must be contiguous float32 (%d,3,%d,%d)" % (n, pipe.res, pipe.res))
        _abi.check(lib.b200_pipeline_postprocess_planned(y.data_ptr(), reqs, n, pipe.res, pipe._k25.data_ptr(),
                                                         scratch.data_ptr(), need, stream))
        boxes_h = torch.empty((n, 4), dtype=torch.int32, pin_memory=True)
        boxes_h.copy_(boxes, non_blocking=True)
    return boxes_h


class MIGAN_Pipeline(_Queued):
    """Drop-in for scripts/create_onnx_pipeline.py:MIGAN_Pipeline.  `model_path`: a state_dict file written by the reference's
    export script (`torch.load`-able), a state_dict, or a ready `migan_b200.Generator`; or a `migan_b200.comodgan.Generator`
    of the same resolution, which draws its noise by `noise_seed` and runs in chunks of `generator_batch` (module doc)."""

    def __init__(self, model_path, resolution: int, padding: int = 128, device: Union[str, torch.device] = "cuda", *,
                 noise_seed: int = 0, generator_batch: int = GENERATOR_BATCH):
        super().__init__(model_path, resolution, device, accept_comodgan=True)
        self.noise = NoiseSeeds(self.model, noise_seed, generator_batch)
        self.register_buffer("gaussian_kernel", ops.feather_kernel(5, 1.0))     # GaussianSmoothing(1, 5, 1.0), :127-128
        self._k25 = ops.feather_kernel(5, 1.0).contiguous()                     # host copy handed to the C ABI
        self.padding = int(padding)
        self.device_ = torch.device(device)
        self.last_box: Tuple[int, int, int, int] = (0, 0, 0, 0)     # the last request's crop window
        self.last_boxes: List[Tuple[int, int, int, int]] = []        # every request's crop window of the last call

    # -- stages (each a call into the C ABI) ------------------------------------------------------------------------
    def get_masked_bbox(self, mask: torch.Tensor) -> Tuple[int, int, int, int]:
        """(x_min, x_max, y_min, y_max) of the crop window for a uint8 CUDA mask [..., H, W] (:133-227)."""
        lib = _abi.load()
        H, W = int(mask.shape[-2]), int(mask.shape[-1])
        mask = mask.reshape(H, W).contiguous()
        flags = torch.empty(W + H, dtype=torch.uint8, device=mask.device)
        with torch.cuda.device(mask.device):
            _abi.check(lib.b200_hole_flags(mask.data_ptr(), H, W, flags.data_ptr(), ops._stream(mask)))
        flags_h = flags.cpu()                                     # the one synchronisation of a request
        box = (ctypes.c_int * 4)()
        _abi.check(lib.migan_crop_box(flags_h.data_ptr(), H, W, self.res, int(self.padding), ctypes.cast(box, ctypes.c_void_p)))
        return int(box[0]), int(box[1]), int(box[2]), int(box[3])

    def _chunk(self, images, masks, seeds) -> torch.Tensor:
        """Enqueue one pass over <= 32 requests: images [3,H,W] uint8 CUDA contiguous (updated in place), masks [h,w] uint8
        CUDA contiguous, all on one device.  Returns the pinned host buffer [n,4] int32 the windows are being copied into."""
        lib = _abi.load()
        dev = images[0].device
        stream = ops._stream(images[0])
        planes, sizes = [], []                                     # resized masks stay alive until the launches are enqueued
        with torch.cuda.device(dev):
            for image, mask in zip(images, masks):
                H, W = int(image.shape[1]), int(image.shape[2])
                if tuple(mask.shape) != (H, W):                   # :255
                    m2 = torch.empty((H, W), dtype=torch.uint8, device=dev)
                    _abi.check(lib.b200_resize_nearest_u8(mask.data_ptr(), int(mask.shape[0]), int(mask.shape[1]), m2.data_ptr(), H, W, stream))
                    mask = m2
                planes.append(mask)
                sizes.append((H, W))
        return _crop_pass(self, images, planes, sizes, _abi.LAYOUT_CHW, seeds)

    def _submit(self, images, masks, copy_back, wait: bool, seeds=None) -> _Call:
        """Enqueue every pass of one call (images [3,H,W] / masks [h,w]: CUDA, contiguous, one device), then the copies of
        the results into the caller's tensors (`copy_back`: (caller tensor, staged device copy) pairs), then the call's
        completion event.  `seeds`: the caller's Co-Mod-GAN seeds or None; the pipeline's counter moves only once every
        request has passed its checks, so a refused call leaves it where it was."""
        for image in images:
            H, W = int(image.shape[1]), int(image.shape[2])
            if H < 3 or W < 3:
                raise RuntimeError("image of %d x %d: the feathering needs at least 3 x 3 pixels" % (H, W))
            if image.device != images[0].device:
                raise RuntimeError("MIGAN_Pipeline: the requests of one call must be on one device (%s and %s)" % (images[0].device, image.device))
        seeds = self.noise.take("MIGAN_Pipeline", len(images), seeds)
        B = _abi.PIPE_MAX_BATCH
        boxes = [self._chunk(images[c:c + B], masks[c:c + B], None if seeds is None else seeds[c:c + B])
                 for c in range(0, len(images), B)]
        for dst, src in copy_back:
            dst.copy_(src, non_blocking=not wait)
        event = None
        if images:
            event = torch.cuda.Event()
            event.record(torch.cuda.current_stream(images[0].device))
        return _Call(event, boxes, (images, masks, copy_back))

    def _set_record(self, record: list) -> None:
        """`record`: the pinned crop-window buffers of the passes waited for, read only now that their copies are done."""
        self.last_boxes = [tuple(int(v) for v in row) for b in record for row in b.tolist()]
        self.last_box = self.last_boxes[-1]

    @torch.no_grad()
    def forward(self, image: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        """image: (N,3,H,W) uint8, mask: (N,1,h,w) uint8 (255 = known).  The image is updated in place and returned (like the
        reference, whose deployed form takes N = 1; N > 1 gives each request its own crop, as if run one after the other)."""
        if image.dtype != torch.uint8 or mask.dtype != torch.uint8:
            raise RuntimeError("MIGAN_Pipeline expects uint8 image and mask")
        if image.dim() != 4 or image.shape[1] != 3 or mask.dim() != 4 or mask.shape[1] != 1 or mask.shape[0] != image.shape[0]:
            raise RuntimeError("MIGAN_Pipeline expects image (N,3,H,W) and mask (N,1,h,w)")
        img_d = image if (image.is_cuda and image.is_contiguous()) else image.to(self.device_).contiguous()
        mask_d = mask.to(img_d.device).contiguous()
        n = img_d.shape[0]
        call = self._submit([img_d[i] for i in range(n)], [mask_d[i, 0] for i in range(n)],
                            [] if img_d is image else [(image, img_d)], wait=True)
        self._finish([call])
        return image

    @torch.no_grad()
    def forward_batch(self, images, masks, wait: bool = True, seeds=None) -> list:
        """Many requests of any sizes in one pass per 32: images[i] (1,3,H_i,W_i) uint8 and masks[i] (1,1,h_i,w_i) uint8
        (255 = known), CUDA or CPU tensors.  Each image is updated in place, and the list of images is returned;
        `forward_batch(images, masks)[i]` is bit-identical to `pipe(images[i], masks[i])`.  `last_boxes` holds every crop
        window.  An image may not overlap another image or any mask: a batch cannot reproduce requests that read what an
        earlier one wrote.

        wait=False only enqueues the work on the current stream and returns: the images are updated, and `last_boxes` set,
        by `wait()`.  CPU images must then be pinned (`pin_memory()`), since their results come back by asynchronous
        copies; pageable CPU masks are staged through pinned memory.  The call keeps its staged device copies alive until
        `wait()`.

        seeds (Co-Mod-GAN only, else ValueError): one 64-bit seed per request instead of the pipeline's counter."""
        images, masks = list(images), list(masks)
        if len(images) != len(masks):
            raise RuntimeError("MIGAN_Pipeline.forward_batch: %d images and %d masks" % (len(images), len(masks)))
        for i, (image, mask) in enumerate(zip(images, masks)):
            if image.dtype != torch.uint8 or mask.dtype != torch.uint8:
                raise RuntimeError("MIGAN_Pipeline expects uint8 images and masks")
            if image.dim() != 4 or tuple(image.shape[:2]) != (1, 3) or mask.dim() != 4 or tuple(mask.shape[:2]) != (1, 1):
                raise RuntimeError("MIGAN_Pipeline.forward_batch expects images (1,3,H,W) and masks (1,1,h,w)")
            if not wait and not image.is_cuda and not (image.is_pinned() and image.is_contiguous()):
                raise RuntimeError("MIGAN_Pipeline.forward_batch(wait=False): CPU image %d must be pinned and contiguous "
                                   "(its result is copied back asynchronously); use image.pin_memory() or wait=True" % i)
        spans = [_span(t) for t in images + masks]
        for i in range(len(images)):
            for j in range(len(spans)):
                if j != i and _overlap(spans[i], spans[j]):
                    raise RuntimeError("MIGAN_Pipeline.forward_batch: image %d overlaps %s %d in memory" % (
                        i, "image" if j < len(images) else "mask", j if j < len(images) else j - len(images)))
        imgs_d = [im if (im.is_cuda and im.is_contiguous()) else im.to(self.device_, non_blocking=not wait).contiguous()
                  for im in images]
        masks_d = [_to(m, im.device, not wait) for m, im in zip(masks, imgs_d)]
        call = self._submit([im[0] for im in imgs_d], [m[0, 0] for m in masks_d],
                            [(image, img_d) for image, img_d in zip(images, imgs_d) if img_d is not image], wait, seeds)
        if wait:
            self._finish([call])
        else:
            self._pending.append(call)
        return images


class CropPipeline(_PhotoPipeline):
    """The crop pipeline on decoded photos and raw masks (module doc).  `model_or_state_dict`: a `migan_b200.Generator`, a
    state_dict, a file `torch.load` reads one from, or a `migan_b200.comodgan.Generator` of the same resolution."""

    def __init__(self, model_or_state_dict, resolution: int, padding: int = 128, device: Union[str, torch.device] = "cuda",
                 *, noise_seed: int = 0, generator_batch: int = GENERATOR_BATCH):
        super().__init__(model_or_state_dict, resolution, device, accept_comodgan=True)
        if int(padding) < 0:
            raise ValueError("CropPipeline: padding must be >= 0, got %d" % padding)
        self.padding = int(padding)
        self._k25 = ops.feather_kernel(5, 1.0).contiguous()      # host copy of the 25 feather taps
        self.noise = NoiseSeeds(self.model, noise_seed, generator_batch)
        self.last_box: Tuple[int, int, int, int] = (0, 0, 0, 0)
        self.last_boxes: List[Tuple[int, int, int, int]] = []     # every request's crop window of the last call(s)

    def _set_record(self, record: list) -> None:
        MIGAN_Pipeline._set_record(self, record)

    def _check_mask_size(self, i, img, mask) -> None:
        """The mask may have any size (it is resized to the photo's); the feathering needs a photo of at least 3 x 3."""
        H, W = int(img.shape[0]), int(img.shape[1])
        if int(mask.shape[0]) < 1 or int(mask.shape[1]) < 1:
            raise ValueError("CropPipeline: request %d: mask of shape %s has no pixels" % (i, tuple(mask.shape)))
        if H < 3 or W < 3:
            raise ValueError("CropPipeline: request %d: photo of %d x %d (H x W); the feathering needs at least 3 x 3"
                             % (i, H, W))

    def _pass(self, outs, masks, inverts, seeds) -> torch.Tensor:
        """Enqueue one pass over <= 32 requests: outs [H,W,3] uint8 CUDA contiguous (the photos, blended in place), masks
        [h,w,C] uint8 CUDA contiguous.  Returns the pinned host buffer of the crop windows."""
        lib = _abi.load()
        n = len(outs)
        dev = outs[0].device
        sizes = [(int(o.shape[0]), int(o.shape[1])) for o in outs]
        raw = (_abi.RawMask * n)()
        planes = [torch.empty(hw, dtype=torch.uint8, device=dev) for hw in sizes]
        for r, m, inv, plane, (H, W) in zip(raw, masks, inverts, planes, sizes):
            r.mask, r.hm, r.wm, r.channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), int(m.shape[2])
            r.invert, r.out, r.H, r.W = int(bool(inv)), plane.data_ptr(), H, W
        with torch.cuda.device(dev):
            _abi.check(lib.b200_pipeline_mask_planes(raw, n, ops._stream(outs[0])))
        return _crop_pass(self, outs, planes, sizes, _abi.LAYOUT_HWC, seeds)

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True, seeds=None) -> list:
        """Many requests of any sizes, one pass per 32.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [h,w] or [h,w,C] at any
        size; numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns new photos [H,W,3]:
        numpy for numpy photos, a tensor otherwise (on the photo's device for CUDA photos).  `last_boxes` holds every
        crop window.

        wait=False only enqueues the work on the current stream and returns the output tensors, which hold the results
        (and `last_boxes` is set) after `wait()`.  CPU photos must then be pinned tensors.

        seeds (Co-Mod-GAN only, else ValueError): one 64-bit seed per request instead of the pipeline's counter."""
        kinds, checked, inverts = self._requests(imgs, masks, invert, wait)
        seeds = self.noise.take("CropPipeline", len(checked), seeds)
        if not checked:
            return []
        dev = self._device()
        nb = not wait
        # a host photo's upload is its output buffer; a CUDA photo is copied, so the caller's stays as it was
        outs_d = [torch.empty(t.shape, dtype=torch.uint8, device=dev).copy_(t) if t.is_cuda else _to(t, dev, nb)
                  for t, _ in checked]
        masks_d = [_to(m, dev, nb) for _, m in checked]
        B = _abi.PIPE_MAX_BATCH
        boxes = [self._pass(outs_d[c:c + B], masks_d[c:c + B], inverts[c:c + B], None if seeds is None else seeds[c:c + B])
                 for c in range(0, len(checked), B)]
        return self._complete(kinds, outs_d, boxes, (outs_d, masks_d), torch.cuda.current_stream(dev), wait)


def _span(t: torch.Tensor):
    """(device, first byte, one past the last byte) of the memory a tensor's elements occupy."""
    if t.numel() == 0:
        return (t.device, 0, 0)
    extent = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    return (t.device, t.data_ptr(), t.data_ptr() + extent * t.element_size())


def _overlap(a, b) -> bool:
    return a[0] == b[0] and a[1] < b[2] and b[1] < a[2]

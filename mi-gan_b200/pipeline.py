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
"""
from __future__ import annotations

import ctypes
from typing import List, Tuple, Union

import torch

from . import _abi, ops
from ._request_path import _Call, _Queued, _to


class MIGAN_Pipeline(_Queued):
    """Drop-in for scripts/create_onnx_pipeline.py:MIGAN_Pipeline.  `model_path`: a state_dict file written by the reference's
    export script (`torch.load`-able), a state_dict, or a ready `migan_b200.Generator`."""

    def __init__(self, model_path, resolution: int, padding: int = 128, device: Union[str, torch.device] = "cuda"):
        super().__init__(model_path, resolution, device)
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

    def _chunk(self, images, masks) -> torch.Tensor:
        """Enqueue one pass over <= 32 requests: images [3,H,W] uint8 CUDA contiguous (updated in place), masks [h,w] uint8
        CUDA contiguous, all on one device.  Nothing here waits for the device: the crop windows are planned on it.  Returns
        the pinned host buffer [n,4] int32 the windows are being copied into."""
        lib = _abi.load()
        n = len(images)
        dev = images[0].device
        stream = ops._stream(images[0])
        reqs = (_abi.PipeRequest * n)()
        keep = []                                                  # resized masks stay alive until the launches are enqueued
        with torch.cuda.device(dev):
            for i, (image, mask) in enumerate(zip(images, masks)):
                H, W = int(image.shape[1]), int(image.shape[2])
                if tuple(mask.shape) != (H, W):                   # :255
                    m2 = torch.empty((H, W), dtype=torch.uint8, device=dev)
                    _abi.check(lib.b200_resize_nearest_u8(mask.data_ptr(), int(mask.shape[0]), int(mask.shape[1]), m2.data_ptr(), H, W, stream))
                    keep.append(m2)
                    mask = m2
                reqs[i].image, reqs[i].mask, reqs[i].H, reqs[i].W = image.data_ptr(), mask.data_ptr(), H, W
            flags = torch.empty(sum(r.W + r.H for r in reqs), dtype=torch.uint8, device=dev)
            _abi.check(lib.b200_hole_flags_batch(reqs, n, flags.data_ptr(), stream))
            need = int(lib.b200_pipeline_batch_scratch_bound(reqs, n, self.res))
            if need == 0:
                _abi.check(_abi.ERR_INVALID)
            # sized from the image sizes alone; the caching allocator hands it to the next pass on this stream in order
            scratch = torch.empty(need, dtype=torch.uint8, device=dev)
            boxes = torch.empty((n, 4), dtype=torch.int32, device=dev)
            _abi.check(lib.b200_pipeline_plan_batch(reqs, n, self.res, int(self.padding), flags.data_ptr(), boxes.data_ptr(),
                                                    scratch.data_ptr(), need, stream))
            x = torch.empty((n, 4, self.res, self.res), dtype=torch.float32, device=dev)
            _abi.check(lib.b200_pipeline_preprocess_planned(reqs, n, self.res, x.data_ptr(), scratch.data_ptr(), need, stream))
            y = self.model(x)
            if y.dtype != torch.float32 or tuple(y.shape) != (n, 3, self.res, self.res) or not y.is_contiguous():
                raise RuntimeError("generator output must be contiguous float32 (%d,3,%d,%d)" % (n, self.res, self.res))
            _abi.check(lib.b200_pipeline_postprocess_planned(y.data_ptr(), reqs, n, self.res, self._k25.data_ptr(),
                                                             scratch.data_ptr(), need, stream))
            boxes_h = torch.empty((n, 4), dtype=torch.int32, pin_memory=True)
            boxes_h.copy_(boxes, non_blocking=True)
        return boxes_h

    def _submit(self, images, masks, copy_back, wait: bool) -> _Call:
        """Enqueue every pass of one call (images [3,H,W] / masks [h,w]: CUDA, contiguous, one device), then the copies of
        the results into the caller's tensors (`copy_back`: (caller tensor, staged device copy) pairs), then the call's
        completion event."""
        for image in images:
            H, W = int(image.shape[1]), int(image.shape[2])
            if H < 3 or W < 3:
                raise RuntimeError("image of %d x %d: the feathering needs at least 3 x 3 pixels" % (H, W))
            if image.device != images[0].device:
                raise RuntimeError("MIGAN_Pipeline: the requests of one call must be on one device (%s and %s)" % (images[0].device, image.device))
        boxes = [self._chunk(images[c:c + _abi.PIPE_MAX_BATCH], masks[c:c + _abi.PIPE_MAX_BATCH])
                 for c in range(0, len(images), _abi.PIPE_MAX_BATCH)]
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
    def forward_batch(self, images, masks, wait: bool = True) -> list:
        """Many requests of any sizes in one pass per 32: images[i] (1,3,H_i,W_i) uint8 and masks[i] (1,1,h_i,w_i) uint8
        (255 = known), CUDA or CPU tensors.  Each image is updated in place, and the list of images is returned;
        `forward_batch(images, masks)[i]` is bit-identical to `pipe(images[i], masks[i])`.  `last_boxes` holds every crop
        window.  An image may not overlap another image or any mask: a batch cannot reproduce requests that read what an
        earlier one wrote.

        wait=False only enqueues the work on the current stream and returns: the images are updated, and `last_boxes` set,
        by `wait()`.  CPU images must then be pinned (`pin_memory()`), since their results come back by asynchronous
        copies; pageable CPU masks are staged through pinned memory.  The call keeps its staged device copies alive until
        `wait()`."""
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
                            [(image, img_d) for image, img_d in zip(images, imgs_d) if img_d is not image], wait)
        if wait:
            self._finish([call])
        else:
            self._pending.append(call)
        return images


def _span(t: torch.Tensor):
    """(device, first byte, one past the last byte) of the memory a tensor's elements occupy."""
    if t.numel() == 0:
        return (t.device, 0, 0)
    extent = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    return (t.device, t.data_ptr(), t.data_ptr() + extent * t.element_size())


def _overlap(a, b) -> bool:
    return a[0] == b[0] and a[1] < b[2] and b[1] < a[2]

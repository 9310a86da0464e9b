"""`FullResPipeline`: inpaint photos of any size at their own resolution, on the GPU.

    pipe = FullResPipeline(state_dict_or_generator, resolution=512)
    out = pipe(img, mask, invert=False)               # img uint8 [H,W,3]; mask uint8 [H,W] / [H,W,1..4]; out [H,W,3]
    outs = pipe.forward_batch(imgs, masks)            # many photos of mixed sizes
    pipe.forward_batch(imgs_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                       # ... outputs written, pipe.last_extents set

The generator's fully convolutional forward (`Generator.forward_fc`) runs at any H, W >= R that are multiples of R/4.  A
photo of another size is padded to the smallest such extent, (Hp, Wp) = (max(R, q ceil(H/q)), max(R, q ceil(W/q))) with
q = R/4, and the result is cropped back:

1. the mask's per-pixel steps are those of demo.py's `read_mask` without its resize: the channel (alpha of LA / RGBA, R of
   RGB, L itself), 255 - v if `invert`, then v < 255 -> 0; a pixel is known where the result is 255;
2. the photo stays at the origin; the bottom and right are filled by reflection without repeating the edge, iterated when
   the pad is longer than the side: numpy's `np.pad(..., mode="reflect")`.  The known-mask is reflected with the photo, so
   a hole that touches the border continues into the pad as a hole;
3. x = cat([mask - 0.5, img * mask]) at (Hp, Wp) -> `forward_fc` -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 on the top-left
   H x W, with the known pixels taken from the photo (demo.py's composite).

So the result is byte for byte `forward_fc_u8` on the reflect-padded photo and mask, cropped to H x W; a photo that is
already a valid size is not padded and gets `forward_fc_u8`'s bytes.  The padding rule decides the pixels the network sees
past the bottom and right edges, so results near those edges depend on it.

Requests are taken in passes of up to 32.  Within a pass they are grouped by extent in order of first appearance and each
group is split into chunks of at most the largest batch the forward accepts at that extent.  A pass is one pre-process
launch for every request, one `migan_forward_hw` per chunk and one post-process launch (kernels in csrc/fullres.cu behind
include/migan_b200.h).  The pipeline keeps one generator workspace, grown to the largest chunk seen, so the library's
per-shape plan cache serves every chunk and pass.  There is no CPU path.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Sequence, Tuple, Union

import torch

from . import _abi
from ._request_path import _PhotoPipeline, _to


class Chunk(NamedTuple):
    """One `migan_forward_hw` call of a pass: the extent and the requests in slot order (slot s is x[s] / y[s])."""
    Hp: int
    Wp: int
    requests: List[int]


def plan_passes(extents: Sequence[Tuple[int, int]], max_n: Dict[Tuple[int, int], int],
                pass_size: int = _abi.PIPE_MAX_BATCH) -> List[List[Chunk]]:
    """The passes of a call: requests [k * pass_size, (k + 1) * pass_size) form pass k; within a pass, requests are grouped
    by extent in order of first appearance and each group is split into chunks of at most max_n[extent]."""
    passes = []
    for p0 in range(0, len(extents), pass_size):
        groups: Dict[Tuple[int, int], List[int]] = {}
        for i in range(p0, min(p0 + pass_size, len(extents))):
            groups.setdefault(tuple(extents[i]), []).append(i)
        chunks = []
        for (Hp, Wp), idx in groups.items():
            m = max_n[(Hp, Wp)]
            chunks += [Chunk(Hp, Wp, idx[c:c + m]) for c in range(0, len(idx), m)]
        passes.append(chunks)
    return passes


def window_passes(pipe: _PhotoPipeline, eng, passes: List[List[Chunk]], wins, imgs, masks, inverts,
                  outs) -> Tuple[list, List[int]]:
    """Enqueue `passes` on the current stream, on the pipeline's one workspace.  wins[j] = (request, (y0, x0, h, w)) is
    read from imgs[request] and written into outs[request], inpainted as a photo of h x w.  Returns (the tensors the work
    uses, the launches of each pass, generator included)."""
    if not passes:
        return [], []
    lib, dev = eng.lib, eng.device
    ws = pipe._workspace(eng, passes)
    path = _abi.path_id(pipe.model.path)
    stream = torch.cuda.current_stream(dev).cuda_stream
    keep, launches = [ws], []
    for chunks in passes:
        n = sum(len(c.requests) for c in chunks)
        reqs = (_abi.WindowRequest * n)()
        xs, ys, k = [], [], 0
        for c in chunks:
            x = torch.empty((len(c.requests), 4, c.Hp, c.Wp), dtype=torch.float32, device=dev)
            y = torch.empty((len(c.requests), 3, c.Hp, c.Wp), dtype=torch.float32, device=dev)
            xs.append(x)
            ys.append(y)
            for slot, j in enumerate(c.requests):
                i, (y0, x0, h, w) = wins[j]
                r = reqs[k]
                k += 1
                img, m = imgs[i], masks[i]
                r.img, r.out, r.H, r.W = img.data_ptr(), outs[i].data_ptr(), int(img.shape[0]), int(img.shape[1])
                r.mask, r.mask_channels, r.invert = m.data_ptr(), int(m.shape[2]), int(bool(inverts[i]))
                r.y0, r.x0, r.h, r.w = y0, x0, h, w
                r.x, r.y, r.Hp, r.Wp = x[slot].data_ptr(), y[slot].data_ptr(), c.Hp, c.Wp
        _abi.check(lib.b200_window_preprocess(reqs, n, stream))
        n_launch = 2
        for c, x, y in zip(chunks, xs, ys):
            _abi.check(lib.migan_forward_hw(eng.handle, x.data_ptr(), y.data_ptr(), len(c.requests), c.Hp, c.Wp,
                                            ws.data_ptr(), ws.numel(), path, stream))
            n_launch += int(lib.migan_last_launch_count(eng.handle))
        _abi.check(lib.b200_window_postprocess(reqs, n, stream))
        keep.append(xs + ys)
        launches.append(n_launch)
    return keep, launches


class FullResPipeline(_PhotoPipeline):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda"):
        super().__init__(model_or_state_dict, resolution, device)
        self.last_extents: List[Tuple[int, int]] = []      # (Hp, Wp) of every result of the last completed call(s)
        self.last_launches = 0                              # kernel launches of the last pass, generator included

    def _set_record(self, record: list) -> None:
        self.last_extents = record

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True) -> list:
        """Many photos of any sizes.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [H,W] or [H,W,C] (C in 1..4) of the same
        H x W; numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns the inpainted photos, uint8
        [H,W,3]: numpy for numpy photos, a tensor on the photo's device otherwise.  `last_extents` holds every (Hp, Wp).
        Every refusal (TypeError for a non-array, ValueError naming the request otherwise) comes before anything is enqueued.

        wait=False only enqueues the work on the current stream and returns the output tensors, which hold the results
        (and `last_extents` is set) after `wait()`.  CPU photos must then be pinned tensors (`pin_memory()`), since they are
        copied asynchronously; pageable CPU masks are staged through pinned memory."""
        kinds, checked, inverts = self._requests(imgs, masks, invert, wait)
        if not checked:
            return []
        dev = self._device()
        with torch.cuda.device(dev):
            eng = self.model._engine(dev)
            wins, extents, max_n = [], [], {}
            for i, (img, _) in enumerate(checked):
                H, W = int(img.shape[0]), int(img.shape[1])
                ext, mx = self._extent(eng, i, H, W)
                wins.append((i, (0, 0, H, W)))
                extents.append(ext)
                max_n[ext] = mx
            nb = not wait
            imgs_d = [_to(t, dev, nb) for t, _ in checked]
            masks_d = [_to(m, dev, nb) for _, m in checked]
            outs_d = [torch.empty((int(t.shape[0]), int(t.shape[1]), 3), dtype=torch.uint8, device=dev) for t, _ in checked]
            keep, launches = window_passes(self, eng, plan_passes(extents, max_n), wins, imgs_d, masks_d, inverts, outs_d)
            self.last_launches = launches[-1]
            return self._complete(kinds, outs_d, extents, [imgs_d, masks_d, outs_d] + keep,
                                  torch.cuda.current_stream(dev), wait)

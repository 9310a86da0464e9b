"""`HoleWindowPipeline`: inpaint only margin-padded windows around the holes of photos of any size, at their own resolution.

    pipe = HoleWindowPipeline(state_dict_or_generator, resolution=512, margin=1)
    out = pipe(img, mask, invert=False)               # img uint8 [H,W,3]; mask uint8 [H,W] / [H,W,1..4]; out [H,W,3]
    outs = pipe.forward_batch(imgs, masks)            # many photos of mixed sizes
    pipe.forward_batch(imgs_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                       # ... outputs written, pipe.last_windows set

A typical object-removal request changes a small part of a large photo.  `FullResPipeline` runs the generator on the whole
photo; this pipeline runs it only on windows around the holes, each inpainted exactly as `FullResPipeline` inpaints a photo
of the window's size.  The rule (include/migan_b200.h, computed by the library), with q = R / 4:

1. the photo is split into q x q cells from the origin; a cell holding a hole pixel (a pixel `FullResPipeline`'s mask
   steps do not mark known) is a hole cell;
2. on each axis of side n, a span of cells [c0, c1] with a margin of m cells gives a = max(0, (c0 - m) q),
   b = min(n, (c1 + 1 + m) q), L = min(n, max(R, q ceil((b - a) / q))), s = min(max(a - (L - (b - a)) // 2, 0), n - L) and
   the window [s, s + L): a valid `forward_fc` size, or the whole side of the photo (then reflect-padded like a photo);
3. the hole cells are visited in row-major order; each starts as its own span and, while its window overlaps a window
   already listed, the first such window is removed and the spans are united; the result is appended.

So the windows are disjoint and hold every hole pixel, and the output is the photo with every window replaced by
`FullResPipeline` on that window's crop.  Only hole pixels change, so the window edges leave no seam.  A photo without a
hole comes back unchanged with no generator work; one whose holes span it gets `FullResPipeline`'s bytes.  A photo too large
for one forward is accepted as long as each of its windows fits one.

Per call: one cells launch per 32 requests (csrc/holewin.cu), all cells back to the host in one copy, the windows planned
by the library, then the windows of all requests in passes of up to 32, grouped by extent (`plan_passes`): a pass is one
pre-process launch, one `migan_forward_hw` per chunk and one post-process launch (csrc/fullres.cu), which writes the
windows into a copy of the photo.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import List, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi
from ._request_path import _PhotoPipeline, _to
from .fullres import plan_passes, window_passes

Window = Tuple[int, int, int, int]          # (y0, x0, h, w)


class HoleWindowPipeline(_PhotoPipeline):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from.  `margin`:
    cells of context (q = R / 4 pixels each) kept around the holes' cells on every side."""

    def __init__(self, model_or_state_dict, resolution: int, margin: int = 1, device: Union[str, torch.device] = "cuda"):
        super().__init__(model_or_state_dict, resolution, device)
        if int(margin) < 0:
            raise ValueError("HoleWindowPipeline: margin of %d cells (0 or more)" % margin)
        self.margin = int(margin)
        self._side = None                                   # the stream of the mask uploads and the cells
        self.last_windows: List[List[Window]] = []          # the windows of every result of the last completed call(s)
        self.last_launches = 0                              # kernel launches of the last call, generator included

    def _set_record(self, record: list) -> None:
        self.last_windows = record

    def _side_stream(self, dev) -> torch.cuda.Stream:
        if self._side is None:
            self._side = torch.cuda.Stream(dev)
        return self._side

    def _cells(self, eng, masks_d, inverts, stream) -> Tuple[List[Tuple[int, int, int]], torch.Tensor, int]:
        """Enqueue the cells of every mask, one launch per 32 on `stream`: ([(offset, H, W)] per request, cells, launches)."""
        lib = eng.lib
        tables, where, total = [], [], 0
        for p0 in range(0, len(masks_d), _abi.PIPE_MAX_BATCH):
            ms = masks_d[p0:p0 + _abi.PIPE_MAX_BATCH]
            t = (_abi.CellsRequest * len(ms))()
            for k, (r, m) in enumerate(zip(t, ms)):
                r.mask, r.H, r.W, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), int(m.shape[2])
                r.invert = int(bool(inverts[p0 + k]))
                where.append((total + int(lib.b200_hole_cells_bytes(t, k, self.res)) if k else total, r.H, r.W))
            nbytes = int(lib.b200_hole_cells_bytes(t, len(ms), self.res))
            if nbytes == 0:
                _abi.check(_abi.ERR_INVALID)
            tables.append((t, total))
            total += nbytes
        cells = torch.empty(total, dtype=torch.uint8, device=eng.device)
        for t, off in tables:
            _abi.check(lib.b200_hole_cells(t, len(t), self.res, cells.data_ptr() + off, stream))
        return where, cells, len(tables)

    def _plan(self, eng, cells_h: np.ndarray, where) -> List[List[Window]]:
        lib = eng.lib
        out = []
        for off, H, W in where:
            mx, cnt = ctypes.c_int(), ctypes.c_int()
            _abi.check(lib.migan_hole_windows_max(H, W, self.res, ctypes.byref(mx)))
            buf = (ctypes.c_int * (4 * mx.value))()
            _abi.check(lib.migan_hole_windows(cells_h.ctypes.data + off, H, W, self.res, self.margin, buf, mx.value,
                                              ctypes.byref(cnt)))
            out.append([tuple(buf[4 * k:4 * k + 4]) for k in range(cnt.value)])
        return out

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True) -> list:
        """Many photos of any sizes.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [H,W] or [H,W,C] (C in 1..4) of the same
        H x W; numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns the inpainted photos, uint8
        [H,W,3]: numpy for numpy photos, a tensor on the photo's device otherwise.  `last_windows` holds every request's
        windows, (y0, x0, h, w) each.  A TypeError (non-array) or ValueError naming the request refuses the call before any
        generator work: the input checks come first, and a window too large for one forward is refused once the cells are
        read back.

        Every call waits for its cells on the host (one round trip) before it enqueues the generator work.  With CPU
        masks, they are uploaded and the cells computed on a side stream, so that wait does not include work queued
        earlier on the current stream; a call with a CUDA mask orders the cells after the current stream (the mask may be
        produced there) and so waits for that stream.

        wait=False enqueues the rest on the current stream and returns the output tensors, which hold the results (and
        `last_windows` is set) after `wait()`.  CPU photos must then be pinned tensors (`pin_memory()`), since they are
        copied asynchronously; pageable CPU masks are staged through pinned memory."""
        kinds, checked, inverts = self._requests(imgs, masks, invert, wait)
        if not checked:
            return []
        dev = self._device()
        with torch.cuda.device(dev):
            eng = self.model._engine(dev)
            nb = not wait
            cur = torch.cuda.current_stream(dev)
            side = self._side_stream(dev)
            if any(m.is_cuda for _, m in checked):
                side.wait_stream(cur)
            with torch.cuda.stream(side):
                masks_d = [_to(m, dev, nb) for _, m in checked]
                where, cells_d, launches = self._cells(eng, masks_d, inverts, side.cuda_stream)
                cells_h = torch.empty(cells_d.shape, dtype=torch.uint8, pin_memory=True)
                cells_h.copy_(cells_d, non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(side)
            ready.synchronize()
            wins_per = self._plan(eng, cells_h.numpy(), where)
            wins, extents, max_n = [], [], {}
            for i, ws_i in enumerate(wins_per):
                for win in ws_i:
                    ext, mx = self._extent(eng, i, win[2], win[3], "window (y0, x0, h, w) = %s: " % (win,))
                    wins.append((i, win))
                    extents.append(ext)
                    max_n[ext] = mx
            passes = plan_passes(extents, max_n)
            cur.wait_event(ready)
            outs_d = []
            for img, _ in checked:                          # the output photo: one copy of the input, windows written
                out = torch.empty((int(img.shape[0]), int(img.shape[1]), 3), dtype=torch.uint8, device=dev)
                out.copy_(img, non_blocking=nb)
                outs_d.append(out)
            keep, pass_launches = window_passes(self, eng, passes, wins, outs_d, masks_d, inverts, outs_d)
            self.last_launches = launches + sum(pass_launches)
            return self._complete(kinds, outs_d, wins_per, [masks_d, outs_d, cells_d, cells_h] + keep, cur, wait)

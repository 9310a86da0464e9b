"""`RandomMaskStream`: the evaluation protocol's free-form masks on the GPU.

    stream = RandomMaskStream(512, seed=0)
    m = stream.next(32)              # CUDA uint8 [32, 512, 512]: 255 known, 0 hole
    state = stream.get_state()       # np.random.get_state()'s tuple

`next(n)` returns the next n results of `RandomMask(s)` (scripts/generate_masks.py, hole_range [0, 1]; the evaluation
script's `InferenceDataset` calls the same function) after `np.random.seed(seed)`: the same bytes, and the state afterwards
is the one numpy's global stream has after those n calls.  How the stream is split into calls does not change the bytes.

How (include/migan_b200.h, csrc/masks.cu): RandomMask draws *attempts* until one has a hole ratio in (0, 1), and an
attempt's draws never depend on earlier results.  So the library plans a batch of attempts on the host (numpy's
MT19937 and legacy distributions, one fixed-size record of rectangles, brush quads and discs per attempt, and the state
after each attempt), the records go to the device through pinned staging, one launch paints every attempt and counts its
holes, and one launch copies the first accepted attempts, in attempt order, into the output.  The hole counts come back
in one small copy; the stream rewinds to the state after the last attempt it used and, when fewer than n were accepted
(the normal case at s = 32, where most attempts are all-hole), plans more.

The masks `torch.utils.data.DataLoader` workers draw on the fly in the reference's training datasets are not this
stream: torch reseeds numpy in every worker, so that stream is not reproducible.  `synthetic.free_form_mask` stays the
project's own (not the reference's) random mask.
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional, Union

import numpy as np
import torch

from . import _abi

_RECORD = ctypes.sizeof(_abi.MaskRecord)
_STATE = ctypes.sizeof(_abi.NpRandom)
_ROUND_BYTES = 1 << 29                         # a round's buffers: [A][s][s] attempts, records (pinned and device), states


class RandomMaskStream:
    """The results of RandomMask(resolution) after np.random.seed(seed), generated on `device`."""

    def __init__(self, resolution: int, seed: int = 0, device: Union[str, torch.device] = "cuda"):
        s = int(resolution)
        if not _abi.MASK_MIN_SIZE <= s <= _abi.MASK_MAX_SIZE:
            raise ValueError("RandomMaskStream: resolution %d (%d to %d)" % (s, _abi.MASK_MIN_SIZE, _abi.MASK_MAX_SIZE))
        if not 0 <= int(seed) <= 0xFFFFFFFF:
            raise ValueError("RandomMaskStream: seed %d (0 to 2**32 - 1, as np.random.seed)" % seed)
        self.resolution = s
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("RandomMaskStream: device %s (the masks are generated on a CUDA device)" % self.device)
        self.lib = _abi.load()
        self._state = _abi.NpRandom()
        _abi.check(self.lib.migan_np_seed(ctypes.byref(self._state), int(seed)))
        self.attempts = 0                      # attempts consumed so far (accepted or not)
        self._accepted = 0
        self._staging = self._records = self._scratch = self._holes = self._holes_h = None

    def get_state(self):
        """The stream's position in np.random.get_state()'s format."""
        st = self._state
        return ("MT19937", np.array(st.key, dtype=np.uint32), int(st.pos), int(st.has_gauss), float(st.gauss))

    def set_state(self, state) -> None:
        """Continue from a state in np.random.get_state()'s format (np.random.set_state's tuple)."""
        name, key, pos, has_gauss, gauss = state
        key = np.asarray(key, dtype=np.uint32)
        if name != "MT19937" or key.shape != (624,) or not 0 <= int(pos) <= 624:
            raise ValueError("RandomMaskStream.set_state: expected ('MT19937', uint32[624], pos 0..624, has_gauss, gauss)")
        st = _abi.NpRandom()
        ctypes.memmove(st.key, key.ctypes.data, 624 * 4)
        st.pos, st.has_gauss, st.gauss = int(pos), int(bool(has_gauss)), float(gauss)
        self._state = st

    def _buffers(self, attempts: int):
        s = self.resolution
        if self._staging is None or self._staging.numel() < attempts * _RECORD:
            self._staging = torch.empty(attempts * _RECORD, dtype=torch.uint8, pin_memory=True)
            self._records = torch.empty(attempts * _RECORD, dtype=torch.uint8, device=self.device)
            self._scratch = torch.empty((attempts, s, s), dtype=torch.uint8, device=self.device)
            self._holes = torch.empty(attempts, dtype=torch.int32, device=self.device)
            self._holes_h = torch.empty(attempts, dtype=torch.int32, pin_memory=True)

    def _round_size(self, need: int) -> int:
        """Attempts to plan for `need` more results: the expected count at the stream's acceptance rate so far, plus a
        margin, capped by the scratch size."""
        rate = (self._accepted + 1) / (self.attempts + 2) if self.attempts else 0.9
        a = int(math.ceil(need / max(rate, 0.05))) + need // 16 + 4
        per_attempt = self.resolution * self.resolution + 2 * _RECORD + _STATE
        cap = max(1, min(_abi.MASK_MAX_ATTEMPTS, _ROUND_BYTES // per_attempt))
        return min(a, cap)

    @torch.no_grad()
    def next(self, n: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The next n masks: CUDA uint8 [n, s, s] (255 known, 0 hole), written into `out` when given (a contiguous,
        16-byte aligned CUDA uint8 tensor of that shape).  Returns when the masks are enqueued on the current stream and
        the stream's state has advanced past them."""
        s, n = self.resolution, int(n)
        if n < 0:
            raise ValueError("RandomMaskStream.next: %d masks" % n)
        if out is None:
            out = torch.empty((n, s, s), dtype=torch.uint8, device=self.device)
        elif (out.dtype != torch.uint8 or not out.is_cuda or tuple(out.shape) != (n, s, s) or not out.is_contiguous()
              or out.data_ptr() % 16):
            raise ValueError("RandomMaskStream.next: out must be a contiguous, 16-byte aligned CUDA uint8 tensor of "
                             "shape %s" % ((n, s, s),))
        lib = self.lib
        with torch.cuda.device(out.device):
            stream = torch.cuda.current_stream(out.device)
            done = 0
            while done < n:
                need = n - done
                a = self._round_size(need)
                self._buffers(a)
                states = (_abi.NpRandom * a)()
                st = _abi.NpRandom.from_buffer_copy(self._state)
                _abi.check(lib.migan_mask_plan(ctypes.byref(st), s, a, self._staging.data_ptr(), states))
                self._records[:a * _RECORD].copy_(self._staging[:a * _RECORD], non_blocking=True)
                _abi.check(lib.b200_mask_raster(self._records.data_ptr(), a, s, self._scratch.data_ptr(),
                                                self._holes.data_ptr(), stream.cuda_stream))
                _abi.check(lib.b200_mask_compact(self._scratch.data_ptr(), self._holes.data_ptr(), a, s, min(need, a),
                                                 out[done].data_ptr(), stream.cuda_stream))
                self._holes_h[:a].copy_(self._holes[:a], non_blocking=True)
                stream.synchronize()              # the staging buffers are reused by the next round or call
                holes = self._holes_h[:a].numpy()
                ok = np.flatnonzero((holes > 0) & (holes < s * s))
                used = int(ok[need - 1]) + 1 if len(ok) >= need else a
                took = min(need, len(ok))
                self._state = _abi.NpRandom.from_buffer_copy(states[used - 1])
                self.attempts += used
                self._accepted += took
                done += took
        return out

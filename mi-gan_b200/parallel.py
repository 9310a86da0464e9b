"""Batch sharding over the GPUs of one box: one process per GPU, weights replicated, each rank
runs `Generator.forward` on its shard and the outputs are all-gathered over NCCL (NVLink).

The reference has no inference parallelism at all (SURVEY.md 2.1); images are independent
(no batch statistics, migan_inference.py:165-167), so this is pure data parallelism with ONE
collective per batch and nothing else on the data path.

The all-gather runs asynchronously on NCCL's stream: `forward_async` returns a handle and the
next batch's kernels start immediately, so the transfer of batch t overlaps the compute of
batch t+1 (in a serving loop the collective is then off the critical path).
"""
from __future__ import annotations

import os
from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist


def resolve_gather(gather: str, world_size: int) -> str:
    """'auto' -> the copy-engine gather at 2 GPUs (no SM is taken from the compute kernels), the NCCL all-gather above
    (the per-peer copies of the copy-engine form serialise against the compute stream as the peer count grows)."""
    if gather != "auto":
        return gather
    return "ce" if world_size == 2 else "nccl"


def nccl_channels_for(world_size: int) -> int:
    """Channels (= SMs left free) for the NCCL all-gather: the bytes to gather grow with the world size while the step
    they should hide under does not, so 8 GPUs get more channels than 4.  Not tuned on H100s."""
    return 12 if world_size > 4 else 8


def configure_overlap(reserve_sms: int = None, nccl_channels: int = None, gather: str = "auto", world_size: int = None) -> None:
    """Call BEFORE `init_process_group` and before the first forward.

    gather = "ce": the output all-gather moves its bytes with the copy engines (peer-to-peer reads over NVLink, see
    `ShardedGenerator`); the only NCCL kernel per step is an 8-byte all-reduce used as the ready signal, so the persistent
    tensor-core kernel keeps every SM (no reservation).
    gather = "nccl": `all_gather_into_tensor` runs on NCCL's SM-resident copy kernels, one SM per channel, concurrently with
    the next batch's kernels.  The persistent kernel uses one CTA per SM -- if they collide, its last CTAs run as a second
    wave -- so NCCL is limited to `nccl_channels` channels (default `nccl_channels_for(world_size)`) and the persistent grids
    leave as many SMs free (`reserve_sms`).
    gather = "auto" (default): see `resolve_gather`; `world_size` defaults to the WORLD_SIZE of the launcher.
    Respects values already present in the environment."""
    if world_size is None:
        world_size = int(os.environ.get("WORLD_SIZE", "1"))
    if resolve_gather(gather, world_size) == "nccl":
        if nccl_channels is None:
            nccl_channels = nccl_channels_for(world_size)
        os.environ.setdefault("NCCL_MAX_NCHANNELS", str(nccl_channels))
        os.environ.setdefault("NCCL_MIN_NCHANNELS", str(nccl_channels))
        os.environ.setdefault("MIGAN_TC_RESERVE_SMS", str(nccl_channels if reserve_sms is None else reserve_sms))
    else:
        os.environ.setdefault("MIGAN_TC_RESERVE_SMS", str(0 if reserve_sms is None else reserve_sms))


def shard_bounds(global_n: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous rank-major shard [lo, hi) of a global batch; the first (global_n % world_size)
    ranks get one extra image."""
    if global_n < 0 or world_size < 1 or not (0 <= rank < world_size):
        raise ValueError("bad shard request (%d, %d, %d)" % (global_n, world_size, rank))
    base, rem = divmod(global_n, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class GatherHandle:
    """Result of `forward_async`: `wait()` makes the current stream wait for the gather and returns the gathered tensor
    [world*n_local, 3, R, R] (rank-major).  `local` is this rank's own output."""

    def __init__(self, out: torch.Tensor, work, local: torch.Tensor, event=None):
        self._out, self._work, self.local, self._event = out, work, local, event

    def wait(self) -> torch.Tensor:
        if self._work is not None:
            self._work.wait()
            self._work = None
        if self._event is not None:
            torch.cuda.current_stream(self._out.device).wait_event(self._event)
            self._event = None
        return self._out


class ShardedGenerator:
    """Data-parallel wrapper.  `model` is any callable x[n,4,R,R] -> y[n,3,R,R] on this rank's device
    (the H100 `Generator`; CPU stand-ins are used by the gloo tests).

    gather = "nccl": one `all_gather_into_tensor` per batch (NCCL's copy kernels, SM-resident).
    gather = "ce" (CUDA tensors, all ranks on one box): the same all-gather with the bytes moved by the copy engines.  Every
      rank publishes a small ring of output buffers to its peers once (CUDA IPC, through torch's tensor sharing); per batch
      it (1) puts its y into the ring, (2) joins an 8-byte NCCL all-reduce -- the only collective kernel, used as the "every
      rank's y is in place" signal -- and (3) pulls the 7 peer shards into a fresh gathered tensor with peer-to-peer
      `cudaMemcpyAsync` reads over NVLink on a side stream.  No SM is taken from the compute kernels, so nothing has to be
      reserved for the collective, and the pull of batch t overlaps the compute of batch t+1.
      Variants that were tried and dropped: a push form with bare `cudaMemcpyAsync` on the sender's own streams, and
      signalling with `cuStreamWaitValue32` plus 4-byte peer writes instead of the all-reduce (a stream parked in a memory
      wait delays the streams sharing its hardware queue).  `tools/p2p_probe.py` measures the primitives.
    gather = "auto" (default): `resolve_gather` -- "ce" at 2 GPUs, "nccl" above."""

    RING = 3   # published y buffers per rank: slot t % RING is rewritten only after the ready signal of step t - RING + 1

    def __init__(self, model: Callable[[torch.Tensor], torch.Tensor], group: Optional[dist.ProcessGroup] = None,
                 gather: str = "auto"):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised (launch with torchrun, one process per GPU)")
        if gather not in ("auto", "ce", "nccl"):
            raise ValueError("gather must be 'auto', 'ce' or 'nccl'")
        self.model = model
        self.group = group
        self.world_size = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.gather = resolve_gather(gather, self.world_size) if gather == "auto" else gather
        self._fallback_ok = (gather == "auto")     # "auto" may fall back to NCCL when the peers cannot map each other's memory
        self._ce = None          # lazily built state of the copy-engine path
        self._step = 0

    def check_replicas(self, state_dict) -> None:
        """All ranks must hold identical weights (analogue of the reference's
        torch_utils/misc.py:178-187 check_ddp_consistency): compare a checksum with rank 0."""
        total = torch.zeros(2, dtype=torch.float64)
        for v in state_dict.values():
            v = v.detach().double().cpu()
            total[0] += v.sum()
            total[1] += v.abs().sum()
        dev = next(iter(state_dict.values())).device
        total = total.to(dev if dev.type == "cuda" else "cpu")
        ref = total.clone()
        dist.broadcast(ref, src=0, group=self.group)
        if not torch.equal(ref, total):
            raise RuntimeError("rank %d holds different weights than rank 0" % self.rank)

    # -- copy-engine all-gather ---------------------------------------------------------------------------------------
    def _setup_ce(self, y: torch.Tensor):
        """Publish RING output buffers of y's shape to every peer and map theirs (one-time, collective)."""
        from torch.multiprocessing.reductions import reduce_tensor
        ring = [torch.empty_like(y) for _ in range(self.RING)]
        mine = [reduce_tensor(t) for t in ring]                       # (rebuild_fn, args): CUDA IPC handle + offset
        everyone = [None] * self.world_size
        dist.all_gather_object(everyone, mine, group=self.group)
        peers = {}
        for p in range(self.world_size):
            if p != self.rank:
                peers[p] = [fn(*args) for fn, args in everyone[p]]    # tensors aliasing rank p's ring (peer-mapped)
                if tuple(peers[p][0].shape) != tuple(y.shape):
                    raise RuntimeError("rank %d published shards of a different shape" % p)
        self._ce = {"ring": ring, "peers": peers, "side": torch.cuda.Stream(device=y.device),
                    "flag": torch.zeros(1, device=y.device), "ready": {}, "shape": tuple(y.shape)}

    def _forward_ce(self, y: torch.Tensor) -> GatherHandle:
        ce, t, n = self._ce, self._step, y.shape[0]
        slot = t % self.RING
        cur = torch.cuda.current_stream(y.device)
        old = ce["ready"].pop(t - self.RING + 1, None)
        if old is not None:
            old.wait()                                # slot's previous content (step t - RING) has been pulled by every peer
        ce["ring"][slot].copy_(y, non_blocking=True)
        out = torch.empty((self.world_size * n,) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
        ev = torch.cuda.Event()
        ev.record(cur)
        side = ce["side"]
        with torch.cuda.stream(side):
            side.wait_event(ev)
            ready = dist.all_reduce(ce["flag"], group=self.group, async_op=True)   # "every rank's y(t) is in its ring"
            ready.wait()                              # the side stream (not the host) waits for it
            for p, bufs in ce["peers"].items():
                out[p * n:(p + 1) * n].copy_(bufs[slot], non_blocking=True)         # peer-to-peer read, copy engine
            out[self.rank * n:(self.rank + 1) * n].copy_(ce["ring"][slot], non_blocking=True)
            done = torch.cuda.Event()
            done.record(side)
        out.record_stream(side)
        ce["ready"][t] = ready
        return GatherHandle(out, None, y, done)

    def forward_async(self, x_local: torch.Tensor) -> GatherHandle:
        y = self.model(x_local)
        if self.world_size == 1:
            return GatherHandle(y, None, y)
        mode = self.gather
        if mode == "ce" and y.is_cuda:
            if self._ce is None or self._ce["shape"] != tuple(y.shape):
                try:
                    self._setup_ce(y)
                except Exception:
                    if not self._fallback_ok:
                        raise
                    self.gather = mode = "nccl"       # e.g. no peer access between the devices
            if mode != "nccl":
                h = self._forward_ce(y)
                self._step += 1
                return h
        out = torch.empty((self.world_size * y.shape[0],) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
        work = dist.all_gather_into_tensor(out, y, group=self.group, async_op=True)
        return GatherHandle(out, work, y)

    def forward(self, x_local: torch.Tensor) -> torch.Tensor:
        """Every rank passes its shard (equal sizes) and receives all outputs, rank-major."""
        return self.forward_async(x_local).wait()

    def forward_global(self, x_global: torch.Tensor) -> torch.Tensor:
        """Every rank passes the same global batch (size divisible by the world size)."""
        if x_global.shape[0] % self.world_size:
            raise ValueError("global batch %d is not divisible by world size %d" % (x_global.shape[0], self.world_size))
        lo, hi = shard_bounds(x_global.shape[0], self.world_size, self.rank)
        return self.forward(x_global[lo:hi].contiguous())

    def forward_host_async(self, x_host_local: torch.Tensor, out_host_local: torch.Tensor) -> None:
        """End-to-end serving step of one rank: pinned host shard -> device, forward, all-gather, and this rank's rows of the
        GATHERED tensor back to pinned host memory (each process returns its part of the batch; the gather sits on the
        path).  Three streams and two device input slots: the H2D copy of batch t+1 and the D2H copy of batch t-1 run under
        the kernels of batch t.  Enqueue-only: call `host_wait()` before reading `out_host_local`."""
        dev = torch.device("cuda", torch.cuda.current_device())
        hs = self.__dict__.get("_host")
        if hs is None or hs["shape"] != tuple(x_host_local.shape):
            hs = {"shape": tuple(x_host_local.shape), "x": [torch.empty(x_host_local.shape, dtype=x_host_local.dtype, device=dev) for _ in range(2)],
                  "h2d": torch.cuda.Stream(device=dev), "d2h": torch.cuda.Stream(device=dev), "done": [None, None], "k": 0}
            self._host = hs
        k = hs["k"]
        slot = k % 2
        cur = torch.cuda.current_stream(dev)
        with torch.cuda.stream(hs["h2d"]):
            if hs["done"][slot] is not None:
                hs["h2d"].wait_event(hs["done"][slot])       # the forward that read this slot two steps ago has finished
            hs["x"][slot].copy_(x_host_local, non_blocking=True)
            ev_in = torch.cuda.Event()
            ev_in.record(hs["h2d"])
        cur.wait_event(ev_in)
        h = self.forward_async(hs["x"][slot])
        g = h.wait()
        ev_c = torch.cuda.Event()
        ev_c.record(cur)
        hs["done"][slot] = ev_c
        n = x_host_local.shape[0]
        with torch.cuda.stream(hs["d2h"]):
            hs["d2h"].wait_event(ev_c)
            out_host_local.copy_(g[self.rank * n:(self.rank + 1) * n], non_blocking=True)
        g.record_stream(hs["d2h"])
        hs["k"] = k + 1

    def close(self) -> None:
        """Drop the peer mappings of the copy-engine path (collective: call on every rank before the process group is destroyed,
        so that no rank frees a published buffer while a peer still maps it)."""
        if self._ce is not None:
            torch.cuda.synchronize()
            dist.barrier(group=self.group)
            self._ce["peers"].clear()
            dist.barrier(group=self.group)
            self._ce = None

    def host_wait(self) -> None:
        hs = self.__dict__.get("_host")
        if hs is not None:
            hs["d2h"].synchronize()

    __call__ = forward

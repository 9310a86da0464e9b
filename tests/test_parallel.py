"""The batch-sharding / all-gather path on CPU: world_size 2 over gloo (no GPU).  The per-rank
"model" is the CPU oracle (tests may use it); on the GPU box bench.py runs the same wrapper over NCCL."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from migan_b200 import parallel
from oracle import migan_oracle as O


def test_shard_bounds():
    assert [parallel.shard_bounds(10, 4, r) for r in range(4)] == [(0, 3), (3, 6), (6, 8), (8, 10)]
    assert parallel.shard_bounds(64, 8, 7) == (56, 64)
    assert parallel.shard_bounds(3, 4, 3) == (3, 3)          # ragged: an empty shard
    with pytest.raises(ValueError):
        parallel.shard_bounds(8, 2, 2)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    R = 32
    sd = O.make_state_dict(R, seed=1)
    model = lambda x: O.generator_forward(sd, x, R)          # noqa: E731  (stand-in for the H100 Generator)
    sg = parallel.ShardedGenerator(model)
    sg.check_replicas(sd)
    x_global = O.make_input(R, 6, seed=3)
    y = sg.forward_global(x_global)                           # every rank gets all 6 outputs, in order
    want = O.generator_forward(sd, x_global, R)
    ok = float((y - want).abs().max()) < 1e-5 and y.shape == want.shape
    # async handle + local shard path (what bench.py uses)
    lo, hi = parallel.shard_bounds(6, world, rank)
    h = sg.forward_async(x_global[lo:hi].contiguous())
    y2 = h.wait()
    ok = ok and float((y2 - want).abs().max()) < 1e-5 and torch.equal(h.local, y2[lo:hi])
    # replica check must fire when weights differ
    bad = dict(sd)
    if rank == 1:
        bad["synthesis.b4.torgb.bias"] = bad["synthesis.b4.torgb.bias"] + 1
    try:
        sg.check_replicas(bad)
        mismatch_detected = (rank == 0)                       # rank 0 compares with itself
    except RuntimeError:
        mismatch_detected = True
    with open(os.path.join(out_dir, "rank%d.ok" % rank), "w") as f:
        f.write("%d %d" % (int(ok), int(mismatch_detected)))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_generator_gloo_world2(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for r in range(world):
        ok, mm = open(tmp_path / ("rank%d.ok" % r)).read().split()
        assert ok == "1" and mm == "1"


def test_gather_policy_follows_measured_world_sizes():
    """'auto' = copy engines at 2 GPUs, NCCL all-gather above (profiles/r02_scale_variants.md); configure_overlap sets the
    matching SM reservation / channel count without overriding the caller's environment."""
    assert parallel.resolve_gather("auto", 2) == "ce" and parallel.resolve_gather("auto", 8) == "nccl"
    assert parallel.resolve_gather("auto", 4) == "nccl" and parallel.resolve_gather("ce", 8) == "ce"
    keys = ("MIGAN_TC_RESERVE_SMS", "NCCL_MAX_NCHANNELS", "NCCL_MIN_NCHANNELS")
    saved = {k: os.environ.pop(k, None) for k in keys}
    try:
        parallel.configure_overlap(world_size=2)
        assert os.environ["MIGAN_TC_RESERVE_SMS"] == "0" and "NCCL_MAX_NCHANNELS" not in os.environ
        del os.environ["MIGAN_TC_RESERVE_SMS"]
        parallel.configure_overlap(world_size=4)
        assert os.environ["MIGAN_TC_RESERVE_SMS"] == "8" and os.environ["NCCL_MAX_NCHANNELS"] == "8"
        for k in keys:
            os.environ.pop(k, None)
        parallel.configure_overlap(world_size=8)            # one SM per channel; more channels where the gather would not hide under a step
        assert os.environ["MIGAN_TC_RESERVE_SMS"] == "12" and os.environ["NCCL_MAX_NCHANNELS"] == "12" == os.environ["NCCL_MIN_NCHANNELS"]
        os.environ["MIGAN_TC_RESERVE_SMS"] = "3"
        parallel.configure_overlap(world_size=8)
        assert os.environ["MIGAN_TC_RESERVE_SMS"] == "3"
    finally:
        for k in keys:
            os.environ.pop(k, None)
            if saved[k] is not None:
                os.environ[k] = saved[k]

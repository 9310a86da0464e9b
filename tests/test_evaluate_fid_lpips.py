"""`python -m migan_b200.evaluate_fid_lpips` on the CPU: the reference's flags and refusals, the sorted image listing and
mask lookup, the round-robin chunking, and the round transport over gloo with stand-in chunk results (world sizes 2 and 3
deliver the chunks to rank 0 in global order, byte for byte what one process computes)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from migan_b200 import evaluate_fid_lpips as E
from migan_b200 import fid


def test_reference_flags_parse():
    a = E.get_args(["--model-name", "migan-512", "--model-path", "m.pt", "--real-dir", "real", "--mask-dir", "masks",
                    "--device", "cuda", "--batch-size", "8", "--num-workers", "4"])
    assert (a.model_name, str(a.model_path), str(a.real_dir), str(a.mask_dir)) == ("migan-512", "m.pt", "real", "masks")
    assert (a.device, a.batch_size, a.num_workers) == ("cuda", 8, 4)
    a = E.get_args(["--model-name", "comodgan-256", "--model-path", "m.pt", "--real-dir", "real", "--noise-seed", "3",
                    "--real-stats", "r.npz", "--inception-weights", "i.pth", "--lpips-weights", "l.pth"])
    assert a.mask_dir is None and a.batch_size == 32 and a.num_workers == 2 and a.noise_seed == 3
    assert str(a.real_stats) == "r.npz" and a.save_real_stats is None
    assert (str(a.inception_weights), str(a.lpips_weights)) == ("i.pth", "l.pth")
    assert [E.resolution(m) for m in ("migan-256", "migan-512", "comodgan-256", "comodgan-512")] == [256, 512, 256, 512]


def test_unknown_model_and_cpu_device_are_refused(tmp_path):
    with pytest.raises(Exception, match="Unsupported model name."):
        E.main(["--model-name", "migan-1024", "--model-path", "m.pt", "--real-dir", str(tmp_path)])
    with pytest.raises(RuntimeError, match="CUDA"):
        E.main(["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", str(tmp_path), "--device", "cpu"])
    assert E.device_for("cuda", 4, 3) == torch.device("cuda", 3)
    with pytest.raises(ValueError):
        E.device_for("cuda:1", 2, 0)


def test_listing_is_sorted_filters_suffixes_and_ignores_subdirectories(tmp_path):
    names = ["b.png", "a.jpg", "C.JPG", "d.jpeg", "e.JPEG", "f.PNG", "g.Png", "h.gif", "i.txt", "j.webp", "k"]
    for n in names:
        (tmp_path / n).write_bytes(b"")
    sub = tmp_path / "sub"
    sub.mkdir()
    (sub / "z.jpg").write_bytes(b"")
    (tmp_path / "dir.png").mkdir()
    got = [p.name for p in E.list_images(tmp_path)]
    assert got == ["C.JPG", "a.jpg", "b.png", "d.jpeg", "e.JPEG", "f.PNG"]


def test_missing_mask_is_named(tmp_path):
    real, masks = tmp_path / "real", tmp_path / "masks"
    real.mkdir()
    masks.mkdir()
    for n in ("x1.jpg", "x2.PNG"):
        (real / n).write_bytes(b"")
    (masks / "x1.png").write_bytes(b"")
    images = E.list_images(real)
    with pytest.raises(FileNotFoundError, match="x2.png"):
        E.list_masks(images, masks)
    (masks / "x2.png").write_bytes(b"")
    assert [p.name for p in E.list_masks(images, masks)] == ["x1.png", "x2.png"]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("batch", [1, 7, 32])
def test_every_image_in_one_chunk_and_equal_rounds(n, world, batch):
    chunks = E.chunk_bounds(n, batch)
    assert chunks[0][0] == 0 and chunks[-1][1] == n
    assert all(b - a == batch for a, b in chunks[:-1]) and 1 <= chunks[-1][1] - chunks[-1][0] <= batch
    assert all(chunks[i][1] == chunks[i + 1][0] for i in range(len(chunks) - 1))
    rounds = E.num_rounds(len(chunks), world)
    seen = []
    for rank in range(world):
        ran = [E.round_chunk(r, rank, len(chunks), world) for r in range(rounds)]
        assert all(j is None or j % world == rank for j in ran)
        seen += [j for j in ran if j is not None]
    assert sorted(seen) == list(range(len(chunks)))
    assert E.round_chunk(rounds, 0, len(chunks), world) is None          # nobody has a chunk after the last round
    order = [E.round_chunk(r, k, len(chunks), world) for r in range(rounds) for k in range(world)]
    assert [j for j in order if j is not None] == list(range(len(chunks)))   # rank order within a round = chunk order
    images = [i for a, b in chunks for i in range(a, b)]
    assert images == list(range(n))


def stand_in(j, chunks, real):
    """A chunk's results as a function of its global image indices: features, then the LPIPS value."""
    a, b = chunks[j]
    idx = torch.arange(a, b, dtype=torch.float32)[:, None]
    col = torch.arange(fid.FEATURES, dtype=torch.float32)[None]
    feats_r = torch.sin(idx * 0.37 + col * 0.011)
    feats_f = torch.cos(idx * 0.53 - col * 0.007) / 3
    return E.ChunkResult(j, a, feats_r if real else None, feats_f, torch.tanh(idx[:, 0] / 9))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


CASES = [(70, 8, True), (70, 32, False), (5, 2, True)]     # ragged last rounds; without real features; fewer chunks than ranks


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    for case, (n, batch, real) in enumerate(CASES):
        chunks = E.chunk_bounds(n, batch)
        width = (2 if real else 1) * fid.FEATURES + 1
        received = []
        for r in range(E.num_rounds(len(chunks), world)):
            j = E.round_chunk(r, rank, len(chunks), world)
            mine = None if j is None else stand_in(j, chunks, real)
            received += E.gather_round(mine, r, chunks, width, "cpu")
        if rank == 0:
            torch.save([tuple(c) for c in received], os.path.join(out_dir, "case%d.pt" % case))
        else:
            assert received == []
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_transport_delivers_chunks_in_global_order_gloo(tmp_path, world):
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for case, (n, batch, real) in enumerate(CASES):
        chunks = E.chunk_bounds(n, batch)
        got = torch.load(tmp_path / ("case%d.pt" % case))
        want = [stand_in(j, chunks, real) for j in range(len(chunks))]         # W = 1: the chunks as computed
        assert [c[0] for c in got] == list(range(len(chunks)))
        for g, w in zip(got, want):
            g = E.ChunkResult(*g)
            assert (g.index, g.start) == (w.index, w.start)
            assert (g.real is None) == (not real)
            if real:
                assert torch.equal(g.real, w.real)
            assert torch.equal(g.fake, w.fake) and torch.equal(g.lpips, w.lpips)
        values = np.concatenate([E.ChunkResult(*g).lpips.numpy() for g in got])
        assert values.shape == (n,) and np.array_equal(values, torch.cat([w.lpips for w in want]).numpy())

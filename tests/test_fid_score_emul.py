"""python -m migan_b200.fid_score without a GPU: the ragged uint8 input stage in the emulation build against torch, its
photo tables, the listing rule, the argument checks and planning pass, the statistics file, and the gloo transport of a
folder's features at world sizes 2 and 3."""
import ctypes
import mmap
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F
from PIL import Image
from torchvision.transforms.functional import to_tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
import migan_b200  # noqa: E402,F401
from migan_b200 import _abi, fid, fid_score  # noqa: E402
from migan_b200.demo_command import PlanError  # noqa: E402

TABLE = 64                         # include/inception_b200.h INCEPTION_U8_TABLE
SIZES = [(1, 1), (1, 37), (41, 1), (299, 299), (97, 131), (640, 480), (1200, 900)]


@pytest.fixture(scope="module")
def emul():
    path = build_emul._compile("inception_emul", [os.path.join(build_emul.CSRC, s) for s in ("inception_abi.cu", "abi_error.cu")])
    return fid.lib(ctypes.CDLL(path))


def _photos(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]


def _pack(photos, gap=0):
    """One buffer with the photos in order, `gap` bytes before each; (buffer, off, h, w)."""
    off, pos = [], 0
    for p in photos:
        pos += gap
        off.append(pos)
        pos += p.size
    buf = np.full(pos, 77, dtype=np.uint8)
    for p, o in zip(photos, off):
        buf[o:o + p.size] = p.reshape(-1)
    h = np.array([p.shape[0] for p in photos], dtype=np.int32)
    w = np.array([p.shape[1] for p in photos], dtype=np.int32)
    return buf, np.array(off, dtype=np.int64), h, w


def _input_u8(lib, base, off, h, w):
    n = len(h)
    y = torch.full((n, 299, 299, 4), -9.0)
    _abi.check(lib.inception_input_u8(base, off.ctypes.data, h.ctypes.data, w.ctypes.data, n, y.data_ptr(), None), lib)
    return y


def _torch_input(photo):
    return F.interpolate(to_tensor(photo)[None], (299, 299), mode="bilinear", align_corners=False) * 2 - 1


def test_ragged_input_matches_torch_bit_for_bit(emul):
    photos = _photos(SIZES, 0)
    buf, off, h, w = _pack(photos)
    y = _input_u8(emul, buf.ctypes.data, off, h, w)
    for i, p in enumerate(photos):
        got = y[i, ..., :3].permute(2, 0, 1)[None]
        assert torch.equal(got, _torch_input(p)), SIZES[i]
        assert (y[i, ..., 3] == 0).all()


def test_float_resize_matches_torch_bit_for_bit(emul):
    # the float path evaluates the same expression: ResizeK on ToTensor(photo) gives the same bytes
    for p in _photos(SIZES[:5], 1):
        x = to_tensor(p)[None].contiguous()
        y = torch.empty(1, 299, 299, 4)
        _abi.check(emul.inception_resize(x.data_ptr(), 1, p.shape[0], p.shape[1], y.data_ptr(), None), emul)
        assert torch.equal(y[..., :3].permute(0, 3, 1, 2), _torch_input(p))


def test_tables_span_launches_and_follow_offsets(emul):
    # TABLE + 3 photos: two launches; the photos sit behind gaps and are listed in a shuffled order
    rng = np.random.default_rng(2)
    sizes = [(int(rng.integers(1, 24)), int(rng.integers(1, 24))) for _ in range(TABLE + 3)]
    photos = _photos(sizes, 3)
    buf, off, h, w = _pack(photos, gap=5)
    order = rng.permutation(len(photos))
    y = _input_u8(emul, buf.ctypes.data, off[order], h[order], w[order])
    for k, i in enumerate(order):
        assert torch.equal(y[k, ..., :3].permute(2, 0, 1)[None], _torch_input(photos[i])), (k, i)


def test_offsets_are_64_bit(emul):
    # a base pointer 2^31 + 8 bytes before the data, so every offset is above 2^31 (the buffer is not allocated)
    photos = _photos([(3, 5), (7, 2)], 4)
    packed, off, h, w = _pack(photos)
    region = mmap.mmap(-1, packed.size)        # anonymous mappings sit far above 2^31 on x86-64 Linux
    buf = np.frombuffer(region, dtype=np.uint8)
    buf[:] = packed
    shift = 2 ** 31 + 8
    assert buf.ctypes.data > shift
    y = _input_u8(emul, buf.ctypes.data - shift, off + shift, h, w)
    del buf
    for i, p in enumerate(photos):
        assert torch.equal(y[i, ..., :3].permute(2, 0, 1)[None], _torch_input(p))


def test_workspace_does_not_depend_on_photo_sizes(emul):
    h = ctypes.c_void_p()
    _abi.check(emul.inception_create(-1, ctypes.byref(h)), emul)
    try:
        for n in (1, 3, TABLE + 1):
            u8 = emul.inception_workspace_bytes_u8(h, n)
            assert u8 > 0
            assert all(emul.inception_workspace_bytes(h, n, H, W) == u8 for H, W in ((1, 1), (97, 131), (1200, 900)))
        assert emul.inception_workspace_bytes_u8(h, 0) == 0
    finally:
        emul.inception_destroy(h)


def test_input_u8_refusals(emul):
    photos = _photos([(4, 4), (2, 3)], 5)
    buf, off, h, w = _pack(photos)
    y = torch.empty(2, 299, 299, 4)
    call = lambda o, hh, ww, n=2, base=buf.ctypes.data: emul.inception_input_u8(  # noqa: E731
        base, o.ctypes.data, hh.ctypes.data, ww.ctypes.data, n, y.data_ptr(), None)
    assert call(off, h, w) == 0
    assert call(off, h, w, n=0) == _abi.ERR_INVALID
    assert call(off, np.array([4, 0], np.int32), w) == _abi.ERR_INVALID
    assert call(off, h, np.array([-1, 3], np.int32)) == _abi.ERR_INVALID
    assert call(np.array([0, -16], np.int64), h, w) == _abi.ERR_INVALID
    assert emul.inception_input_u8(None, off.ctypes.data, h.ctypes.data, w.ctypes.data, 2, y.data_ptr(), None) == \
        _abi.ERR_INVALID
    assert emul.inception_input_u8(buf.ctypes.data, off.ctypes.data, h.ctypes.data, w.ctypes.data, 2, None, None) == \
        _abi.ERR_INVALID


# -- the command's host side ----------------------------------------------------------------------------------------

def _write(path, size=(6, 5), seed=0, fmt=None):
    rng = np.random.default_rng(seed)
    Image.fromarray(rng.integers(0, 256, size=(size[1], size[0], 3), dtype=np.uint8)).save(path, format=fmt)


def test_listing_rule(tmp_path):
    for name in ("b.png", "a.jpg", "c.jpeg", "d.bmp", "e.ppm", "f.tif", "g.tiff", "h.webp", "i.pgm",
                 "J.PNG", "k.JPG", "l.txt", "m.png.bak"):
        (tmp_path / name).write_bytes(b"x")
    (tmp_path / "sub").mkdir()
    (tmp_path / "sub" / "n.png").write_bytes(b"x")
    got = [p.name for p in fid_score.list_images(tmp_path)]
    assert got == ["a.jpg", "b.png", "c.jpeg", "d.bmp", "e.ppm", "f.tif", "g.tiff", "h.webp", "i.pgm"]


def test_argument_checks(tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir()
    b.mkdir()
    stats = tmp_path / "s.npz"
    fid_score.save_stats(stats, np.zeros(3), np.eye(3))
    with pytest.raises(RuntimeError, match="Invalid path: .*nowhere"):
        fid_score.check_paths([str(a), str(tmp_path / "nowhere")])
    for flag in ("kid", "prdc"):
        with pytest.raises(ValueError, match="--%s.*s.npz" % flag):
            fid_score.check_paths([str(a), str(stats)], **{flag: True})
    with pytest.raises(RuntimeError, match="Existing output file: .*s.npz"):
        fid_score.check_paths([str(a), str(stats)], save_stats=True)
    with pytest.raises(ValueError, match="first path must be a directory"):
        fid_score.check_paths([str(stats), str(tmp_path / "out.npz")], save_stats=True)
    fid_score.check_paths([str(a), str(stats)])
    fid_score.check_paths([str(a), str(tmp_path / "out.npz")], save_stats=True)
    with pytest.raises(SystemExit):
        fid_score.get_args([str(a), str(b), "--dims", "768"])
    with pytest.raises(ValueError, match="2048"):
        fid_score.check_dims(768)


def test_too_few_images_and_unreadable_files_are_refused_before_gpu_work(tmp_path, monkeypatch):
    def no_gpu(*a, **k):
        raise AssertionError("GPU work started before the planning pass finished")

    monkeypatch.setattr(fid_score.fid, "InceptionV3", no_gpu)
    monkeypatch.setattr(fid_score, "folder_features", no_gpu)
    one, two = tmp_path / "one", tmp_path / "two"
    one.mkdir()
    two.mkdir()
    _write(one / "a.png")
    _write(two / "a.png")
    _write(two / "b.jpg", seed=1, fmt="JPEG")
    with pytest.raises(ValueError, match="1 images"):
        fid_score.score_paths([str(two), str(one)], device="cuda")
    _write(one / "b.png", seed=2)
    (one / "c.png").write_bytes(b"not a png")
    (two / "d.webp").write_bytes(b"")
    with pytest.raises(PlanError) as e:
        fid_score.score_paths([str(two), str(one)], device="cuda")
    assert len(e.value.problems) == 2
    assert "d.webp" in e.value.problems[0] and "c.png" in e.value.problems[1]


def test_stats_file_round_trip(tmp_path):
    rng = np.random.default_rng(6)
    x = rng.normal(size=(40, 8))
    mu, sigma = x.mean(0), np.cov(x, rowvar=False)
    path = tmp_path / "stats.npz"
    fid_score.save_stats(path, mu, sigma)
    with np.load(path) as f:
        assert sorted(f.files) == ["mu", "sigma"] and f["mu"].dtype == np.float64
    m2, s2 = fid_score.load_stats(path)
    assert np.array_equal(m2, mu) and np.array_equal(s2, sigma)
    assert fid_score.folder_statistics(str(path))[0].tobytes() == mu.tobytes()


# -- the gloo transport -----------------------------------------------------------------------------------------------

class StandIn:
    """A deterministic stand-in for InceptionV3.features_u8 on the CPU: each row depends on its own photo only."""

    def features_u8(self, photos, device):
        col = torch.arange(fid.FEATURES, dtype=torch.float64)
        rows = []
        for p in photos:
            t = torch.from_numpy(p.astype(np.float64))
            rows.append(torch.sin(col * t.mean() / 97 + p.shape[0] * 0.3 + p.shape[1] * 0.7) * t.std())
        return torch.stack(rows).float().to(device)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


BATCHES = (3, 4, 32)


def _worker(rank, world, port, folder, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    files = fid_score.plan_folder(folder)
    for batch in BATCHES:
        got = fid_score.folder_features(files, StandIn(), batch, "cpu", num_workers=2).features
        if rank == 0:
            torch.save(got, os.path.join(out_dir, "b%d.pt" % batch))
        else:
            assert got is None
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_features_equal_one_process(tmp_path, world):
    folder = tmp_path / "imgs"
    folder.mkdir()
    rng = np.random.default_rng(7)
    for k in range(11):
        size = (int(rng.integers(1, 40)), int(rng.integers(1, 40)))
        _write(folder / ("%02d.png" % k), size=size, seed=k)
    files = fid_score.plan_folder(folder)
    want = fid_score.folder_features(files, StandIn(), 5, "cpu").features
    assert want.shape == (11, fid.FEATURES)
    out = tmp_path / "out"
    out.mkdir()
    mp.spawn(_worker, args=(world, _free_port(), str(folder), str(out)), nprocs=world, join=True)
    for batch in BATCHES:
        assert torch.equal(torch.load(out / ("b%d.pt" % batch)), want), batch

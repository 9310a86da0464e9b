"""python -m migan_b200.fid_score on the H100: `InceptionV3.features_u8` against the float path bit for bit, at any batch
size; the command's FID, KID and manifold-metric lines against the library on the float path's features; the stored
statistics; the launches of the uint8 path."""
import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image
from torchvision.transforms.functional import to_tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import migan_b200  # noqa: E402,F401
from migan_b200 import _abi, fid, fid_score, prdc  # noqa: E402
from migan_b200 import kid as kid_metric  # noqa: E402
from oracle import fid_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TABLE = 64                         # include/inception_b200.h INCEPTION_U8_TABLE


@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


@pytest.fixture(scope="module")
def net(sd):
    return fid.InceptionV3(weights=sd)


@pytest.fixture(scope="module")
def weights_file(sd, tmp_path_factory):
    path = tmp_path_factory.mktemp("w") / "inception.pth"
    torch.save(sd, path)
    return path


def _photos(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]


def _float_features(net, photos):
    return torch.cat([net(to_tensor(p)[None].to(DEV))[0].view(1, fid.FEATURES) for p in photos])


MIXED = [(1, 1), (1, 37), (41, 1), (299, 299), (97, 131), (640, 480), (1200, 900), (256, 256), (512, 512)]


def test_device_input_stages_match_torch_cpu_bit_for_bit():
    photos = _photos(MIXED, 0)
    sizes = np.array([p.size for p in photos], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(sizes[:-1])]).astype(np.int64)
    h = np.array([p.shape[0] for p in photos], dtype=np.int32)
    w = np.array([p.shape[1] for p in photos], dtype=np.int32)
    packed = torch.from_numpy(np.concatenate([p.reshape(-1) for p in photos])).to(DEV)
    y = torch.empty(len(photos), 299, 299, 4, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    _abi.check(fid.lib().inception_input_u8(packed.data_ptr(), off.ctypes.data, h.ctypes.data, w.ctypes.data,
                                            len(photos), y.data_ptr(), stream))
    got = y.cpu()
    for i, p in enumerate(photos):
        x = to_tensor(p)[None]
        want = F.interpolate(x, (299, 299), mode="bilinear", align_corners=False) * 2 - 1
        assert torch.equal(got[i, ..., :3].permute(2, 0, 1)[None], want), MIXED[i]
        assert (got[i, ..., 3] == 0).all()
        yf = torch.empty(1, 299, 299, 4, device=DEV)
        _abi.check(fid.lib().inception_resize(x.to(DEV).data_ptr(), 1, p.shape[0], p.shape[1], yf.data_ptr(), stream))
        assert torch.equal(yf.cpu()[0], got[i]), MIXED[i]


def test_features_u8_equal_the_float_path_at_any_batch_size(net):
    rng = np.random.default_rng(1)
    sizes = MIXED + [(int(rng.integers(1, 400)), int(rng.integers(1, 400))) for _ in range(TABLE + 5 - len(MIXED))]
    photos = _photos(sizes, 2)
    full = net.features_u8(photos)
    assert full.shape == (len(photos), fid.FEATURES) and full.dtype == torch.float32 and full.is_cuda
    assert net.last_launch_count() == 108 + 2                    # two input tables, then the float walk's 108
    assert torch.equal(full, _float_features(net, photos))
    for bs in (1, 3, 64):
        got = torch.cat([net.features_u8(photos[a:a + bs]) for a in range(0, len(photos), bs)])
        assert torch.equal(got, full), bs
    assert net.features_u8([]).shape == (0, fid.FEATURES)
    with pytest.raises(ValueError, match="photo 1"):
        net.features_u8([photos[0], photos[1][..., :2]])


def test_profiler_shows_one_input_launch_per_table(net):
    photos = _photos([(50 + k, 70 + 2 * k) for k in range(TABLE + 1)], 3)
    net.features_u8(photos)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        pad = torch.zeros(1, device=DEV)            # lead with uncounted kernels (see test_fid_gpu)
        for _ in range(256):
            pad.add_(1)
        torch.cuda.synchronize()
        net.features_u8(photos)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
    ours = sorted((e for e in kernels if "incep" in e.name or "ck_items_kernel" in e.name), key=lambda e: e.time_range.start)
    assert len(ours) == net.last_launch_count() == 110
    assert all("ResizeU8K" in e.name for e in ours[:2])
    assert not any("ResizeU8K" in e.name or "ResizeK" in e.name for e in ours[2:])


def _folder(path, sizes, seed, fmt):
    path.mkdir()
    for k, p in enumerate(_photos(sizes, seed)):
        Image.fromarray(p).save(path / ("%03d.%s" % (k, fmt)))
    return [fid_score.E.decode_photo(f) for f in fid_score.list_images(path)]


@pytest.fixture(scope="module")
def folders(tmp_path_factory):
    root = tmp_path_factory.mktemp("folders")
    rng = np.random.default_rng(4)
    sa = [(int(rng.integers(40, 500)), int(rng.integers(40, 500))) for _ in range(37)]
    sb = [(int(rng.integers(40, 500)), int(rng.integers(40, 500))) for _ in range(29)]
    return (root / "a", _folder(root / "a", sa, 5, "png")), (root / "b", _folder(root / "b", sb, 6, "jpg"))


def _run(argv):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        fid_score.main(argv)
    return out.getvalue().splitlines()


def test_command_lines_equal_the_library_on_float_features(net, folders, weights_file):
    (a, pa), (b, pb) = folders
    fa, fb = _float_features(net, pa), _float_features(net, pb)
    sa, sb = fid.FeatureStatistics(device=DEV), fid.FeatureStatistics(device=DEV)
    sa.add(fa)
    sb.add(fb)
    want_fid = sa.frechet_distance(sb)
    lines = _run([str(a), str(b), "--inception-weights", str(weights_file), "--batch-size", "8", "--num-workers", "3",
                  "--kid", "--prdc"])
    k = kid_metric.kernel_inception_distance(fa, fb).kid
    r = prdc.precision_recall_density_coverage(fa, fb, k=3)
    assert lines == ["FID:  %s" % want_fid, "KID: %r" % float(k), "Precision: %r" % float(r.precision),
                     "Recall: %r" % float(r.recall), "Density: %r" % float(r.density),
                     "Coverage: %r" % float(r.coverage)]
    for bs in (1, 50):
        got = fid_score.score_paths([str(a), str(b)], batch_size=bs, device=DEV, model=net)
        assert got.fid == want_fid, bs


def test_folder_against_itself_is_zero(net, folders):
    (a, _), _ = folders
    got = fid_score.score_paths([str(a), str(a)], device=DEV, model=net).fid
    mu, sigma = fid_score.folder_statistics(str(a), net, device=DEV)
    assert abs(got) <= 1e-6 * 2 * np.trace(sigma), got


def test_saved_stats_stand_in_for_the_folder(net, folders, weights_file, tmp_path):
    (a, _), (b, _) = folders
    out = tmp_path / "a_stats.npz"
    assert _run(["--save-stats", str(a), str(out), "--inception-weights", str(weights_file), "--batch-size", "7"]) == []
    mu, sigma = fid_score.load_stats(out)
    assert mu.shape == (2048,) and sigma.shape == (2048, 2048)
    folder = fid_score.score_paths([str(a), str(b)], device=DEV, model=net).fid
    assert fid_score.score_paths([str(out), str(b)], device=DEV, model=net).fid == folder
    with pytest.raises(RuntimeError, match="Existing output file"):
        _run(["--save-stats", str(a), str(out), "--inception-weights", str(weights_file)])

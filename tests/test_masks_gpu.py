"""GPU checks of `RandomMaskStream` and `python -m migan_b200.generate_masks` against the reference's masks
(tests/golden/masks.npz, drawn by scripts/generate_masks.py's RandomMask): bytes, attempts and numpy state, for
several ways of splitting the stream, repeated planning at s = 32, the 2000-mask digest stream at 512, and the files the
command writes."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import masks_oracle as M  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "masks.npz"))


def golden_masks(seed, s):
    bits = GOLDEN["m%d_%d" % (seed, s)]
    return np.where(np.unpackbits(bits, axis=1, count=s * s).reshape(-1, s, s) == 1, 255, 0).astype(np.uint8)


def golden_state(prefix):
    rest = GOLDEN[prefix + "_rest"]
    return ("MT19937", GOLDEN[prefix + "_state"], int(rest[0]), int(rest[1]), float(rest[2]))


def assert_state(got, want):
    assert got[0] == want[0]
    np.testing.assert_array_equal(got[1], want[1])
    assert tuple(got[2:]) == tuple(want[2:])


def take(stream, n, split):
    parts, left = [], n
    while left:
        k = min(split, left)
        m = stream.next(k)
        assert m.is_cuda and m.dtype == torch.uint8 and tuple(m.shape) == (k, stream.resolution, stream.resolution)
        parts.append(m.cpu().numpy())
        left -= k
    return np.concatenate(parts)


@pytest.mark.parametrize("split", [1, 7, 32, 100])
@pytest.mark.parametrize("seed,s", [(0, 64), (0, 256), (7, 128)])
def test_next_equals_fixture(lib, cuda_device, seed, s, split):
    import migan_b200
    want = golden_masks(seed, s)
    stream = migan_b200.RandomMaskStream(s, seed=seed, device=cuda_device)
    np.testing.assert_array_equal(take(stream, len(want), split), want)
    assert stream.attempts == int(GOLDEN["m%d_%d_attempts" % (seed, s)])
    assert_state(stream.get_state(), golden_state("m%d_%d" % (seed, s)))


@pytest.mark.parametrize("split", [1, 7, 32, 200])
def test_s32_repeated_planning(lib, cuda_device, split):
    """At s = 32 about two attempts in three are all-hole, so a call plans again until it has its masks."""
    import migan_b200
    want = golden_masks(0, 32)
    stream = migan_b200.RandomMaskStream(32, seed=0, device=cuda_device)
    np.testing.assert_array_equal(take(stream, len(want), split), want)
    assert stream.attempts == int(GOLDEN["m0_32_attempts"])
    assert_state(stream.get_state(), golden_state("m0_32"))


def test_s512_and_out(lib, cuda_device):
    import migan_b200
    want = golden_masks(0, 512)
    stream = migan_b200.RandomMaskStream(512, seed=0, device=cuda_device)
    out = torch.full((len(want), 512, 512), 7, dtype=torch.uint8, device=cuda_device)
    assert stream.next(len(want), out=out) is out
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    assert_state(stream.get_state(), golden_state("m0_512"))


@pytest.mark.parametrize("s,batch", [(512, 256), (256, 100)])
def test_digest_stream(lib, cuda_device, s, batch):
    import migan_b200
    want = GOLDEN["digest0_%d" % s]
    stream = migan_b200.RandomMaskStream(s, seed=0, device=cuda_device)
    got = take(stream, len(want), batch)
    digests = np.frombuffer(b"".join(M.digest(m) for m in got), np.uint8).reshape(-1, 8)
    np.testing.assert_array_equal(digests, want)
    assert stream.attempts == int(GOLDEN["digest0_%d_attempts" % s])
    assert_state(stream.get_state(), golden_state("digest0_%d" % s))


def test_set_state_continues_numpy(lib, cuda_device):
    """A stream set to numpy's state after k RandomMask calls continues with mask k."""
    import migan_b200
    want = golden_masks(0, 64)
    rs = np.random.RandomState(0)
    M.random_masks(64, 30, rs=rs)
    stream = migan_b200.RandomMaskStream(64, seed=123, device=cuda_device)
    stream.set_state(rs.get_state())
    np.testing.assert_array_equal(stream.next(70).cpu().numpy(), want[30:])
    assert_state(stream.get_state(), golden_state("m0_64"))


def test_refusals(lib, cuda_device):
    import migan_b200
    for s in (1, 4097):
        with pytest.raises(ValueError):
            migan_b200.RandomMaskStream(s, device=cuda_device)
    stream = migan_b200.RandomMaskStream(64, device=cuda_device)
    with pytest.raises(ValueError):
        stream.next(2, out=torch.empty((2, 64, 63), dtype=torch.uint8, device=cuda_device))
    assert stream.next(0).shape == (0, 64, 64) and stream.attempts == 0


def test_generate_masks_files(lib, cuda_device, tmp_path):
    from PIL import Image

    from migan_b200 import generate_masks
    images = tmp_path / "images"
    names = ["b/z.png", "a.jpg", "a/c.jpeg", "b/y/x.jpg", "q.png", "skip.JPG", "skip.txt", "skip.webp"]
    for name in names:
        p = images / name
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(b"not read")
    out = tmp_path / "masks"
    generate_masks.main(["--images-dir", str(images), "--output-dir", str(out), "--resolution", "64"])
    order = sorted(str(images / n) for n in names if not n.startswith("skip"))
    stems = [os.path.splitext(os.path.basename(p))[0] for p in order]
    assert sorted(os.listdir(out)) == sorted(s + ".png" for s in stems)
    want = golden_masks(0, 64)
    for k, stem in enumerate(stems):
        img = Image.open(out / (stem + ".png"))
        assert img.mode == "L"
        np.testing.assert_array_equal(np.asarray(img), want[k], err_msg=stem)

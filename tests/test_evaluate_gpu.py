"""GPU checks of `EvalPipeline` (scripts/evaluate_fid_lpips.py's batch around the generator) against a torch-CPU
restatement of `InferenceDataset.__getitem__` (PIL resizes, `mask // 255`, x) and of :246-249 (composite and
normalisations), applied to the same generator output: bit for bit, for photos at, above and below R x R (and mixed), for
directory masks of other sizes and generated masks (tests/golden/masks.npz, the reference's RandomMask), over two passes.
The launch count per pass is stated by `EvalPipeline.pass_launches` and checked with torch.profiler."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import migan_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

R = 64
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "masks.npz"))


def golden_masks(seed, s):
    bits = GOLDEN["m%d_%d" % (seed, s)]
    return np.where(np.unpackbits(bits, axis=1, count=s * s).reshape(-1, s, s) == 1, 255, 0).astype(np.uint8)


def dataset_item(img, mask, from_dir):
    """InferenceDataset.__getitem__ on a decoded photo and mask: (x, img, mask) as the script's tensors."""
    from PIL import Image
    im = Image.fromarray(img).convert("RGB")
    if im.size[0] != R or im.size[1] != R:
        im = im.resize((R, R), Image.BICUBIC)
    mk = Image.fromarray(mask).convert("L")
    if from_dir:
        mk = mk.resize((R, R), Image.NEAREST)
    a = np.array(im)
    m = np.array(mk)[:, :, np.newaxis] // 255
    a = torch.Tensor(a).float() * 2 / 255 - 1
    m = torch.Tensor(m).float()
    a = a.permute(2, 0, 1)
    m = m.permute(2, 0, 1)
    return torch.cat([m - 0.5, a * m], dim=0), a, m


def reference(pipe, imgs, masks, from_dir):
    items = [dataset_item(i, m, from_dir) for i, m in zip(imgs, masks)]
    reals, composeds = [], []
    for c in range(0, len(items), 32):
        x = torch.stack([t[0] for t in items[c:c + 32]])
        im = torch.stack([t[1] for t in items[c:c + 32]])
        mk = torch.stack([t[2] for t in items[c:c + 32]])
        y = pipe.model(x.cuda()).cpu()
        composed = mk * im + (1 - mk) * y
        reals.append((im * 0.5 + 0.5).clamp(0, 1))
        composeds.append((composed * 0.5 + 0.5).clamp(0, 1))
    return torch.cat(reals), torch.cat(composeds)


def photos(rng, sizes):
    return [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in sizes]


@pytest.fixture(scope="module")
def pipe_factory(lib, cuda_device):
    import migan_b200
    sd = O.make_state_dict(R, seed=1)
    return lambda: migan_b200.EvalPipeline(sd, R, device=cuda_device, seed=0)


SIZES = [(64, 64), (100, 80), (40, 30), (64, 200), (50, 64), (17, 300), (333, 64)]


def test_directory_masks(pipe_factory):
    rng = np.random.RandomState(0)
    imgs = photos(rng, SIZES * 5)                                   # 35 images: two passes
    masks = []
    for k in range(len(imgs)):
        h, w = [(64, 64), (96, 70), (30, 41), (64, 64)][k % 4]
        m = np.where(rng.rand(h, w) < 0.3, 0, 255).astype(np.uint8)
        m[rng.rand(h, w) < 0.05] = 254                              # // 255 -> 0: a hole
        masks.append(m)
    pipe = pipe_factory()
    real, composed = pipe.forward_batch(imgs, masks)
    assert real.is_cuda and real.dtype == torch.float32 and tuple(real.shape) == (len(imgs), 3, R, R)
    want_real, want_composed = reference(pipe, imgs, masks, True)
    assert torch.equal(real.cpu(), want_real)
    assert torch.equal(composed.cpu(), want_composed)
    assert len(pipe.last_launches) == 2


def test_generated_masks(pipe_factory):
    rng = np.random.RandomState(1)
    want_masks = golden_masks(0, R)
    pipe = pipe_factory()
    got_r, got_c, all_imgs = [], [], []
    for n in (5, 40):                                               # the stream carries over between calls
        imgs = photos(rng, [SIZES[k % len(SIZES)] for k in range(n)])
        r, c = pipe.forward_batch(imgs)
        got_r.append(r.cpu())
        got_c.append(c.cpu())
        all_imgs += imgs
    want_r, want_c = [], []
    for lo, hi in ((0, 5), (5, 45)):
        r, c = reference(pipe, all_imgs[lo:hi], list(want_masks[lo:hi]), False)
        want_r.append(r)
        want_c.append(c)
    for g, w in zip(got_r + got_c, want_r + want_c):
        assert torch.equal(g, w)
    import migan_b200
    alone = migan_b200.RandomMaskStream(R, seed=0)
    alone.next(45)
    assert pipe.masks.attempts == alone.attempts
    np.testing.assert_array_equal(pipe.masks.get_state()[1], alone.get_state()[1])


def test_photos_at_resolution_only(pipe_factory):
    rng = np.random.RandomState(2)
    imgs = photos(rng, [(R, R)] * 3)
    masks = [np.full((R, R), 255, np.uint8), np.zeros((R, R), np.uint8), golden_masks(0, R)[7]]
    pipe = pipe_factory()
    real, composed = pipe.forward_batch(imgs, masks)
    want_real, want_composed = reference(pipe, imgs, masks, True)
    assert torch.equal(real.cpu(), want_real) and torch.equal(composed.cpu(), want_composed)
    assert torch.equal(composed[0], real[0])                        # all known: the photo itself


@pytest.mark.parametrize("sizes", [[(R, R)] * 4, [(R, R), (80, 90)]])
def test_launch_count(pipe_factory, sizes):
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.RandomState(3)
    imgs = photos(rng, sizes)
    masks = [np.full((R, R), 255, np.uint8)] * len(imgs)
    pipe = pipe_factory()
    pipe.forward_batch(imgs, masks)                                 # warm-up: plans and modules
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.forward_batch(imgs, masks)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    resized = any(s != (R, R) for s in sizes)
    assert pipe.last_launches == [pipe.pass_launches(resized, pipe.model.last_launch_count())]
    assert pipe.last_launches[0] == (4 if resized else 2) + pipe.model.last_launch_count() + 1
    assert len(kernels) == pipe.last_launches[0], sorted({e.name for e in kernels})


def test_refusals(pipe_factory):
    pipe = pipe_factory()
    with pytest.raises(ValueError):
        pipe.forward_batch([np.zeros((8, 8), np.uint8)])
    with pytest.raises(ValueError):
        pipe.forward_batch([np.zeros((8, 8, 3), np.uint8)], [np.zeros((8, 8, 3), np.uint8)])
    with pytest.raises(ValueError):
        pipe.forward_batch([np.zeros((8, 8, 3), np.uint8)] * 2, [np.zeros((8, 8), np.uint8)])

"""Co-Mod-GAN through the request pipelines on the H100: the seeded noise against numpy's Philox
(oracle/comodgan_noise_oracle.py), `forward(seeds=...)` against the RANDOM-mode forward on the same draws, determinism,
and `EvalPipeline` / `DemoPipeline` with comodgan-256 against their torch-CPU and numpy restatements on the same generator
output, bit for bit.  Weights are the seeded ones of oracle/comodgan_oracle.make_state_dict.

The forward is not batch invariant: the demodulated layers scale the styles by one RMS over the whole batch
(stylegan.py:146, `InvRmsAllK`).  A request's draws are, so its bytes are the same for the same chunking and within
rounding otherwise."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import comodgan_noise_oracle as N  # noqa: E402
from oracle import comodgan_oracle as C  # noqa: E402
from oracle import demo_oracle as D  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-3          # tests/test_comodgan_gpu.py's Co-Mod-GAN tolerance


def _ulps(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    g, w = got.astype(np.float32).view(np.int32).astype(np.int64), want.astype(np.float32).view(np.int32).astype(np.int64)
    g = np.where(g < 0, -(g & 0x7FFFFFFF), g)
    w = np.where(w < 0, -(w & 0x7FFFFFFF), w)
    return np.abs(g - w)


@pytest.fixture(scope="module")
def gen256(lib, cuda_device):
    from migan_b200 import comodgan
    sd = C.make_state_dict(256, seed=1)
    return comodgan.load(sd, 256).to(cuda_device), sd


def test_device_noise_against_numpy(gen256):
    g, _ = gen256
    seeds = [0, 1, 2 ** 32 + 5, 2 ** 64 - 1, 987654321]
    z, planes = g.seeded_noise(seeds)
    z_or, planes_or = N.seeded_noise(seeds, 256)
    dz, dp = _ulps(z.cpu().numpy(), z_or), _ulps(planes.cpu().numpy(), planes_or)
    print("device noise: %d of %d values differ from numpy by one float32 ulp"
          % (int((dz != 0).sum() + (dp != 0).sum()), dz.size + dp.size))
    assert int(dz.max()) <= 1 and int(dp.max()) <= 1
    # a request's draws do not depend on the call
    z1, p1 = g.seeded_noise(seeds[3:4])
    assert torch.equal(z1[0], z[3])
    off = 0
    for r in N.plane_res(256):
        assert torch.equal(planes[off * 5 + 3 * r * r:off * 5 + 4 * r * r], p1[off:off + r * r])
        off += r * r


def test_forward_seeds_equals_random_mode_and_repeats(gen256, cuda_device):
    g, _ = gen256
    x = O.make_input(256, 5, seed=31).to(cuda_device)
    seeds = [11, 12, 13, 14, 15]
    y = g(x, seeds=seeds)
    z, planes = g.seeded_noise(seeds)
    assert torch.equal(y, g(x, z=z, noise=planes))
    assert torch.equal(y, g(x, seeds=seeds))                       # two calls, the same bytes
    assert torch.equal(y, g(x, z=z, seeds=seeds))
    # batch coupling: alone, request 3 gets its own draws and rounding-level differences only
    y1 = g(x[3:4], seeds=seeds[3:4])
    err = float((y1[0] - y[3]).abs().max())
    print("request 3 alone vs at position 3 of 5: max-abs %.3e (bitwise equal: %s)" % (err, bool(torch.equal(y1[0], y[3]))))
    assert err < TOL


def dataset_item(img, mask, from_dir, R):
    """InferenceDataset.__getitem__ on a decoded photo and mask (as in tests/test_evaluate_gpu.py)."""
    from PIL import Image
    im = Image.fromarray(img).convert("RGB")
    if im.size[0] != R or im.size[1] != R:
        im = im.resize((R, R), Image.BICUBIC)
    mk = Image.fromarray(mask).convert("L")
    if from_dir:
        mk = mk.resize((R, R), Image.NEAREST)
    a = torch.Tensor(np.array(im)).float() * 2 / 255 - 1
    m = torch.Tensor(np.array(mk)[:, :, np.newaxis] // 255).float()
    a, m = a.permute(2, 0, 1), m.permute(2, 0, 1)
    return torch.cat([m - 0.5, a * m], dim=0), a, m


def generator_chunks(model, x, seeds, gb):
    return torch.cat([model(x[c:c + gb], seeds=seeds[c:c + gb]) for c in range(0, x.shape[0], gb)])


@pytest.mark.parametrize("from_dir", [True, False])
def test_eval_pipeline_comodgan_256(gen256, cuda_device, from_dir):
    import migan_b200
    g, _ = gen256
    R, gb = 256, 4
    rng = np.random.RandomState(5)
    sizes = [(256, 256), (300, 200), (120, 256), (256, 256), (64, 80), (256, 511)]
    imgs = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in sizes]
    pipe = migan_b200.EvalPipeline(g, R, device=cuda_device, seed=0, noise_seed=3, generator_batch=gb)
    if from_dir:
        masks = [np.where(rng.rand(200, 150) < 0.3, 0, 255).astype(np.uint8) for _ in imgs]
        real, composed = pipe.forward_batch(imgs, masks)
    else:
        masks = list(migan_b200.RandomMaskStream(R, seed=0, device=cuda_device).next(len(imgs)).cpu().numpy())
        real, composed = pipe.forward_batch(imgs)
    assert pipe.noise_index == len(imgs)
    seeds = np.array([(3 << 32) + k for k in range(len(imgs))], np.uint64)
    items = [dataset_item(i, m, from_dir, R) for i, m in zip(imgs, masks)]
    x = torch.stack([t[0] for t in items])
    im = torch.stack([t[1] for t in items])
    mk = torch.stack([t[2] for t in items])
    y = generator_chunks(g, x.to(cuda_device), seeds, gb).cpu()
    assert torch.equal(real.cpu(), (im * 0.5 + 0.5).clamp(0, 1))
    assert torch.equal(composed.cpu(), ((mk * im + (1 - mk) * y) * 0.5 + 0.5).clamp(0, 1))
    # the launch record: the pass's stages around the generator's chunks, each with its noise launch
    assert pipe.last_launches[0] > 2 * 50
    # explicit seeds: the same bytes; a MI-GAN-only argument is refused on MI-GAN
    pipe.noise_index = 0
    if from_dir:
        real2, composed2 = pipe.forward_batch(imgs, masks, seeds=seeds)
        assert torch.equal(composed2, composed) and pipe.noise_index == 0


def test_demo_pipeline_comodgan_256(gen256, cuda_device):
    from migan_b200.demo import DemoPipeline
    g, _ = gen256
    res, gb = 256, 3
    rng = np.random.default_rng(8)
    reqs = []
    for W, H in [(256, 256), (400, 300), (200, 120), (256, 700), (90, 90)]:
        img = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
        mask = np.where(rng.random((H, W)) < 0.3, 0, 255).astype(np.uint8)
        reqs.append((img, mask))
    pipe = DemoPipeline(g, res, device=cuda_device, noise_seed=1, generator_batch=gb)
    got = pipe.forward_batch([r[0] for r in reqs], [r[1] for r in reqs])
    seeds = np.array([(1 << 32) + k for k in range(len(reqs))], np.uint64)
    pre = [D.demo_pre(img, mask, False, res) for img, mask in reqs]
    x = torch.from_numpy(np.stack([p[2] for p in pre])).to(cuda_device)
    y = generator_chunks(g, x, seeds, gb).cpu().numpy()
    for k, (rs, m, _) in enumerate(pre):
        assert np.array_equal(got[k], D.demo_post(y[k], rs, m)), k
    assert pipe.noise_index == len(reqs)
    # wait=False: the seeds are kernel parameters, nothing waits; the same seeds give the same bytes
    imgs_t = [torch.from_numpy(r[0]).pin_memory() for r in reqs]
    outs = pipe.forward_batch(imgs_t, [r[1] for r in reqs], wait=False, seeds=seeds)
    pipe.wait()
    for k in range(len(reqs)):
        assert np.array_equal(outs[k].numpy(), got[k]), k
    # generator_batch: one chunk of five against chunks of three, within rounding (the style RMS couples a chunk)
    pipe5 = DemoPipeline(g, res, device=cuda_device, noise_seed=1, generator_batch=5)
    got5 = pipe5.forward_batch([r[0] for r in reqs], [r[1] for r in reqs])
    diff = max(int(np.abs(a.astype(np.int16) - b.astype(np.int16)).max()) for a, b in zip(got, got5))
    print("DemoPipeline comodgan-256: generator_batch 3 vs 5: max uint8 difference %d" % diff)
    assert diff <= 2


def test_migan_pipelines_refuse_seeds(lib, cuda_device):
    import migan_b200
    from migan_b200.demo import DemoPipeline
    sd = O.make_state_dict(64, seed=1)
    pipe = migan_b200.EvalPipeline(sd, 64, device=cuda_device)
    img = np.zeros((64, 64, 3), np.uint8)
    with pytest.raises(ValueError):
        pipe.forward_batch([img], seeds=[1])
    demo = DemoPipeline(sd, 64, device=cuda_device)
    with pytest.raises(ValueError):
        demo.forward_batch([img], [np.full((64, 64), 255, np.uint8)], seeds=[1])


def test_comodgan_512_seeded_against_oracle(lib, cuda_device):
    from migan_b200 import comodgan
    sd = C.make_state_dict(512, seed=2)
    g = comodgan.load(sd, 512).to(cuda_device)
    assert g.num_ws == 16
    x = O.make_input(512, 2, seed=3)
    seeds = [21, 2 ** 64 - 2]
    y = g(x.to(cuda_device), seeds=seeds).cpu()
    z_or, planes_or = N.seeded_noise(seeds, 512)
    noise = {k: torch.from_numpy(v) for k, v in N.plane_dict(planes_or, C.noise_keys(512), 2).items()}
    want = C.generator_forward(sd, x, torch.from_numpy(z_or), 512, noise_mode="random", noise=noise)
    err = (y - want).abs()
    print("comodgan-512 n=2 seeded: max-abs %.3e mean-abs %.3e" % (float(err.max()), float(err.mean())))
    assert float(err.max()) < TOL

"""`CropPipeline` and `python -m migan_b200.crop_results` on the H100.

* `CropPipeline(img, mask, invert)` equals `MIGAN_Pipeline` on the photo transposed to [3,H,W] and create_onnx_pipeline.py's
  `read_mask(mask, invert)`, byte for byte and with the same `last_boxes`: numpy, CPU, pinned and CUDA photos; masks of 1
  to 4 channels, larger, smaller and of the photo's size; one call, splits of it, and `wait=False` / `wait()`;
* the stored reference vectors (tests/golden/pipeline.npz, the cases with binary masks) reproduce through it;
* Co-Mod-GAN (comodgan-256, seeded) in both crop classes equals a hand composition byte for byte: the oracle's
  pre-processing of the crop, the GPU seeded forward on that x in the same generator chunks, the oracle's
  post-processing and blend; a refused call takes no seeds;
* the command's files equal a per-photo restatement of the reference loop through `MIGAN_Pipeline`, are the same bytes
  at virtual W = 1, 2 and 3 and at --batch-size 8 and 32, and comodgan-256 runs through the command."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from oracle import comodgan_oracle as CO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402
from oracle import pipeline_oracle as PO  # noqa: E402
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)

pytestmark = pytest.mark.gpu
R = 256


def read_mask(mask: np.ndarray, invert: bool) -> np.ndarray:
    """create_onnx_pipeline.py:27-45 on a decoded mask array: the [h,w] plane `.convert("L")` gives."""
    from PIL import Image
    if mask.ndim == 3:
        v = mask[:, :, {4: 3, 2: 1, 3: 0, 1: 0}[mask.shape[2]]]
    else:
        v = mask
    v = np.dstack([v, v, v])
    if invert:
        v = 255 - v
    v[v < 255] = 0
    return np.array(Image.fromarray(v).convert("L"))


def reference_call(pipe, img: np.ndarray, mask: np.ndarray, invert: bool) -> np.ndarray:
    """The reference loop's pipeline call (create_onnx_pipeline.py:336-341 with its torch line) through MIGAN_Pipeline."""
    image = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1)[None]))
    m = torch.from_numpy(read_mask(mask, invert)[None, None])
    return pipe(image, m)[0].numpy().transpose(1, 2, 0)


@pytest.fixture(scope="module")
def migan(lib, cuda_device):
    from migan_b200.generator import Generator
    g = Generator(resolution=R)
    g.load_state_dict(MO.make_state_dict(R, seed=3))
    return g.to(cuda_device).eval()


def _requests(rng, n):
    """Photos of odd sizes with local holes; masks of 1 to 4 channels, at, above and below the photo's size."""
    out = []
    for i in range(n):
        H, W = int(rng.integers(3, 700)), int(rng.integers(3, 700))
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        C = 1 + i % 4
        scale = [1.0, 1.7, 0.4][i % 3]
        hm, wm = max(1, int(H * scale)), max(1, int(W * scale))
        v = np.full((hm, wm), 255, np.uint8)
        if i % 5 != 4:
            a, b = sorted(rng.integers(0, hm, 2)); c, d = sorted(rng.integers(0, wm, 2))
            v[a:b + 1, c:d + 1] = 0
        v[rng.random((hm, wm)) < 0.002] = 128
        if C == 1:
            mask = v if i % 2 else v[:, :, None]
        else:
            mask = rng.integers(0, 256, (hm, wm, C), dtype=np.uint8)
            mask[:, :, {4: 3, 2: 1, 3: 0}[C]] = v
        out.append((img, np.ascontiguousarray(mask)))
    return out


@pytest.mark.parametrize("invert", [False, True], ids=["plain", "inverted"])
def test_crop_pipeline_equals_migan_pipeline(migan, cuda_device, invert):
    from migan_b200.pipeline import CropPipeline, MIGAN_Pipeline
    rng = np.random.default_rng(5 + invert)
    reqs = _requests(rng, 37)                           # two passes: 32 + 5
    ref = MIGAN_Pipeline(migan, R, device=cuda_device)
    want, boxes = [], []
    for img, mask in reqs:
        want.append(reference_call(ref, img, mask, invert))
        boxes.append(ref.last_box)
    pipe = CropPipeline(migan, R, device=cuda_device)
    imgs = [img for img, _ in reqs]
    masks = [m for _, m in reqs]
    before = [img.copy() for img in imgs]
    got = pipe.forward_batch(imgs, masks, invert=invert)
    assert all(isinstance(g, np.ndarray) for g in got)
    assert all(np.array_equal(a, b) for a, b in zip(imgs, before))          # the caller's photos are not written
    for i, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), i
    assert pipe.last_boxes == boxes
    # one request at a time, and splits of the call
    assert np.array_equal(pipe(imgs[3], masks[3], invert), want[3]) and pipe.last_boxes == [boxes[3]]
    for a, b in ((0, 1), (1, 20), (20, 37)):
        got = pipe.forward_batch(imgs[a:b], masks[a:b], invert=[invert] * (b - a))
        assert all(np.array_equal(g, w) for g, w in zip(got, want[a:b])) and pipe.last_boxes == boxes[a:b]
    # CPU, pinned and CUDA tensors; wait=False then wait()
    cpu = [torch.from_numpy(img) for img in imgs[:6]]
    got = pipe.forward_batch(cpu, masks[:6], invert)
    assert all(isinstance(g, torch.Tensor) and not g.is_cuda for g in got)
    assert all(np.array_equal(g.numpy(), w) for g, w in zip(got, want[:6]))
    cuda = [torch.from_numpy(img).to(cuda_device) for img in imgs[:6]]
    cuda_masks = [torch.from_numpy(m).to(cuda_device) for m in masks[:6]]
    got = pipe.forward_batch(cuda, cuda_masks, invert)
    assert all(g.is_cuda and np.array_equal(g.cpu().numpy(), w) for g, w in zip(got, want[:6]))
    assert all(np.array_equal(c.cpu().numpy(), b) for c, b in zip(cuda, before[:6]))
    pinned = [torch.from_numpy(img).pin_memory() for img in imgs[6:16]]
    first = pipe.forward_batch(pinned[:4], masks[6:10], invert, wait=False)
    second = pipe.forward_batch(pinned[4:], [torch.from_numpy(m) for m in masks[10:16]], invert, wait=False)
    pipe.wait()
    assert all(np.array_equal(g.numpy(), w) for g, w in zip(first + second, want[6:16]))
    assert pipe.last_boxes == boxes[6:16]
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch(imgs[:1], masks[:1], wait=False)
    with pytest.raises(ValueError, match="seeds"):
        pipe.forward_batch(imgs[:1], masks[:1], seeds=[1])
    with pytest.raises(ValueError, match="3 x 3"):
        pipe(np.zeros((2, 9, 3), np.uint8), np.zeros((5, 5), np.uint8))


class GivenOutput(torch.nn.Module):
    """Stands in for the generator: records the model input, returns a fixed y."""

    def __init__(self, y):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1, device=y.device))
        self.y, self.x = y, None

    def forward(self, x):
        self.x = x.clone()
        return self.y


BINARY = [c for c in MG.CASES if c[-1] != "gray"]         # read_mask keeps only 0 / 255


@pytest.mark.parametrize("case", BINARY, ids=[c[0] for c in BINARY])
def test_reference_vectors_through_crop_pipeline(migan, cuda_device, case):
    from migan_b200 import synthetic
    from migan_b200.pipeline import CropPipeline
    gold = MG.load_fixture()
    tag, res, pad = case[0], case[1], case[2]
    image, mask = MG.case_inputs(case)
    pipe = CropPipeline(synthetic.export_style_state_dict(res, seed=11), res, padding=pad, device=cuda_device)
    pipe.model = GivenOutput(torch.from_numpy(gold["y_" + tag]).to(cuda_device))
    out = pipe(image.numpy()[0].transpose(1, 2, 0), mask.numpy()[0, 0])
    assert pipe.last_box == tuple(int(v) for v in gold["box_" + tag])
    assert torch.equal(MG.on_stored_rows(gold, "x", tag, pipe.model.x.cpu()), torch.from_numpy(gold["x_" + tag]))
    assert np.array_equal(MG.on_stored_rows(gold, "final", tag, out.transpose(2, 0, 1)[None]), gold["final_" + tag])


def _oracle_blend(chw, plane, y, box):
    """The oracle's composed value before `.to(torch.uint8)` (pipeline_oracle.postprocess), [H,W,3] float32, inside the
    crop window; NaN outside it."""
    import torch.nn.functional as F
    from oracle import prepost_oracle as P
    x0, x1, y0, y1 = box
    H, W = chw.shape[2], chw.shape[3]
    m = PO.resize_nearest(plane, H, W)[:, :, y0:y1, x0:x1].to(torch.float32)
    out = PO.resize_bilinear_aa(((y * 0.5 + 0.5) * 255).clamp(0, 255), y1 - y0, x1 - x0)
    m = F.max_pool2d(m, 3, stride=1, padding=1)
    m = F.conv2d(F.pad(m, (2, 2, 2, 2), mode="reflect"), P.gaussian_kernel_5x5().view(1, 1, 5, 5)) / torch.tensor(255)
    composed = chw[:, :, y0:y1, x0:x1].to(torch.float32) * m + out * (1 - m)
    full = np.full((H, W, 3), np.nan, np.float32)
    full[y0:y1, x0:x1] = composed[0].numpy().transpose(1, 2, 0)
    return full


def test_comodgan_matches_hand_composition(lib, cuda_device):
    """The hand composition is the oracle's: its pre-processing of each crop gives x, the GPU's seeded Co-Mod-GAN forward
    runs on that x in the pipeline's generator chunks, and its post-processing and blend compose the result.

    The photos are the first six of this seeded set.  Its seventh (569 x 405, 3-channel mask) hits the known rounding
    difference of the anti-aliased crop resize: at x[0, 1, 200, 216] the kernel rounds the resized value to 140 where
    torch's CPU resize gives 139 (tests/test_crop_photos_emul.py pins it).  The one-level change of x changes the
    generator's output, so that photo cannot match the oracle's composition byte for byte; MIGAN_Pipeline has the same
    difference.

    The result is compared byte for byte, except at a pixel whose blend value in the oracle lies within 1e-4 of an
    integer (e.g. 163.999997): there the value before `.to(uint8)` sits on the truncation boundary, and the kernel's
    blend weight (smoothing summed in double, then rounded) or resized output may be one float ulp from torch's, which
    moves it by one level.  Such pixels are allowed one level.  They are common where the generator saturates: the clamped
    255s resize to 255 plus or minus an ulp, whichever way the taps' sum rounds."""
    from migan_b200 import comodgan
    from migan_b200.pipeline import CropPipeline, MIGAN_Pipeline
    g = comodgan.load(CO.make_state_dict(R, seed=1), R).to(cuda_device)
    reqs = _requests(np.random.default_rng(21), 7)[:6]
    GB = 4                                                # two generator chunks: 4 + 2
    seeds = np.array([(9 << 32) + k for k in range(len(reqs))], dtype=np.uint64)
    imgs, masks = [img for img, _ in reqs], [m for _, m in reqs]
    chws = [torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1)[None])) for img in imgs]
    planes = [torch.from_numpy(read_mask(m, False)[None, None]) for m in masks]
    xs, boxes = [], []
    for chw, plane in zip(chws, planes):
        taps = {}
        PO.forward(lambda x: torch.zeros(1, 3, R, R), chw.clone(), plane, R, 128, taps)
        xs.append(taps["x"])
        boxes.append(taps["box"])
    x = torch.cat(xs).to(cuda_device)
    y = torch.cat([g(x[c:c + GB], seeds=seeds[c:c + GB]) for c in range(0, len(reqs), GB)]).cpu()
    want = [PO.forward(lambda _x: y[i:i + 1], chws[i].clone(), planes[i], R, 128).numpy()[0].transpose(1, 2, 0)
            for i in range(len(reqs))]
    pipe = CropPipeline(g, R, device=cuda_device, noise_seed=9, generator_batch=GB)
    got = pipe.forward_batch(imgs, masks)
    assert pipe.last_boxes == boxes
    for i, (a, b) in enumerate(zip(got, want)):
        d = a != b
        if d.any():                         # only on a truncation boundary of the oracle's float blend (docstring)
            v = _oracle_blend(chws[i], planes[i], y[i:i + 1], boxes[i])[d]
            assert np.abs(v - np.round(v)).max() < 1e-4 and np.abs(a.astype(int) - b.astype(int)).max() == 1, (i, v)
    want = got                              # the pipeline's bytes, for the calls below
    got = pipe.forward_batch(imgs, masks, seeds=seeds)                      # explicit seeds leave the counter
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert pipe.noise.noise_index == len(reqs)
    ref = MIGAN_Pipeline(g, R, device=cuda_device, noise_seed=9, generator_batch=GB)
    with pytest.raises(RuntimeError, match="3 x 3"):                         # a refused call takes no seeds
        ref(torch.zeros(1, 3, 2, 9, dtype=torch.uint8), torch.zeros(1, 1, 2, 9, dtype=torch.uint8))
    assert ref.noise.noise_index == 0
    images = [chw.clone() for chw in chws]
    ref.forward_batch(images, planes)
    assert all(np.array_equal(im[0].numpy().transpose(1, 2, 0), w) for im, w in zip(images, want))
    assert ref.noise.noise_index == len(reqs)
    with pytest.raises(RuntimeError, match="resolution"):
        CropPipeline(g, 512, device=cuda_device)


# -- the command --------------------------------------------------------------------------------------------------------

# (path under the images directory, W, H, mask mode, mask size factor)
PHOTOS = [("p00.jpg", 256, 256, "L", 1.0), ("sub/p01.png", 397, 263, "LA", 0.5), ("sub/deep/p02.jpeg", 200, 150, "RGB", 2.0),
          ("p03.png", 640, 720, "RGBA", 1.0), ("a.b.jpg", 300, 500, "P", 0.7), ("dup.png", 320, 240, "RGB", 1.0),
          ("sub/dup.jpg", 330, 250, "L", 1.3), ("p05.png", 1024, 768, "LA", 1.0), ("sub/p06.jpg", 255, 257, "P", 1.0),
          ("p07.jpeg", 777, 131, "RGBA", 0.3), ("p08.png", 3, 3, "L", 1.0)]


def _mask_image(rng, h, w, mode):
    from PIL import Image
    v = np.full((h, w), 255, np.uint8)
    hh, ww = max(1, int(rng.integers(h // 10 + 1, h // 3 + 2))), max(1, int(rng.integers(w // 10 + 1, w // 3 + 2)))
    y0, x0 = int(rng.integers(0, max(1, h - hh))), int(rng.integers(0, max(1, w - ww)))
    v[y0:y0 + hh, x0:x0 + ww] = 0
    if mode == "L":
        return Image.fromarray(v)
    if mode == "P":
        im = Image.frombytes("P", (w, h), v.tobytes())
        im.putpalette([c for i in range(256) for c in (i, 255 - i, i // 2)])
        return im
    if mode == "LA":
        return Image.fromarray(np.dstack([rng.integers(0, 256, (h, w), dtype=np.uint8), v]), "LA")
    if mode == "RGB":
        return Image.fromarray(np.dstack([v, rng.integers(0, 256, (h, w, 2), dtype=np.uint8)]), "RGB")
    return Image.fromarray(np.dstack([rng.integers(0, 256, (h, w, 3), dtype=np.uint8), v]), "RGBA")


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("cropdata")
    images, masks = root / "images", root / "masks"
    masks.mkdir()
    rng = np.random.default_rng(17)
    for path, w, h, mode, f in PHOTOS:
        p = images / path
        p.parent.mkdir(parents=True, exist_ok=True)
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p, quality=90)
        _mask_image(rng, max(1, int(h * f)), max(1, int(w * f)), mode).save(
            masks / ("".join(os.path.basename(path).split(".")[:-1]) + ".png"))
    files = root / "files"
    files.mkdir()
    sd = MO.make_state_dict(R, seed=3)
    torch.save(sd, files / "migan.pth")
    return {"images": images, "masks": masks, "files": files, "migan": sd, "comodgan": CO.make_state_dict(R, seed=1)}


def _files(d):
    return {p.name: p.read_bytes() for p in sorted(d.iterdir())}


def _reference_loop(data, out, invert, cuda_device):
    """create_onnx_pipeline.py:323-344 with its torch pipeline call, one photo at a time."""
    from PIL import Image
    from migan_b200.pipeline import MIGAN_Pipeline
    from migan_b200 import demo_command as D
    pipe = MIGAN_Pipeline(data["migan"], R, device=cuda_device)
    out.mkdir(parents=True)
    for p in D.list_photos(data["images"]):
        img = np.array(Image.open(p).convert("RGB"))
        mask = np.array(Image.open(D.mask_path(data["masks"], p)))
        Image.fromarray(reference_call(pipe, img, mask, invert)).save(out / D.output_name(p))


@pytest.mark.parametrize("invert", [False, True], ids=["plain", "inverted"])
def test_command_files_equal_reference_loop(data, tmp_path, cuda_device, invert):
    from migan_b200 import crop_results as C
    _reference_loop(data, tmp_path / "ref", invert, cuda_device)
    want = _files(tmp_path / "ref")
    assert len(want) == len(PHOTOS) - 1
    C.crop_results(data["files"] / "migan.pth", R, data["images"], data["masks"], tmp_path / "out", invert_mask=invert,
                   device=cuda_device, batch_size=4, num_workers=3)
    assert _files(tmp_path / "out" / "sample_results") == want
    if not invert:                                     # as a command
        cmd = [sys.executable, "-m", "migan_b200.crop_results", "--resolution", str(R), "--model-path",
               str(data["files"] / "migan.pth"), "--images-dir", str(data["images"]), "--masks-dir", str(data["masks"]),
               "--output-dir", str(tmp_path / "cmd"), "--batch-size", "32"]
        subprocess.run(cmd, cwd=ROOT, check=True)
        assert _files(tmp_path / "cmd" / "sample_results") == want


def _virtual_ranks(data, out, world, cuda_device, **kw):
    from migan_b200 import crop_results as C
    from migan_b200 import demo_command as D
    first = None
    for rank in range(world):
        model = first.model if first else data["migan"]
        setup = C.CropSetup(model, R, data["images"], data["masks"], out, device=cuda_device, **kw)
        first = first or setup
        D.run_rank(setup, rank, world)
    return _files(out / "sample_results")


def test_command_files_do_not_depend_on_ranks_or_batch(data, tmp_path, cuda_device):
    base = _virtual_ranks(data, tmp_path / "w1", 1, cuda_device, batch_size=8)
    assert len(base) == len(PHOTOS) - 1
    for world in (2, 3):
        assert _virtual_ranks(data, tmp_path / ("w%d" % world), world, cuda_device, batch_size=8) == base
    assert _virtual_ranks(data, tmp_path / "b32", 1, cuda_device, batch_size=32) == base


def test_command_comodgan_256(data, tmp_path, cuda_device):
    from PIL import Image
    from migan_b200 import comodgan
    from migan_b200.pipeline import CropPipeline
    from migan_b200 import crop_results as C
    from migan_b200 import demo_command as D
    g = comodgan.load(data["comodgan"], R).to(cuda_device)
    C.crop_results(g, R, data["images"], data["masks"], tmp_path / "out", generator="comodgan", device=cuda_device,
                   batch_size=4, noise_seed=2)
    got = _files(tmp_path / "out" / "sample_results")
    items = D.plan_items(D.list_photos(data["images"]), data["masks"])
    pipe = CropPipeline(g, R, device=cuda_device)
    for a in range(0, len(items), 4):
        chunk = items[a:a + 4]
        imgs = [np.array(Image.open(it.photo).convert("RGB")) for it in chunk]
        masks = [np.array(Image.open(it.mask)) for it in chunk]
        seeds = [(2 << 32) + it.index for it in chunk]
        for it, out in zip(chunk, pipe.forward_batch(imgs, masks, seeds=seeds)):
            Image.fromarray(out).save(tmp_path / "want.png")
            assert got[it.output] == (tmp_path / "want.png").read_bytes(), it.output
    with pytest.raises(ValueError, match="comodgan"):
        C.crop_results(g, 384, data["images"], data["masks"], tmp_path / "bad", generator="comodgan", device=cuda_device)

"""`python -m migan_b200.demo` on the H100, on a data set written here with seeded MI-GAN-256 and Co-Mod-GAN-256 weights:
JPEG and PNG photos in nested directories, below and above R and of odd sizes, a name with an inner dot, two photos with
one output name, an upper-case suffix that is not listed, and masks in modes L, LA, RGB, RGBA and P (one larger than
512), each of its photo's size.

* the command's files are byte for byte a loop of one-request `DemoPipeline` calls saved with PIL, with and without
  `--invert-mask`, run as `python -m migan_b200.demo` and in process;
* against the whole reference algorithm on the CPU (oracle/demo_oracle.py around the oracle generator), known pixels
  are equal and hole pixels within 1;
* W = 2 and 3 virtual ranks (every rank's `run_rank` in one process) write the files of W = 1, for migan-256 and
  comodgan-256;
* Co-Mod-GAN's files are `DemoPipeline.forward_batch` on the same chunks with seeds noise_seed * 2**32 + k, k the index in
  the full sorted list;
* `--pipeline fullres` / `holewindow` files are each pipeline's result for the photo alone;
* `torchrun --nproc_per_node=2` writes the files of one process (skipped with fewer than two GPUs)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import comodgan_oracle as C  # noqa: E402
from oracle import demo_oracle as O  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

R = 256
BATCH = 3            # 10 planned photos: 4 chunks, the last one short; W = 3 ends on a ragged round
# The two photos named dup share one mask file, so they have one size: demo.py composes both with it.
# (path under the images directory, W, H, mask mode)
PHOTOS = [("p00.jpg", 256, 256, "L"), ("sub/p01.png", 397, 263, "LA"), ("sub/deep/p02.jpeg", 200, 150, "RGB"),
          ("p03.png", 640, 720, "RGBA"), ("a.b.jpg", 300, 500, "P"), ("dup.png", 320, 240, "RGB"),
          ("sub/dup.jpg", 320, 240, "L"), ("p05.png", 1024, 768, "LA"), ("sub/p06.jpg", 255, 257, "P"),
          ("p07.jpeg", 777, 131, "RGBA"), ("p08.png", 512, 384, "L")]


def _photo(rng, h, w):
    from PIL import Image
    low = rng.random((max(2, h // 24), max(2, w // 24), 3))
    img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BILINEAR), dtype=np.float64)
    return np.clip(0.85 * img + 0.15 * rng.integers(0, 256, (h, w, 3)), 0, 255).astype(np.uint8)


def _mask(rng, h, w, mode):
    """255 = known, 0 = hole (before any --invert-mask), in `mode` with the value in the channel read_mask reads."""
    from PIL import Image
    v = np.full((h, w), 255, np.uint8)
    for _ in range(2):
        hh, ww = int(rng.integers(h // 8, h // 3)), int(rng.integers(w // 8, w // 3))
        y0, x0 = int(rng.integers(0, h - hh)), int(rng.integers(0, w - ww))
        v[y0:y0 + hh, x0:x0 + ww] = 0
    v[rng.random((h, w)) < 0.01] = 128
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
    root = tmp_path_factory.mktemp("demodata")
    images, masks = root / "images", root / "masks"
    masks.mkdir()
    rng = np.random.default_rng(11)
    for path, w, h, mode in PHOTOS:
        p = images / path
        p.parent.mkdir(parents=True, exist_ok=True)
        Image.fromarray(_photo(rng, h, w)).save(p, quality=90)              # quality: JPEG only
        m = _mask(rng, h, w, mode)
        m.save(masks / ("".join(os.path.basename(path).split(".")[:-1]) + ".png"))
        O.demo_sizes(w, h, w, h, R)                                          # demo.py composes each pair
    Image.fromarray(_photo(rng, 64, 64)).save(images / "upper.JPG")           # not listed: no mask needed
    files = root / "files"
    files.mkdir()
    sd = MO.make_state_dict(R, seed=3)
    torch.save(sd, files / "migan.pth")
    return {"root": root, "images": images, "masks": masks, "files": files, "migan": sd,
            "comodgan": C.make_state_dict(R, seed=1)}


def _files(d):
    return {p.name: p.read_bytes() for p in sorted(d.iterdir())}


def run(data, out, model_name="migan-256", model=None, **kw):
    from migan_b200 import demo_command as D
    kw.setdefault("batch_size", BATCH)
    kw.setdefault("num_workers", 3)
    model = data[model_name.split("-")[0]] if model is None else model
    return D.demo(model_name, model, data["images"], data["masks"], out, **kw)


def _decoded(item):
    from PIL import Image
    img = np.array(Image.open(item.photo).convert("RGB"))
    return img, np.array(Image.open(item.mask))


def _plan(data):
    from migan_b200 import demo_command as D
    photos = D.list_photos(data["images"])
    assert len(photos) == len(PHOTOS)
    items = D.plan_items(photos, data["masks"])
    assert len(items) == len(PHOTOS) - 1 and [it.index for it in items] != list(range(len(items)))
    return items


def _command(data, out, *extra):
    return ["-m", "migan_b200.demo", "--model-name", "migan-256", "--model-path", str(data["files"] / "migan.pth"),
            "--images-dir", str(data["images"]), "--masks-dir", str(data["masks"]), "--output-dir", str(out),
            "--batch-size", str(BATCH), "--num-workers", "3"] + list(extra)


@pytest.mark.parametrize("invert", [False, True], ids=["plain", "inverted"])
def test_files_equal_one_request_loop(data, tmp_path, invert):
    from PIL import Image

    from migan_b200 import demo_command as D
    from migan_b200.demo import DemoPipeline
    loop = tmp_path / "loop"
    loop.mkdir()
    pipe = DemoPipeline(data["migan"], R)
    for p in D.list_photos(data["images"]):                   # demo.py's loop: every photo, later ones overwrite
        img = np.array(Image.open(p).convert("RGB"))
        mask = np.array(Image.open(D.mask_path(data["masks"], p)))
        Image.fromarray(pipe(img, mask, invert)).save(loop / D.output_name(p))
    out = tmp_path / "out"
    if invert:
        D.main(_command(data, out, "--invert-mask")[2:])
    else:
        env = dict(os.environ, PYTHONPATH=ROOT)
        p = subprocess.run([sys.executable] + _command(data, out), cwd=ROOT, env=env, capture_output=True, text=True,
                           timeout=900)
        assert p.returncode == 0, p.stderr
        assert "RuntimeWarning" not in p.stderr, p.stderr
    want, got = _files(loop), _files(out)
    assert len(got) == len(PHOTOS) - 1 and "a.b.png" in got and "dup.png" in got
    assert list(got) == list(want)
    for name in want:
        assert got[name] == want[name], name


def test_files_against_reference_algorithm(data, tmp_path):
    from PIL import Image
    out = tmp_path / "out"
    run(data, out)
    items = _plan(data)
    pre = [O.demo_pre(*_decoded(it), False, R) for it in items]
    x = torch.from_numpy(np.stack([p[2] for p in pre]))
    y = MO.generator_forward(data["migan"], x, R).numpy()
    worst = 0
    for it, (rs, m, _), yi in zip(items, pre, y):
        want = O.demo_post(yi, rs, m)
        got = np.array(Image.open(out / it.output))
        assert got.shape == want.shape, it.photo
        known = m == 255
        assert np.array_equal(got[known], want[known]), it.photo
        d = np.abs(got.astype(int) - want.astype(int)).max()
        worst = max(worst, int(d))
        assert d <= 1, (it.photo, d)
    print("largest hole-pixel difference from the CPU reference algorithm: %d" % worst)


def _virtual_ranks(data, setup_of, world, out):
    from migan_b200 import demo_command as D
    setup = setup_of(out)
    for rank in range(world):
        D.run_rank(setup, rank, world)
    return _files(out)


@pytest.mark.parametrize("model_name", ["migan-256", "comodgan-256"])
def test_virtual_ranks_write_the_files_of_one_rank(data, tmp_path, model_name):
    from migan_b200 import demo_command as D
    first = D.DemoSetup(model_name, data[model_name.split("-")[0]], data["images"], data["masks"], tmp_path / "w1",
                        batch_size=BATCH, noise_seed=5)
    assert len(first.chunks) == 4 and first.chunks[-1] == (9, 10)

    def setup_of(out, noise_seed=5):
        return D.DemoSetup(model_name, first.model, data["images"], data["masks"], out, batch_size=BATCH,
                           noise_seed=noise_seed)
    one = _virtual_ranks(data, lambda out: first, 1, tmp_path / "w1")
    assert len(one) == len(PHOTOS) - 1
    for world in (2, 3):
        got = _virtual_ranks(data, setup_of, world, tmp_path / ("w%d" % world))
        assert got == one, world
    if model_name.startswith("comodgan"):
        other = _virtual_ranks(data, lambda out: setup_of(out, noise_seed=6), 1, tmp_path / "seed6")
        assert all(other[k] != one[k] for k in one)                 # the seeds reach the generator


def test_comodgan_files_use_global_seeds(data, tmp_path):
    from PIL import Image

    from migan_b200 import comodgan
    from migan_b200.demo import DemoPipeline
    out = tmp_path / "out"
    run(data, out, "comodgan-256", noise_seed=7)
    items = _plan(data)
    pipe = DemoPipeline(comodgan.load(data["comodgan"], R), R)
    want = tmp_path / "want"
    want.mkdir()
    for a in range(0, len(items), BATCH):
        chunk = items[a:a + BATCH]
        decoded = [_decoded(it) for it in chunk]
        seeds = [(7 << 32) + it.index for it in chunk]
        outs = pipe.forward_batch([d[0] for d in decoded], [d[1] for d in decoded], seeds=seeds)
        for it, o in zip(chunk, outs):
            Image.fromarray(o).save(want / it.output)
    assert _files(out) == _files(want)


@pytest.mark.parametrize("pipeline", ["fullres", "holewindow"])
def test_other_pipelines_equal_each_photo_alone(data, tmp_path, pipeline):
    from PIL import Image

    from migan_b200 import FullResPipeline, HoleWindowPipeline
    out = tmp_path / "out"
    run(data, out, pipeline=pipeline, invert_mask=True)
    pipe = FullResPipeline(data["migan"], R) if pipeline == "fullres" else HoleWindowPipeline(data["migan"], R, margin=1)
    got = _files(out)
    assert len(got) == len(PHOTOS) - 1
    for it in _plan(data):
        img, mask = _decoded(it)
        want = pipe(img, mask, invert=True)
        assert want.shape == img.shape
        assert np.array_equal(np.array(Image.open(out / it.output)), want), it.photo


def test_torchrun_two_gpus_writes_the_same_files(data, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs for torchrun --nproc_per_node=2; %d visible" % torch.cuda.device_count())
    env = dict(os.environ, PYTHONPATH=ROOT)
    one = subprocess.run([sys.executable] + _command(data, tmp_path / "one"), cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900)
    two = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2"]
                         + _command(data, tmp_path / "two"), cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=900)
    assert one.returncode == 0, one.stderr
    assert two.returncode == 0, two.stderr
    assert _files(tmp_path / "two") == _files(tmp_path / "one")


def test_wait_for_the_oldest_call_only(data):
    """`wait(1)`, which the command's loop uses: the oldest queued call is finished and its record set, the later one
    stays queued until `wait()`."""
    from migan_b200.demo import DemoPipeline
    items = _plan(data)
    pipe = DemoPipeline(data["migan"], R)
    calls = []
    for chunk in (items[:2], items[2:5]):
        decoded = [_decoded(it) for it in chunk]
        photos = [torch.from_numpy(d[0]).pin_memory() for d in decoded]
        calls.append(pipe.forward_batch(photos, [d[1] for d in decoded], wait=False))
    pipe.wait(1)
    assert len(pipe._pending) == 1 and len(pipe.last_sizes) == 2
    first = [o.clone() for o in calls[0]]
    pipe.wait()
    assert not pipe._pending and len(pipe.last_sizes) == 3
    want = pipe.forward_batch([_decoded(it)[0] for it in items[:5]], [_decoded(it)[1] for it in items[:5]])
    assert all(np.array_equal(a.numpy(), b) for a, b in zip(first + calls[1], want))

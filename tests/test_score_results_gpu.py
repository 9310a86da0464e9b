"""`migan_b200.score_results` and `ResultsPipeline` on the H100, on directories written here: 37 photos of mixed sizes
(R x R among them, JPEGs and PNGs), one result per photo at R x R or at another size, a mask directory, and seeded
Inception and LPIPS weights.

* `ResultsPipeline.forward_batch` gives `real` and `composed` equal to a torch-CPU restatement of the script's lines (PIL
  BICUBIC of the photo and of the result, the mask's NEAREST and `// 255`, :244-249 in float32), over two passes, with
  directory masks and with generated masks;
* `score` gives the FID and LPIPS bits of a hand loop over the same sorted list and chunking;
* W = 2, 3 and 8 virtual ranks give the bits of W = 1, with ragged last rounds;
* the real photos scored as their own results give an LPIPS of exactly 0 and an FID near 0;
* `--save-real-stats` of `score` and of `evaluate_fid_lpips.evaluate` store the same members, byte for byte (the zip
  entries' write times aside);
* the files of `python -m migan_b200.demo` score through the command, which prints `score`'s values, in one process and
  under torchrun on 2 GPUs."""
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import fid_oracle as FO  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

R = 256
N = 37
BATCH = 8            # 5 chunks, the last one short: W = 2, 3 and 8 all end on a ragged round
DEMO_N = 10


def _photo(rng, h, w):
    from PIL import Image
    low = rng.random((max(2, h // 32), max(2, w // 32), 3))
    img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BILINEAR), dtype=np.float64)
    return np.clip(0.85 * img + 0.15 * rng.integers(0, 256, (h, w, 3)), 0, 255).astype(np.uint8)


def _mask(rng, h, w):
    from PIL import Image
    m = np.where(rng.random((max(1, h // 16), max(1, w // 16))) < 0.35, 0, 255).astype(np.uint8)
    return np.asarray(Image.fromarray(m).resize((w, h), Image.NEAREST))


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("scoredata")
    dirs = {k: root / k for k in ("real", "results", "masks", "ident", "files", "demo_real", "demo_masks")}
    for d in dirs.values():
        d.mkdir()
    rng = np.random.default_rng(11)
    sizes = [(R, R), (R + 44, R * 3 // 2), (200, 180), (R * 2, R * 3 // 2), (R // 2 + 3, R + 9)]
    result_sizes = [(R, R), (R, R), (300, 170), (R // 2, R // 2)]
    for i in range(N):
        h, w = sizes[i % len(sizes)]
        suffix = ".PNG" if i == 4 else (".jpg" if i % 3 == 0 else ".png")
        stem = "img_%03d" % ((i * 17) % N)                     # names not written in sorted order
        path = dirs["real"] / (stem + suffix)
        Image.fromarray(_photo(rng, h, w)).save(path, quality=90)
        with Image.open(path) as im:                           # the decoded photo, losslessly: its own result
            im.convert("RGB").save(dirs["ident"] / (stem + ".png"))
        rh, rw = result_sizes[i % len(result_sizes)]
        Image.fromarray(_photo(rng, rh, rw)).save(dirs["results"] / (stem + ".png"))
        mh, mw = (h, w) if i % 2 else (R, R)
        Image.fromarray(_mask(rng, mh, mw)).save(dirs["masks"] / (stem + ".png"))
    Image.fromarray(_photo(rng, R, R)).save(dirs["results"] / "unrelated.png")   # extra results are ignored
    (dirs["results"] / "notes.txt").write_text("not a result")
    for i in range(DEMO_N):                                    # the demo's set: masks of the photo's size
        h, w = sizes[i % len(sizes)]
        stem = "demo_%02d" % i
        Image.fromarray(_photo(rng, h, w)).save(dirs["demo_real"] / (stem + (".jpg" if i % 2 else ".png")), quality=90)
        Image.fromarray(_mask(rng, h, w)).save(dirs["demo_masks"] / (stem + ".png"))
    weights = {"model": MO.make_state_dict(R, seed=3), "inception": FO.seeded_state_dict(0),
               "lpips": LO.seeded_state_dict(0)}
    for k, v in weights.items():
        torch.save(v, dirs["files"] / ("%s.pth" % k))
    return {**dirs, **weights}


def score(data, results="results", mask_dir="masks", real="real", **kw):
    from migan_b200 import score_results as S
    return S.score(data[real], data[results], None if mask_dir is None else data[mask_dir], resolution=R,
                   batch_size=kw.pop("batch_size", BATCH), inception_weights=data["inception"],
                   lpips_weights=data["lpips"], **kw)


def _decoded(paths, mode):
    from PIL import Image
    out = []
    for p in paths:
        with Image.open(p) as im:
            out.append(np.array(im.convert(mode)))
    return out


def _files(data, with_masks):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import score_results as S
    paths = E.list_images(data["real"])
    assert len(paths) == N
    photos = _decoded(paths, "RGB")
    results = _decoded(S.list_results(paths, data["results"]), "RGB")
    masks = _decoded(E.list_masks(paths, data["masks"]), "L") if with_masks else None
    return photos, results, masks


def restated(photo, result, mask, from_dir):
    """InferenceDataset.__getitem__ on the photo, the same PIL BICUBIC stage on the result, and :244-249, float32."""
    from PIL import Image

    def square(a):
        im = Image.fromarray(a)
        if im.size != (R, R):
            im = im.resize((R, R), Image.BICUBIC)
        return (torch.Tensor(np.array(im)).float() * 2 / 255 - 1).permute(2, 0, 1)
    mk = Image.fromarray(mask)
    if from_dir:
        mk = mk.resize((R, R), Image.NEAREST)
    m = torch.Tensor(np.array(mk)[:, :, np.newaxis] // 255).float().permute(2, 0, 1)
    img, res = square(photo), square(result)
    composed = m * img + (1 - m) * res
    return (img * 0.5 + 0.5).clamp(0, 1), (composed * 0.5 + 0.5).clamp(0, 1)


@pytest.mark.parametrize("with_masks", [True, False], ids=["mask_dir", "generated"])
def test_results_pipeline_bit_for_bit(data, with_masks):
    import migan_b200
    photos, results, masks = _files(data, with_masks)
    pipe = migan_b200.ResultsPipeline(R, device="cuda", seed=0)
    real, composed = pipe.forward_batch(photos, results, masks)            # 37 images: two passes
    assert real.is_cuda and real.dtype == torch.float32 and tuple(real.shape) == (N, 3, R, R)
    assert composed.dtype == torch.float32 and tuple(composed.shape) == (N, 3, R, R)
    if masks is None:
        masks = list(migan_b200.RandomMaskStream(R, seed=0, device="cuda").next(N).cpu().numpy())
    want = [restated(p, r, m, with_masks) for p, r, m in zip(photos, results, masks)]
    assert torch.equal(real.cpu(), torch.stack([w[0] for w in want]))
    assert torch.equal(composed.cpu(), torch.stack([w[1] for w in want]))
    assert pipe.last_launches == [pipe.pass_launches(True, pipe.preprocess_launches(True))] * 2
    same = pipe.forward_batch(photos[:3], photos[:3], masks[:3])           # a photo as its own result
    assert torch.equal(same[0], same[1])


def test_results_pipeline_refusals(data):
    import migan_b200
    pipe = migan_b200.ResultsPipeline(R)
    img = np.zeros((8, 8, 3), np.uint8)
    for imgs, results, masks in (([img], [np.zeros((8, 8), np.uint8)], None),          # a result without channels
                                 ([img], [np.zeros((8, 8, 4), np.uint8)], None),       # RGBA, not converted
                                 ([img], [img.astype(np.uint16)], None),
                                 ([img, img], [img], None),
                                 ([img], [img], [img])):                                # a mask with channels
        with pytest.raises(ValueError):
            pipe.forward_batch(imgs, results, masks)
    with pytest.raises(RuntimeError, match="CUDA"):
        migan_b200.ResultsPipeline(R, device="cpu")
    real, composed = pipe.forward_batch([], [])
    assert real.shape == (0, 3, R, R) and composed.shape == (0, 3, R, R)


def hand_loop(data, with_masks):
    """ResultsPipeline + LPIPS + InceptionV3 + FeatureStatistics over the sorted list in chunks of BATCH."""
    from migan_b200 import ResultsPipeline, fid, lpips
    photos, results, masks = _files(data, with_masks)
    pipe = ResultsPipeline(R)
    inception = fid.InceptionV3(weights=data["inception"])
    compute_lpips = lpips.LPIPS(net="alex", weights=data["lpips"]).to("cuda")
    stats_real, stats_fake = fid.FeatureStatistics(device="cuda"), fid.FeatureStatistics(device="cuda")
    vals = []
    for b0 in range(0, N, BATCH):
        s = slice(b0, b0 + BATCH)
        imgs, composed_imgs = pipe.forward_batch(photos[s], results[s], None if masks is None else masks[s])
        stats_real.add(inception(imgs)[0])
        stats_fake.add(inception(composed_imgs)[0])
        vals.extend(compute_lpips(imgs, composed_imgs, normalize=True).detach().cpu().numpy().reshape(-1).tolist())
    return stats_real.frechet_distance(stats_fake), np.mean(vals), np.array(vals)


@pytest.mark.parametrize("with_masks", [True, False], ids=["mask_dir", "generated"])
def test_score_matches_hand_loop(data, with_masks):
    res = score(data, mask_dir="masks" if with_masks else None)
    fid_h, lp_h, vals_h = hand_loop(data, with_masks)
    print("%s: FID %r LPIPS %r, hand loop FID %r LPIPS %r" % (with_masks, res.fid, res.lpips, fid_h, lp_h))
    assert res.count == N and np.array_equal(res.lpips_values, vals_h)
    assert res.fid == fid_h and res.lpips == lp_h
    assert np.isfinite(res.fid) and res.fid > 0 and res.lpips > 0


@pytest.mark.parametrize("mask_dir", ["masks", None], ids=["mask_dir", "generated"])
def test_virtual_ranks_match_one_rank(data, mask_dir):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import score_results as S
    results = S.list_results(E.list_images(data["real"]), data["results"])
    setup = E.EvalSetup(None, None, data["real"], None if mask_dir is None else data[mask_dir], batch_size=BATCH,
                        inception_weights=data["inception"], lpips_weights=data["lpips"], results=results, res=R)
    assert len(setup.chunks) == 5 and setup.chunks[-1] == (32, 37)

    def virtual(world):
        merge = E.Merge(N, setup.device, setup.real_features)
        workers = [E.RankWorker(setup, k, world) for k in range(world)]
        try:
            for r in range(workers[0].rounds):
                for w in workers:
                    got = w.run_round(r)
                    if got is not None:
                        merge.add(got)
        finally:
            for w in workers:
                w.close()
        return merge.result()
    one = virtual(1)
    want = score(data, mask_dir=mask_dir)
    assert one.fid == want.fid and one.lpips == want.lpips and np.array_equal(one.lpips_values, want.lpips_values)
    for world in (2, 3, 8):
        got = virtual(world)
        print("%s W=%d: FID %r LPIPS %r (W=1: %r %r)" % (mask_dir, world, got.fid, got.lpips, one.fid, one.lpips))
        assert got.fid == one.fid and got.lpips == one.lpips and np.array_equal(got.lpips_values, one.lpips_values)


def test_photos_as_their_own_results(data, tmp_path):
    res = score(data, results="ident", save_real_stats_to=tmp_path / "stats.npz")
    with np.load(tmp_path / "stats.npz") as f:
        trace = float(np.trace(f["sigma"]))
    print("identity: FID %r (trace of sigma %r), LPIPS %r" % (res.fid, trace, res.lpips))
    assert res.lpips == 0.0 and not res.lpips_values.any()
    assert np.isfinite(res.fid) and abs(res.fid) <= 1e-3 * trace
    gen = score(data, results="ident", mask_dir=None)
    assert gen.lpips == 0.0 and np.isfinite(gen.fid) and abs(gen.fid) <= 1e-3 * trace


def test_real_statistics_shared_with_the_evaluation_command(data, tmp_path):
    from migan_b200 import evaluate_fid_lpips as E
    mine, theirs = tmp_path / "score.npz", tmp_path / "evaluate.npz"
    first = score(data, save_real_stats_to=mine)
    E.evaluate("migan-256", data["model"], data["real"], data["masks"], batch_size=BATCH, save_real_stats_to=theirs,
               inception_weights=data["inception"], lpips_weights=data["lpips"])
    with zipfile.ZipFile(mine) as a, zipfile.ZipFile(theirs) as b:
        assert a.namelist() == b.namelist() == ["mu.npy", "sigma.npy"]
        for name in a.namelist():
            assert a.read(name) == b.read(name), name
    again = score(data, real_stats=theirs)
    assert again.fid == first.fid and again.lpips == first.lpips


def _command(data, out_dir, *extra):
    return ["-m", "migan_b200.score_results", "--resolution", str(R), "--real-dir", str(data["demo_real"]),
            "--results-dir", str(out_dir), "--mask-dir", str(data["demo_masks"]), "--batch-size", "4",
            "--num-workers", "3", "--inception-weights", str(data["files"] / "inception.pth"),
            "--lpips-weights", str(data["files"] / "lpips.pth"), "--ids"] + list(extra)


def _lines(out):
    lines = [ln for ln in out.splitlines() if ln.startswith(("FID:", "LPIPS:", "P-IDS:", "U-IDS:"))]
    assert len(lines) == 4, out
    return lines


@pytest.fixture(scope="module")
def demo_out(data, tmp_path_factory):
    from migan_b200 import demo_command
    out = tmp_path_factory.mktemp("demo_out")
    demo_command.main(["--model-name", "migan-256", "--model-path", str(data["files"] / "model.pth"),
                       "--images-dir", str(data["demo_real"]), "--masks-dir", str(data["demo_masks"]),
                       "--output-dir", str(out), "--batch-size", "4"])
    assert len(list(out.iterdir())) == DEMO_N
    return out


def test_demo_outputs_score_through_the_command(data, demo_out):
    from migan_b200 import score_results as S
    res = S.score(data["demo_real"], demo_out, data["demo_masks"], resolution=R, batch_size=4, num_workers=3,
                  inception_weights=data["inception"], lpips_weights=data["lpips"], ids=True)
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable] + _command(data, demo_out), cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stderr
    print("demo round trip: FID %r LPIPS %r P-IDS %r U-IDS %r" % (res.fid, res.lpips, res.p_ids, res.u_ids))
    assert _lines(p.stdout) == ["FID: %r" % res.fid, "LPIPS:  %r" % res.lpips, "P-IDS: %r" % res.p_ids,
                                "U-IDS: %r" % res.u_ids]
    assert res.count == DEMO_N and np.isfinite(res.fid) and res.lpips > 0


def test_torchrun_two_gpus_prints_the_same_lines(data, demo_out):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs for torchrun --nproc_per_node=2; %d visible" % torch.cuda.device_count())
    env = dict(os.environ, PYTHONPATH=ROOT)
    one = subprocess.run([sys.executable] + _command(data, demo_out), cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900)
    two = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2"]
                         + _command(data, demo_out), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert one.returncode == 0, one.stderr
    assert two.returncode == 0, two.stderr
    assert _lines(two.stdout) == _lines(one.stdout)

"""`migan_b200.evaluate_fid_lpips` on the H100, on a photo directory written here (70 photos of mixed sizes, R x R
among them, JPEGs and PNGs, one upper-case suffix, plus a mask directory) with seeded MI-GAN-256, Inception and LPIPS
weights:

* `evaluate` gives the FID and LPIPS bits of INTEGRATION.md's hand-written loop over the same sorted list and chunking,
  with directory masks and with generated masks;
* W = 2, 3 and 8 virtual ranks (`RankWorker`s in one process on one device, merged by rank 0's `Merge` in chunk order)
  give the bits of W = 1, with ragged last rounds, for MI-GAN and for Co-Mod-GAN-256 with its seeds;
* stored real statistics give the same FID bits, and the stored mu / sigma are the hand loop's `mean_cov()`;
* the command prints the two result lines with `evaluate`'s values, in one process and under torchrun on 2 GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import comodgan_oracle as C  # noqa: E402
from oracle import fid_oracle as FO  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

R = 256
N = 70
BATCH = 8            # 9 chunks: the last one short; W = 2 and 8 end on a ragged round


def _photo(rng, h, w):
    low = rng.random((max(2, h // 32), max(2, w // 32), 3))
    from PIL import Image
    img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BILINEAR), dtype=np.float64)
    return np.clip(0.85 * img + 0.15 * rng.integers(0, 256, (h, w, 3)), 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("evaldata")
    real, masks = root / "real", root / "masks"
    real.mkdir()
    masks.mkdir()
    rng = np.random.default_rng(7)
    sizes = [(R, R), (R + 44, R * 3 // 2), (200, 180), (R * 2, R * 3 // 2), (R // 2 + 3, R + 9)]
    for i in range(N):
        h, w = sizes[i % len(sizes)]
        suffix = ".PNG" if i == 5 else (".jpg" if i % 3 == 0 else (".jpeg" if i % 7 == 1 else ".png"))
        stem = "img_%03d" % ((i * 37) % N)                    # names not written in sorted order
        Image.fromarray(_photo(rng, h, w)).save(real / (stem + suffix), quality=90)   # quality: JPEG only
        mh, mw = (h, w) if i % 2 else (R, R)
        m = np.where(rng.random((max(1, mh // 16), max(1, mw // 16))) < 0.35, 0, 255).astype(np.uint8)
        Image.fromarray(m).resize((mw, mh), Image.NEAREST).save(masks / (stem + ".png"))
    (real / "notes.txt").write_text("not an image")
    (real / "sub").mkdir()
    Image.fromarray(_photo(rng, R, R)).save(real / "sub" / "nested.png")
    files = root / "files"
    files.mkdir()
    weights = {"model": MO.make_state_dict(R, seed=3), "inception": FO.seeded_state_dict(0),
               "lpips": LO.seeded_state_dict(0)}
    for k, v in weights.items():
        torch.save(v, files / ("%s.pth" % k))
    return {"real": real, "masks": masks, "files": files, **weights}


def run(data, model_name="migan-256", model=None, mask_dir="masks", **kw):
    from migan_b200 import evaluate_fid_lpips as E
    return E.evaluate(model_name, data["model"] if model is None else model, data["real"],
                      None if mask_dir is None else data[mask_dir], batch_size=kw.pop("batch_size", BATCH),
                      inception_weights=data["inception"], lpips_weights=data["lpips"], **kw)


def hand_loop(data, with_masks):
    """INTEGRATION.md's loop ("FID on the GPU") over the sorted list in chunks of BATCH."""
    from PIL import Image

    from migan_b200 import EvalPipeline, fid, lpips
    from migan_b200 import evaluate_fid_lpips as E
    paths = E.list_images(data["real"])
    assert len(paths) == N
    pipe = EvalPipeline(data["model"], R)
    inception = fid.InceptionV3(weights=data["inception"])
    compute_lpips = lpips.LPIPS(net="alex", weights=data["lpips"]).to("cuda")
    stats_real, stats_fake = fid.FeatureStatistics(device="cuda"), fid.FeatureStatistics(device="cuda")
    lpips_vals = []
    for b0 in range(0, len(paths), BATCH):
        batch = paths[b0:b0 + BATCH]
        photos = [np.array(Image.open(p).convert("RGB")) for p in batch]
        masks = [np.array(Image.open(data["masks"] / ("%s.png" % p.stem)).convert("L")) for p in batch] \
            if with_masks else None
        imgs, composed_imgs = pipe.forward_batch(photos, masks)
        stats_real.add(inception(imgs)[0])
        stats_fake.add(inception(composed_imgs)[0])
        lpips_vals.extend(compute_lpips(imgs, composed_imgs, normalize=True).detach().cpu().numpy().tolist())
    # lpips_vals holds [[[v]]] per image, as in the script
    return stats_real.frechet_distance(stats_fake), np.mean(lpips_vals), np.array(lpips_vals).reshape(-1), \
        stats_real.mean_cov()


@pytest.fixture(scope="module")
def hand(data):
    return {True: hand_loop(data, True), False: hand_loop(data, False)}


@pytest.mark.parametrize("with_masks", [True, False], ids=["mask_dir", "generated"])
def test_evaluate_matches_hand_loop(data, hand, with_masks):
    res = run(data, mask_dir="masks" if with_masks else None)
    fid_h, lp_h, vals_h, _ = hand[with_masks]
    print("%s: FID %r LPIPS %r, hand loop FID %r LPIPS %r" % (with_masks, res.fid, res.lpips, fid_h, lp_h))
    assert res.count == N and res.lpips_values.dtype == np.float64
    assert np.array_equal(res.lpips_values, vals_h)
    assert res.fid == fid_h and res.lpips == lp_h
    assert np.isfinite(res.fid) and res.fid > 0 and res.lpips > 0


def virtual_ranks(setup, world):
    """W ranks run in one process: rank 0's merge takes each round's chunks in rank (= chunk) order."""
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features)
    workers = [E.RankWorker(setup, k, world) for k in range(world)]
    try:
        assert len({w.rounds for w in workers}) == 1
        for r in range(workers[0].rounds):
            for w in workers:
                got = w.run_round(r)
                if got is not None:
                    merge.add(got)
    finally:
        for w in workers:
            w.close()
    return merge.result()


@pytest.mark.parametrize("model_name,mask_dir", [("migan-256", "masks"), ("migan-256", None), ("comodgan-256", "masks")],
                         ids=["migan_mask_dir", "migan_generated", "comodgan"])
def test_virtual_ranks_match_one_rank(data, model_name, mask_dir):
    from migan_b200 import evaluate_fid_lpips as E
    model = data["model"] if model_name.startswith("migan") else C.make_state_dict(R, seed=1)
    setup = E.EvalSetup(model_name, model, data["real"], None if mask_dir is None else data[mask_dir], batch_size=BATCH,
                        noise_seed=5, inception_weights=data["inception"], lpips_weights=data["lpips"])
    assert len(setup.chunks) == 9 and setup.chunks[-1] == (64, 70)
    one = virtual_ranks(setup, 1)
    want = run(data, model_name, setup.model, mask_dir, noise_seed=5)       # the command's own single-process path
    assert one.fid == want.fid and one.lpips == want.lpips and np.array_equal(one.lpips_values, want.lpips_values)
    for world in (2, 3, 8):
        got = virtual_ranks(setup, world)
        print("%s %s W=%d: FID %r LPIPS %r (W=1: %r %r)" % (model_name, mask_dir, world, got.fid, got.lpips, one.fid,
                                                             one.lpips))
        assert got.fid == one.fid and got.lpips == one.lpips
        assert np.array_equal(got.lpips_values, one.lpips_values)
    if model_name.startswith("comodgan"):
        other = run(data, model_name, setup.model, mask_dir, noise_seed=6)
        assert other.fid != one.fid                           # the seeds reach the generator


def test_real_statistics_cache(data, hand, tmp_path):
    from migan_b200 import evaluate_fid_lpips as E
    path = tmp_path / "real_stats"                            # written as given, no suffix appended
    first = run(data, save_real_stats_to=path)
    with np.load(path) as f:
        mu, sigma = f["mu"], f["sigma"]
    mu_h, sigma_h = hand[True][3]
    assert mu.dtype == np.float64 and np.array_equal(mu, mu_h) and np.array_equal(sigma, sigma_h)
    again = run(data, real_stats=path)
    assert again.fid == first.fid and again.lpips == first.lpips
    with pytest.raises(ValueError):
        run(data, real_stats=path, save_real_stats_to=tmp_path / "x.npz")
    assert E.load_real_stats(path)[0].shape == (2048,)


def _command(data, *extra):
    return ["-m", "migan_b200.evaluate_fid_lpips", "--model-name", "migan-256",
            "--model-path", str(data["files"] / "model.pth"), "--real-dir", str(data["real"]),
            "--mask-dir", str(data["masks"]), "--batch-size", str(BATCH), "--num-workers", "3",
            "--inception-weights", str(data["files"] / "inception.pth"),
            "--lpips-weights", str(data["files"] / "lpips.pth")] + list(extra)


def _lines(out):
    lines = [ln for ln in out.splitlines() if ln.startswith(("FID:", "LPIPS:"))]
    assert len(lines) == 2, out
    return lines


def test_command_prints_the_two_lines(data):
    res = run(data, num_workers=3)
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable] + _command(data), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr
    assert _lines(p.stdout) == ["FID: %r" % res.fid, "LPIPS:  %r" % res.lpips]


def test_torchrun_two_gpus_prints_the_same_lines(data):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs for torchrun --nproc_per_node=2; %d visible" % torch.cuda.device_count())
    env = dict(os.environ, PYTHONPATH=ROOT)
    one = subprocess.run([sys.executable] + _command(data), cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=900)
    two = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2"]
                         + _command(data), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert one.returncode == 0, one.stderr
    assert two.returncode == 0, two.stderr
    assert _lines(two.stdout) == _lines(one.stdout)

"""Per-image scores, SSIM and PSNR of `evaluate_fid_lpips` and `score_results` on the H100, on directories written here:
37 photos of mixed sizes (R x R among them, JPEGs and PNGs), one result per photo, the photos' own decoded pixels as
results, a mask directory, and seeded MI-GAN-256, Co-Mod-GAN-256, Inception and LPIPS weights.

* every chunk's LPIPS, SSIM and PSNR values are the bits of `lpips.LPIPS`, `metrics.compute_ssim(real, composed, 11,
  size_average=False)` and `metrics.compute_psnr(composed, real, for_dataset=None)` called by hand on that chunk's
  `real` and `composed`, and its hole fraction is 1 - mean of the R x R mask, with directory and generated masks;
* W = 2, 3 and 8 virtual ranks give the CSV bytes, the printed lines and the means of W = 1;
* MI-GAN's per-image values are the same at --batch-size 8 and 32, and with stored real statistics;
* the photos scored as their own results give LPIPS 0, SSIM 1 and PSNR inf for every image;
* the commands print the lines in order and write the CSV of the library call; without the new flags they print only
  FID and LPIPS, with the values of a call without them;
* comodgan-256 runs with all three flags."""
import io
import math
import os
import subprocess
import sys
from contextlib import redirect_stdout

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
N = 37
BATCH = 8            # 5 chunks, the last one short: W = 2, 3 and 8 all end on a ragged round
ALL = dict(ssim=True, psnr=True, per_image=True)
PREFIXES = ("FID:", "LPIPS:", "SSIM:", "PSNR:", "P-IDS:", "U-IDS:")


def _photo(rng, h, w):
    from PIL import Image
    low = rng.random((max(2, h // 32), max(2, w // 32), 3))
    img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BILINEAR), dtype=np.float64)
    return np.clip(0.85 * img + 0.15 * rng.integers(0, 256, (h, w, 3)), 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("perimage")
    dirs = {k: root / k for k in ("real", "results", "masks", "ident", "files")}
    for d in dirs.values():
        d.mkdir()
    rng = np.random.default_rng(23)
    sizes = [(R, R), (R + 44, R * 3 // 2), (200, 180), (R * 2, R * 3 // 2), (R // 2 + 3, R + 9)]
    for i in range(N):
        h, w = sizes[i % len(sizes)]
        stem = "img,%03d" % ((i * 17) % N) if i == 3 else "img_%03d" % ((i * 17) % N)   # one name the CSV quotes
        path = dirs["real"] / (stem + (".jpg" if i % 3 == 0 else ".png"))
        Image.fromarray(_photo(rng, h, w)).save(path, quality=90)
        with Image.open(path) as im:
            im.convert("RGB").save(dirs["ident"] / (stem + ".png"))
        Image.fromarray(_photo(rng, R, R)).save(dirs["results"] / (stem + ".png"))
        mh, mw = (h, w) if i % 2 else (R, R)
        m = np.where(rng.random((max(1, mh // 16), max(1, mw // 16))) < 0.35, 0, 255).astype(np.uint8)
        Image.fromarray(m).resize((mw, mh), Image.NEAREST).save(dirs["masks"] / (stem + ".png"))
    weights = {"model": MO.make_state_dict(R, seed=3), "inception": FO.seeded_state_dict(0),
               "lpips": LO.seeded_state_dict(0)}
    for k, v in weights.items():
        torch.save(v, dirs["files"] / ("%s.pth" % k))
    return {**dirs, **weights}


def evaluate(data, mask_dir="masks", model_name="migan-256", model=None, **kw):
    from migan_b200 import evaluate_fid_lpips as E
    return E.evaluate(model_name, data["model"] if model is None else model, data["real"],
                      None if mask_dir is None else data[mask_dir], batch_size=kw.pop("batch_size", BATCH),
                      inception_weights=data["inception"], lpips_weights=data["lpips"], **kw)


def score(data, results="results", mask_dir="masks", **kw):
    from migan_b200 import score_results as S
    return S.score(data["real"], data[results], None if mask_dir is None else data[mask_dir], resolution=R,
                   batch_size=kw.pop("batch_size", BATCH), inception_weights=data["inception"],
                   lpips_weights=data["lpips"], **kw)


def setup_for(data, mask_dir, **kw):
    from migan_b200 import evaluate_fid_lpips as E
    return E.EvalSetup("migan-256", data["model"], data["real"], None if mask_dir is None else data[mask_dir],
                       batch_size=BATCH, inception_weights=data["inception"], lpips_weights=data["lpips"], **kw)


def csv_of(res, path):
    from migan_b200 import evaluate_fid_lpips as E
    E.write_per_image(path, res.per_image)
    return path.read_bytes()


def printed(res, **flags):
    from migan_b200 import evaluate_fid_lpips as E
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, flags.get("ids", False), flags.get("ssim", False), flags.get("psnr", False))
    return out.getvalue().splitlines()


def _mask_r(path):
    """The R x R mask the composite uses, float32 0 / 1: PIL NEAREST of the file, // 255."""
    from PIL import Image
    with Image.open(path) as im:
        return torch.from_numpy((np.array(im.convert("L").resize((R, R), Image.NEAREST)) // 255).astype(np.float32))


@pytest.mark.parametrize("with_masks", [True, False], ids=["mask_dir", "generated"])
def test_chunk_values_are_hand_calls_on_real_and_composed(data, with_masks):
    from PIL import Image

    import migan_b200
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import lpips, metrics
    setup = setup_for(data, "masks" if with_masks else None, **ALL)
    assert setup.extra_values == ("hole_fraction", "ssim", "psnr")
    assert setup.feature_width == 2 * 2048 + 1 + 3
    pipe = migan_b200.EvalPipeline(data["model"], R)
    net = lpips.LPIPS(net="alex", weights=data["lpips"]).to("cuda")
    generated = None if with_masks else migan_b200.RandomMaskStream(R, seed=0, device="cuda").next(N).cpu()
    with E.RankWorker(setup, 0, 1) as worker:
        for j, (a, b) in enumerate(setup.chunks):
            got = worker.run_chunk(j)
            photos = [np.array(Image.open(p).convert("RGB")) for p in setup.images[a:b]]
            masks = [np.array(Image.open(m).convert("L")) for m in setup.masks[a:b]] if with_masks else None
            real, composed, hole = pipe.forward_batch(photos, masks, hole_fraction=True)
            assert hole.dtype == torch.float32 and hole.is_cuda and tuple(hole.shape) == (b - a,)
            want_lpips = net(real, composed, normalize=True).view(-1)
            want_ssim = metrics.compute_ssim(real, composed, window_size=11, size_average=False)
            want_psnr = metrics.compute_psnr(composed, real, for_dataset=None)
            assert got.extra.dtype == torch.float32 and tuple(got.extra.shape) == (b - a, 3)
            assert torch.equal(got.lpips, want_lpips)
            assert torch.equal(got.extra[:, 0], hole)
            assert torch.equal(got.extra[:, 1], want_ssim)
            assert torch.equal(got.extra[:, 2], want_psnr)
            r_masks = [_mask_r(m) for m in setup.masks[a:b]] if with_masks else \
                [(generated[i] // 255).float() for i in range(a, b)]
            assert torch.equal(hole.cpu(), torch.stack([1 - m.mean() for m in r_masks]))
            assert 0 < float(hole.min()) and float(hole.max()) < 1
    res = evaluate(data, "masks" if with_masks else None, **ALL)
    vals = res.per_image
    assert list(vals) == ["name", "hole_fraction", "lpips", "ssim", "psnr"]
    assert vals["name"] == [p.name for p in setup.images] and "img,014.jpg" in vals["name"]
    assert res.ssim == float(np.mean(vals["ssim"])) and res.psnr == float(np.mean(vals["psnr"]))
    print("%s: SSIM %r PSNR %r, hole fraction %.3f..%.3f" % (with_masks, res.ssim, res.psnr, vals["hole_fraction"].min(),
                                                             vals["hole_fraction"].max()))


def virtual_ranks(setup, world):
    """W ranks in one process: rank 0's merge takes each round's chunks in rank (= chunk) order."""
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features, extra_values=setup.extra_values,
                    names=setup.names if setup.per_image else None)
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


@pytest.mark.parametrize("mask_dir", ["masks", None], ids=["mask_dir", "generated"])
def test_virtual_ranks_write_the_csv_of_one_rank(data, mask_dir, tmp_path):
    setup = setup_for(data, mask_dir, **ALL)
    one = virtual_ranks(setup, 1)
    want = evaluate(data, mask_dir, **ALL)                                 # the command's single-process path
    assert csv_of(one, tmp_path / "one.csv") == csv_of(want, tmp_path / "want.csv")
    assert printed(one, **ALL) == printed(want, **ALL)
    plain = evaluate(data, mask_dir)                                       # the new values change nothing else
    assert (want.fid, want.lpips) == (plain.fid, plain.lpips) and np.array_equal(want.lpips_values, plain.lpips_values)
    assert (plain.ssim, plain.psnr, plain.per_image) == (None, None, None)
    for world in (2, 3, 8):
        got = virtual_ranks(setup, world)
        print("%s W=%d: SSIM %r PSNR %r (W=1: %r %r)" % (mask_dir, world, got.ssim, got.psnr, one.ssim, one.psnr))
        assert csv_of(got, tmp_path / ("w%d.csv" % world)) == csv_of(one, tmp_path / "one.csv")
        assert printed(got, **ALL) == printed(one, **ALL)


def test_migan_values_do_not_depend_on_batch_size_or_stored_statistics(data, tmp_path):
    at8 = evaluate(data, **ALL, save_real_stats_to=tmp_path / "stats.npz")
    at32 = evaluate(data, batch_size=32, **ALL)
    stored = evaluate(data, real_stats=tmp_path / "stats.npz", **ALL)
    for k in ("hole_fraction", "lpips", "ssim", "psnr"):
        assert np.array_equal(at8.per_image[k], at32.per_image[k]), k
        assert np.array_equal(at8.per_image[k], stored.per_image[k]), k
    assert (at8.ssim, at8.psnr) == (at32.ssim, at32.psnr) == (stored.ssim, stored.psnr)
    assert stored.fid == at8.fid
    assert csv_of(at8, tmp_path / "8.csv") == csv_of(at32, tmp_path / "32.csv")


def test_photos_as_their_own_results(data):
    res = score(data, results="ident", **ALL)
    vals = res.per_image
    print("identity: SSIM %r PSNR %r LPIPS %r" % (res.ssim, res.psnr, res.lpips))
    assert not vals["lpips"].any() and res.lpips == 0.0
    assert (vals["ssim"] == 1.0).all() and res.ssim == 1.0
    assert np.isposinf(vals["psnr"]).all() and res.psnr == math.inf
    assert printed(res, **ALL)[2:] == ["SSIM: 1.0", "PSNR: inf"]
    gen = score(data, results="ident", mask_dir=None, psnr=True)
    assert gen.per_image is None and gen.ssim is None and gen.psnr == math.inf


def _run(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr
    return [ln for ln in p.stdout.splitlines() if ln.startswith(PREFIXES)]


def _common(data, *extra):
    return ["--real-dir", str(data["real"]), "--mask-dir", str(data["masks"]), "--batch-size", str(BATCH),
            "--inception-weights", str(data["files"] / "inception.pth"),
            "--lpips-weights", str(data["files"] / "lpips.pth")] + list(extra)


def test_commands_print_the_lines_and_write_the_csv(data, tmp_path):
    evaluate_args = ["migan_b200.evaluate_fid_lpips", "--model-name", "migan-256",
                     "--model-path", str(data["files"] / "model.pth")]
    plain = evaluate(data)
    assert _run(evaluate_args + _common(data)) == ["FID: %r" % plain.fid, "LPIPS:  %r" % plain.lpips]

    res = evaluate(data, **ALL)
    lines = _run(evaluate_args + _common(data, "--ssim", "--psnr", "--per-image", str(tmp_path / "eval.csv")))
    assert lines == printed(res, **ALL) and [ln.split(":")[0] for ln in lines] == ["FID", "LPIPS", "SSIM", "PSNR"]
    assert (tmp_path / "eval.csv").read_bytes() == csv_of(res, tmp_path / "eval_lib.csv")

    res = score(data, ids=True, **ALL)
    lines = _run(["migan_b200.score_results", "--resolution", str(R), "--results-dir", str(data["results"])]
                 + _common(data, "--ids", "--psnr", "--ssim", "--per-image", str(tmp_path / "score.csv")))
    assert lines == printed(res, ids=True, **ALL)
    assert [ln.split(":")[0] for ln in lines] == ["FID", "LPIPS", "SSIM", "PSNR", "P-IDS", "U-IDS"]
    assert (tmp_path / "score.csv").read_bytes() == csv_of(res, tmp_path / "score_lib.csv")
    assert not list(tmp_path.glob(".*.tmp"))


def test_comodgan_with_every_new_flag(data):
    model = C.make_state_dict(R, seed=1)
    res = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5, **ALL)
    plain = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5)
    vals = res.per_image
    print("comodgan-256: FID %r LPIPS %r SSIM %r PSNR %r" % (res.fid, res.lpips, res.ssim, res.psnr))
    assert (res.fid, res.lpips) == (plain.fid, plain.lpips) and len(vals["name"]) == N
    assert ((vals["hole_fraction"] > 0) & (vals["hole_fraction"] < 1)).all()
    assert ((vals["ssim"] > -1) & (vals["ssim"] < 1)).all() and np.isfinite(vals["psnr"]).all()
    assert res.ssim == float(np.mean(vals["ssim"])) and res.psnr == float(np.mean(vals["psnr"]))

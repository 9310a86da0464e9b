"""Scores by hole size on the H100: `RandomMaskStream(s, seed, hole_range)`, `fid.BinnedFeatureStatistics` and the
`--hole-bins` / `--hole-range` flags of `evaluate_fid_lpips` and `score_results`.

* the stream equals tests/golden/masks_hole_range.npz (the reference's RandomMask(s, hole_range)) at 32, 256 and 512 for
  every stored range: bytes or digests, hole counts and final state, however `next(n)` is split;
* the binned statistics are bit for bit one `FeatureStatistics` per bin (rows of bin -1 and bins that are empty in
  early calls included), at d = 2048;
* the commands on 37 photos at R = 256 (seeded MI-GAN-256, Co-Mod-GAN-256, Inception and LPIPS weights):
  `--hole-bins 0,1` repeats the overall FID, LPIPS, SSIM, PSNR, P-IDS and U-IDS bit for bit; with 5 bins every bin
  equals hand computations from the per-image values and the kept features; W = 2, 3 and 8 virtual ranks give the
  lines of W = 1; without the new flags the lines are the plain call's; with `--hole-range` every mask's hole fraction
  lies inside the range and the masks are the stream's; `score_results` and comodgan-256 run once each."""
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
from oracle import masks_oracle as M  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "masks_hole_range.npz"))
RANGES = [tuple(r) for r in GOLDEN["ranges"]]
R = 256
N = 37
BATCH = 8
EDGES5 = (0.0, 0.2, 0.35, 0.5, 0.7, 1.0)


def _golden_state(key):
    rest = GOLDEN[key + "_rest"]
    return GOLDEN[key + "_state"], int(rest[0]), int(rest[1]), float(rest[2])


def _assert_state(stream, key):
    name, k, pos, has_gauss, gauss = stream.get_state()
    want = _golden_state(key)
    assert name == "MT19937" and np.array_equal(k, want[0]) and (pos, has_gauss, gauss) == want[1:]


def _check_masks(masks, key, s):
    n = masks.shape[0]
    assert np.array_equal((masks == 0).reshape(n, -1).sum(1), GOLDEN[key + "_holes"])
    if s == 32:
        bits = np.unpackbits(GOLDEN[key], axis=1, count=s * s).reshape(-1, s, s)
        assert np.array_equal(masks, np.where(bits == 1, 255, 0).astype(np.uint8))
    else:
        got = np.frombuffer(b"".join(M.digest(m) for m in masks), np.uint8).reshape(n, 8)
        assert np.array_equal(got, GOLDEN[key + "_digest"])


@pytest.mark.parametrize("s", [32, 256, 512])
@pytest.mark.parametrize("i", range(5))
def test_stream_equals_fixture_however_split(lib, i, s):
    from migan_b200 import RandomMaskStream
    key = "r%d_%d" % (i, s)
    n = GOLDEN[key + "_holes"].shape[0]
    for split in ([n], [1, 3, n - 4], [1] * n):
        stream = RandomMaskStream(s, 0, "cuda", hole_range=RANGES[i])
        masks = np.concatenate([stream.next(k).cpu().numpy() for k in split])
        torch.cuda.synchronize()
        _check_masks(masks, key, s)
        assert stream.attempts == int(GOLDEN[key + "_attempts"])
        _assert_state(stream, key)


def test_binned_statistics_equal_one_statistics_per_bin(lib):
    from migan_b200 import fid
    g = torch.Generator(device="cuda").manual_seed(5)
    nbins, dim = 5, fid.FEATURES
    binned = fid.BinnedFeatureStatistics(nbins, dim)
    single = [fid.FeatureStatistics(dim) for _ in range(nbins)]
    calls = [[0, 0, -1, 1], [2] * 32, list(range(-1, 5)) * 5 + [4, 4], [4], [-1, 3, 0, 3]]
    for bins in calls:
        n = len(bins)
        x = torch.randn((n, dim), generator=g, device="cuda") * 3 + 100
        b = torch.tensor(bins, dtype=torch.int32, device="cuda")
        binned.add(x, b)
        for k in range(nbins):
            if (b == k).any():
                single[k].add(x[b == k])
    assert binned.counts().tolist() == [s.count for s in single]
    for k in range(nbins):
        assert torch.equal(binned.shift[k], single[k].shift), k
        assert torch.equal(binned.sum[k], single[k].sum), k
        assert torch.equal(binned.sumsq[k], single[k].sumsq), k
        mu, sigma = binned.mean_cov_device(k)
        mu1, sigma1 = single[k].mean_cov_device()
        assert torch.equal(mu, mu1) and torch.equal(sigma, sigma1)


# -- the commands -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("holebins")
    dirs = {k: root / k for k in ("real", "results", "masks", "files")}
    for d in dirs.values():
        d.mkdir()
    rng = np.random.default_rng(31)
    for i in range(N):
        stem = "img_%03d" % ((i * 17) % N)
        h, w = (R, R) if i % 2 else (R + 40, R * 3 // 2)
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(dirs["real"] / (stem + ".png"))
        Image.fromarray(rng.integers(0, 256, (R, R, 3), dtype=np.uint8)).save(dirs["results"] / (stem + ".png"))
        m = np.where(rng.random((R // 16, R // 16)) < 0.1 + 0.8 * i / N, 0, 255).astype(np.uint8)
        Image.fromarray(m).resize((R, R), Image.NEAREST).save(dirs["masks"] / (stem + ".png"))
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


def printed(res, ids=True, ssim=True, psnr=True):
    from migan_b200 import evaluate_fid_lpips as E
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, ids, ssim, psnr)
    return out.getvalue().splitlines()


ALL = dict(ssim=True, psnr=True, per_image=True, ids=True)


def test_one_bin_repeats_the_overall_scores(data):
    res = evaluate(data, hole_bins=(0, 1), **ALL)
    (b,) = res.by_hole
    print("one bin:", b)
    assert (b.lo, b.hi, b.count) == (0.0, 1.0, N)
    assert (b.fid, b.lpips, b.ssim, b.psnr, b.p_ids, b.u_ids) == (res.fid, res.lpips, res.ssim, res.psnr, res.p_ids,
                                                                 res.u_ids)
    plain = evaluate(data, **ALL)
    assert plain.by_hole is None and printed(plain) == printed(res)[:-1]
    assert (plain.fid, plain.lpips, plain.p_ids) == (res.fid, res.lpips, res.p_ids)


def _virtual_ranks(setup, world, ids):
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features, keep_features=ids,
                    extra_values=setup.extra_values, names=setup.names if setup.per_image else None,
                    hole_bins=setup.hole_bins)
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


def test_five_bins_are_hand_computations_and_do_not_depend_on_ranks(data):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import fid, ids
    setup = E.EvalSetup("migan-256", data["model"], data["real"], data["masks"], batch_size=BATCH,
                        inception_weights=data["inception"], lpips_weights=data["lpips"], ssim=True, psnr=True,
                        per_image=True, hole_bins=EDGES5)
    merge = E.Merge(N, "cuda", True, keep_features=True, extra_values=setup.extra_values, names=setup.names,
                    hole_bins=EDGES5)
    with E.RankWorker(setup, 0, 1) as worker:
        chunks = [worker.run_chunk(j) for j in range(len(setup.chunks))]
    for c in chunks:
        merge.add(c)
    res = merge.result()
    h = res.per_image["hole_fraction"]
    bins = np.searchsorted(np.array(EDGES5[1:-1]), h, side="right")
    assert sorted(set(bins.tolist())) == list(range(5)), bins          # the masks put images in every bin
    real = fid.FeatureStatistics()
    for c in chunks:
        real.add(c.real)
    mu_r, sigma_r = real.mean_cov_device()
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert (b.lo, b.hi, b.count) == (EDGES5[k], EDGES5[k + 1], len(idx))
        for name in ("lpips", "ssim", "psnr"):
            assert getattr(b, name) == float(np.mean(res.per_image[name][idx])), (k, name)
        fake = fid.FeatureStatistics()
        for c in chunks:
            sel = torch.from_numpy(bins[c.start:c.start + c.fake.shape[0]] == k).cuda()
            if bool(sel.any()):
                fake.add(c.fake[sel])
        if len(idx) >= 2:
            assert b.fid == fid.frechet_distance(mu_r, sigma_r, *fake.mean_cov_device())
            at = torch.from_numpy(idx).cuda()
            s = ids.inception_discriminative_scores(merge.kept[0][at], merge.kept[1][at])
            assert (b.p_ids, b.u_ids) == (s.p_ids, s.u_ids)
        else:
            assert math.isnan(b.fid) and math.isnan(b.p_ids)
    lines = printed(res)
    print("\n".join(lines))
    for world in (2, 3, 8):
        assert printed(_virtual_ranks(setup, world, True)) == lines, world


def test_hole_range_masks_lie_in_the_range(data):
    from migan_b200 import RandomMaskStream
    lo, hi = 0.5, 0.6
    res = evaluate(data, mask_dir=None, per_image=True, hole_range=(lo, hi), hole_bins=(0, 0.55, 1))
    h = res.per_image["hole_fraction"]
    want = RandomMaskStream(R, 0, "cuda", hole_range=(lo, hi)).next(N)
    assert np.array_equal(h, (1 - (want // 255).float().mean((1, 2))).cpu().numpy().astype(np.float64))
    assert ((h > lo) & (h < hi)).all(), h
    assert sum(b.count for b in res.by_hole) == N
    print("hole range:", h.min(), h.max(), [b.count for b in res.by_hole])


PREFIXES = ("FID:", "LPIPS:", "SSIM:", "PSNR:", "P-IDS:", "U-IDS:", "HOLE ")


def _run(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr
    return [ln for ln in p.stdout.splitlines() if ln.startswith(PREFIXES)]


def test_commands_and_comodgan(data):
    from migan_b200 import score_results as S
    common = ["--real-dir", str(data["real"]), "--batch-size", str(BATCH),
              "--inception-weights", str(data["files"] / "inception.pth"),
              "--lpips-weights", str(data["files"] / "lpips.pth")]
    res = evaluate(data, mask_dir=None, hole_bins=EDGES5, hole_range=(0.2, 0.4), ids=True, psnr=True)
    lines = _run(["migan_b200.evaluate_fid_lpips", "--model-name", "migan-256", "--model-path",
                  str(data["files"] / "model.pth"), "--hole-bins", ",".join(map(str, EDGES5)), "--hole-range", "0.2",
                  "0.4", "--ids", "--psnr"] + common)
    assert lines == printed(res, True, False, True) and len(lines) == 5 + 5
    assert lines[-1].startswith("HOLE [0.7, 1.0]: images ")
    res = S.score(data["real"], data["results"], data["masks"], resolution=R, batch_size=BATCH,
                  inception_weights=data["inception"], lpips_weights=data["lpips"], hole_bins=(0, 0.5, 1), ssim=True)
    lines = _run(["migan_b200.score_results", "--resolution", str(R), "--results-dir", str(data["results"]),
                  "--mask-dir", str(data["masks"]), "--hole-bins", "0,0.5,1", "--ssim"] + common)
    assert lines == printed(res, False, True, False) and len(lines) == 3 + 2
    print("\n".join(lines))
    model = C.make_state_dict(R, seed=1)
    res = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5, hole_bins=EDGES5)
    plain = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5)
    assert (res.fid, res.lpips) == (plain.fid, plain.lpips) and sum(b.count for b in res.by_hole) == N
    print("\n".join(printed(res, False, False, False)))


def test_generate_masks_with_a_hole_range(lib, tmp_path):
    from PIL import Image

    from migan_b200 import RandomMaskStream, generate_masks
    images = tmp_path / "images"
    images.mkdir()
    for k in range(6):
        Image.new("RGB", (8, 8)).save(images / ("p%d.png" % k))
    generate_masks.main(["--images-dir", str(images), "--output-dir", str(tmp_path / "out"), "--resolution", "64",
                         "--hole-range", "0.5", "0.6"])
    want = RandomMaskStream(64, 0, "cuda", hole_range=(0.5, 0.6)).next(6).cpu().numpy()
    for k in range(6):
        got = np.array(Image.open(tmp_path / "out" / ("p%d.png" % k)))
        assert np.array_equal(got, want[k])
        assert 0.5 < 1 - (got == 255).mean() < 0.6

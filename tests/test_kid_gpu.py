"""KID on the H100: `kid.kernel_inception_distance` and `--kid` in `evaluate_fid_lpips` and `score_results`.

* the library's per-subset terms and KID equal the float64 oracle within 1e-12 of each subset's cancellation scale, at
  10,000 x 2048 with the default 100 subsets of 1,000 and in ragged cases (m of 2, 63, 64, 65 and 130, m = n,
  n_r != n_f, d of 37 and 2048);
* two calls give the same bytes, on the default stream and on a side stream; float32 input gives the bytes of the same
  values in float64;
* `evaluate(kid=True)` on 37 photos at R = 256 (seeded MI-GAN-256, Inception and LPIPS weights), with directory and
  with generated masks: its KID is `kernel_inception_distance` of the merged features bit for bit, and W = 2, 3 and 8
  virtual ranks print the lines of W = 1; `--hole-bins 0,1 --kid` repeats the overall KID, and five bins equal hand
  calls on each bin's rows; `score_results --kid` and comodgan-256 run."""
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
from oracle import kid_oracle as O  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

BOUND = 1e-12       # as in test_kid_emul.py, in units of each subset's cancellation scale
R = 256
N = 37
BATCH = 8
EDGES5 = (0.0, 0.2, 0.35, 0.5, 0.7, 1.0)


def scale(T, m):
    return ((np.abs(T[:, 0]) + np.abs(T[:, 1])) / (m - 1) + 2 * np.abs(T[:, 2]) / m) / m


def terms_on_device(real, fake, S, max_subset_size=1000, seed=0, stream=None):
    from migan_b200 import kid
    m = O.subset_size(len(real), len(fake), max_subset_size)
    fi, ri = kid.draw_subsets(len(real), len(fake), S, m, seed)
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
        T = kid.subset_terms(real, fake, ri, fi)
        out = T.cpu().numpy()
    return out, m


def check_against_oracle(real, fake, S, max_subset_size):
    from migan_b200 import kid
    res = kid.kernel_inception_distance(real, fake, S, max_subset_size)
    T, m = terms_on_device(torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda(), S, max_subset_size)
    want = O.kid(real, fake, S, max_subset_size)
    c = scale(want.terms, m)
    diff = ((np.abs(T[:, 0] - want.terms[:, 0]) + np.abs(T[:, 1] - want.terms[:, 1])) / (m - 1)
            + 2 * np.abs(T[:, 2] - want.terms[:, 2]) / m) / m
    ratio = max(float((diff / c).max()), abs(res.kid - want.kid) / float(c.mean()))
    print("n_r %d n_f %d d %d m %d: KID %r (oracle %r) std %r, max error / scale %.3g"
          % (len(real), len(fake), real.shape[1], m, res.kid, want.kid, res.std, ratio))
    assert (res.subsets, res.subset_size) == (S, m)
    assert ratio <= BOUND
    assert abs(res.std - want.std) <= BOUND * float(c.max())
    return res


def test_library_matches_the_oracle_at_10000_by_2048(lib):
    real, fake = O.features(10000, 2048, 1), O.features(10000, 2048, 2, 0.05)
    check_against_oracle(real, fake, 100, 1000)


@pytest.mark.parametrize("n_r,n_f,d,max_subset,dtype", [
    (2, 5, 37, 1000, np.float32), (63, 63, 37, 1000, np.float64), (100, 80, 37, 64, np.float32),
    (65, 90, 2048, 1000, np.float64), (150, 130, 37, 1000, np.float32), (140, 200, 2048, 130, np.float32),
    (3000, 1700, 2048, 1000, np.float32)])
def test_library_matches_the_oracle_in_ragged_cases(lib, n_r, n_f, d, max_subset, dtype):
    real, fake = O.features(n_r, d, 11).astype(dtype), O.features(n_f, d, 12, 0.1).astype(dtype)
    check_against_oracle(real, fake, 5, max_subset)


def test_same_bytes_on_every_call_and_stream(lib):
    real = torch.from_numpy(O.features(3000, 2048, 5)).cuda()
    fake = torch.from_numpy(O.features(2500, 2048, 6, 0.1)).cuda()
    a, _ = terms_on_device(real, fake, 20)
    b, _ = terms_on_device(real, fake, 20)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    c, _ = terms_on_device(real, fake, 20, stream=side)
    assert a.tobytes() == b.tobytes() == c.tobytes()
    d, _ = terms_on_device(real.double(), fake.double(), 20)
    assert a.tobytes() == d.tobytes()
    from migan_b200 import kid
    assert kid.kernel_inception_distance(real, fake, 20) == kid.kernel_inception_distance(real.double(),
                                                                                          fake.cpu().numpy(), 20)


# -- the commands -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("kid")
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


def printed(res, ids=False, ssim=False, psnr=False, kid=True):
    from migan_b200 import evaluate_fid_lpips as E
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, ids, ssim, psnr, kid)
    return out.getvalue().splitlines()


def virtual_ranks(setup, world, ids=False):
    """Rank 0's merge of `world` virtual ranks run in turn on one GPU: (merge, result)."""
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features, keep_features=ids,
                    extra_values=setup.extra_values, hole_bins=setup.hole_bins, kid=True)
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
    return merge, merge.result()


@pytest.mark.parametrize("mask_dir", ["masks", None], ids=["directory masks", "generated masks"])
def test_evaluate_kid_is_the_kid_of_the_merged_features(data, mask_dir):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import kid
    res = evaluate(data, mask_dir=mask_dir, kid=True, ids=True)
    setup = E.EvalSetup("migan-256", data["model"], data["real"], None if mask_dir is None else data[mask_dir],
                        batch_size=BATCH, inception_weights=data["inception"], lpips_weights=data["lpips"])
    merge, one = virtual_ranks(setup, 1, ids=True)
    assert res.kid == kid.kernel_inception_distance(*merge.kept).kid == one.kid
    assert (res.fid, res.p_ids) == (one.fid, one.p_ids) and len(res) == 8
    plain = evaluate(data, mask_dir=mask_dir, ids=True)
    assert plain.kid is None and (plain.fid, plain.lpips, plain.p_ids) == (res.fid, res.lpips, res.p_ids)
    lines = printed(res, ids=True)
    print("\n".join(lines))
    assert lines[-1] == "KID: %r" % res.kid and lines[:-1] == printed(plain, ids=True, kid=False)
    for world in (2, 3, 8):
        assert printed(virtual_ranks(setup, world, ids=True)[1], ids=True) == lines, world


def test_hole_bins_kid(data):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import kid
    res = evaluate(data, hole_bins=(0, 1), kid=True)
    assert res.by_hole[0].kid == res.kid and res.by_hole[0].count == N
    setup = E.EvalSetup("migan-256", data["model"], data["real"], data["masks"], batch_size=BATCH,
                        inception_weights=data["inception"], lpips_weights=data["lpips"], hole_bins=EDGES5)
    merge, res = virtual_ranks(setup, 1)
    h = merge.extra[:, 0].cpu().numpy().astype(np.float64)
    bins = np.searchsorted(np.array(EDGES5[1:-1]), h, side="right")
    assert sorted(set(bins.tolist())) == list(range(5)), bins
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert b.count == len(idx)
        if len(idx) >= 2:
            at = torch.from_numpy(idx).cuda()
            assert b.kid == kid.kernel_inception_distance(merge.kept[0], merge.kept[1][at]).kid, k
        else:
            assert math.isnan(b.kid)
    lines = printed(res)
    print("\n".join(lines))
    assert all(ln.split(" KID ")[1] == repr(b.kid) for ln, b in zip(lines[-5:], res.by_hole))
    for world in (2, 3):
        assert printed(virtual_ranks(setup, world)[1]) == lines, world


PREFIXES = ("FID:", "LPIPS:", "SSIM:", "PSNR:", "P-IDS:", "U-IDS:", "KID:", "HOLE ")


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
    res = S.score(data["real"], data["results"], data["masks"], resolution=R, batch_size=BATCH,
                  inception_weights=data["inception"], lpips_weights=data["lpips"], hole_bins=(0, 0.5, 1), kid=True,
                  ids=True)
    lines = _run(["migan_b200.score_results", "--resolution", str(R), "--results-dir", str(data["results"]),
                  "--mask-dir", str(data["masks"]), "--hole-bins", "0,0.5,1", "--kid", "--ids"] + common)
    assert lines == printed(res, ids=True) and len(lines) == 5 + 2 and lines[4].startswith("KID: ")
    print("\n".join(lines))
    lines = _run(["migan_b200.evaluate_fid_lpips", "--model-name", "migan-256", "--model-path",
                  str(data["files"] / "model.pth"), "--kid"] + common)
    assert lines == printed(evaluate(data, mask_dir=None, kid=True))
    model = C.make_state_dict(R, seed=1)
    res = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5, kid=True)
    plain = evaluate(data, model_name="comodgan-256", model=model, noise_seed=5)
    assert (res.fid, res.lpips) == (plain.fid, plain.lpips) and math.isfinite(res.kid)
    print("\n".join(printed(res)))

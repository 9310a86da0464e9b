"""Precision, recall, density and coverage on the H100: `prdc.precision_recall_density_coverage` and `--prdc` in
`evaluate_fid_lpips` and `score_results`.

* the library's counts equal the float64 oracle's (squared differences summed directly) in ragged cases (N != M, sizes
  not multiples of 64, d of 37, 100 and 2048, k of 1, 3 and 5, float32 and float64), with the smallest decision margin
  far above the rounding bound, and at 10,000 x 2048 per side, where the oracle's distances run on the GPU in float64;
* small integer-valued features with duplicated rows within and across the sets, where every distance is exact and
  ties are everywhere: the same counts as the oracle, which pins `<=` and the self-inclusive (k + 1)-th value;
* two calls give the same bytes, on the default stream and on a side stream; float32 input gives the counts of the same
  values in float64; permuting the rows leaves every count as it is; `RealRadii` gives `prdc_counts`'s counts;
* `evaluate(prdc=True)` on 37 photos at R = 256: `EvalResult.prdc` is the call on the merged features, the bins' values
  are the calls on each bin's rows against the radii of all real rows (nan at k or fewer images), and W = 2 and 3
  virtual ranks print the lines of W = 1; `score_results --prdc` prints the lines in their order."""
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

from oracle import fid_oracle as FO  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402
from oracle import prdc_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

R = 256
N = 37
BATCH = 8
EDGES5 = (0.0, 0.2, 0.35, 0.5, 0.7, 1.0)


def device_counts(real, fake, k=3, stream=None):
    from migan_b200 import prdc
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
        out = prdc.prdc_counts(real, fake, k).cpu().numpy()
    return out


def check_against_oracle(real, fake, k, oracle_real=None, oracle_fake=None):
    """The library's counts and ratios against the oracle's, and the oracle's smallest margin above the bound."""
    from migan_b200 import prdc
    res = prdc.precision_recall_density_coverage(torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda(), k)
    got = device_counts(torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda(), k)
    want = O.prdc(real if oracle_real is None else oracle_real, fake if oracle_fake is None else oracle_fake, k,
                  chunk=64 if oracle_real is None else 8)
    bound = O.rounding_bound(real, fake)
    print("N %d M %d d %d k %d: counts %s (oracle %s), margin %.3g, bound %.3g"
          % (len(real), len(fake), real.shape[1], k, got.tolist(), want.counts.tolist(), want.margin, bound))
    assert (got == want.counts).all()
    assert tuple(res[:4]) == (want.precision, want.recall, want.density, want.coverage)
    assert res[4:] == (k, len(real), len(fake))
    return want, bound


@pytest.mark.parametrize("n_r,n_f,d,k,dtype", [
    (150, 97, 37, 3, np.float32), (70, 130, 100, 1, np.float64), (65, 66, 2048, 5, np.float32),
    (200, 201, 37, 3, np.float64), (300, 280, 2048, 3, np.float32)])
def test_library_matches_the_oracle_in_ragged_cases(lib, n_r, n_f, d, k, dtype):
    real, fake = O.features(n_r, d, 11).astype(dtype), O.features(n_f, d, 12, 0.02).astype(dtype)
    want, bound = check_against_oracle(real, fake, k)
    assert want.margin > 100 * bound
    assert 0 < want.counts[0] < n_f and 0 < want.counts[3] < n_r


def test_library_matches_the_oracle_at_10000_by_2048(lib):
    real, fake = O.features(10000, 2048, 1), O.features(10000, 2048, 2, 0.02)
    want, bound = check_against_oracle(real, fake, 3, torch.from_numpy(real).cuda().double(),
                                       torch.from_numpy(fake).cuda().double())
    assert want.margin > 100 * bound


@pytest.mark.parametrize("k", [1, 3, 5])
def test_integer_ties(lib, k):
    real = O.integer_features(150, 5, 3)
    fake = O.integer_features(97, 5, 4, dup_of=real, dups=30)
    got = device_counts(torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda(), k)
    want = O.prdc(real, fake, k)
    assert want.margin == 0.0 and (got == want.counts).all(), (got, want.counts)


def test_same_bytes_on_every_call_stream_dtype_and_order(lib):
    from migan_b200 import prdc
    real = torch.from_numpy(O.features(3000, 2048, 5)).cuda()
    fake = torch.from_numpy(O.features(2500, 2048, 6, 0.02)).cuda()
    a = device_counts(real, fake)
    b = device_counts(real, fake)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    c = device_counts(real, fake, stream=side)
    d = device_counts(real.double(), fake.double())
    pr, pf = torch.randperm(3000, generator=torch.Generator().manual_seed(1)), torch.randperm(
        2500, generator=torch.Generator().manual_seed(2))
    e = device_counts(real[pr.cuda()].contiguous(), fake[pf.cuda()].contiguous())
    print("counts", a.tolist())
    assert a.tobytes() == b.tobytes() == c.tobytes() == d.tobytes() == e.tobytes()
    swapped = device_counts(fake, real)
    assert (swapped[[1, 0]] == a[[0, 1]]).all()
    radii = prdc.RealRadii(real, 3, max_fake=2500)
    for rows in (fake, fake[:1000], fake[1500:].double()):
        want = prdc.precision_recall_density_coverage(real, rows)
        assert prdc.precision_recall_density_coverage(radii, rows) == want


# -- the commands -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("prdc")
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


def evaluate(data, mask_dir="masks", **kw):
    from migan_b200 import evaluate_fid_lpips as E
    return E.evaluate("migan-256", data["model"], data["real"], None if mask_dir is None else data[mask_dir],
                      batch_size=BATCH, inception_weights=data["inception"], lpips_weights=data["lpips"], **kw)


def printed(res, kid=False, prdc=True):
    from migan_b200 import evaluate_fid_lpips as E
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, False, False, False, kid, prdc)
    return out.getvalue().splitlines()


def virtual_ranks(setup, world):
    """Rank 0's merge of `world` virtual ranks run in turn on one GPU: (merge, result)."""
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features, extra_values=setup.extra_values,
                    hole_bins=setup.hole_bins, prdc=True)
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


def test_evaluate_prdc_is_the_call_on_the_merged_features(data):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import prdc
    res = evaluate(data, prdc=True, kid=True)
    setup = E.EvalSetup("migan-256", data["model"], data["real"], data["masks"], batch_size=BATCH,
                        inception_weights=data["inception"], lpips_weights=data["lpips"])
    merge, one = virtual_ranks(setup, 1)
    assert res.prdc == prdc.precision_recall_density_coverage(*merge.kept) == one.prdc and len(res) == 8
    plain = evaluate(data, kid=True)
    assert plain.prdc is None and (plain.fid, plain.lpips, plain.kid) == (res.fid, res.lpips, res.kid)
    lines = printed(res, kid=True)
    print("\n".join(lines))
    assert [ln.split(":")[0] for ln in lines[-4:]] == ["Precision", "Recall", "Density", "Coverage"]
    assert lines[-5].startswith("KID: ") and lines[:-4] == printed(plain, kid=True, prdc=False)
    for world in (2, 3):
        assert printed(virtual_ranks(setup, world)[1]) == printed(one), world


def test_hole_bins_prdc(data):
    from migan_b200 import evaluate_fid_lpips as E
    from migan_b200 import prdc
    res = evaluate(data, hole_bins=(0, 1), prdc=True)
    assert tuple(res.by_hole[0][-4:]) == tuple(res.prdc[:4]) and res.by_hole[0].count == N
    setup = E.EvalSetup("migan-256", data["model"], data["real"], data["masks"], batch_size=BATCH,
                        inception_weights=data["inception"], lpips_weights=data["lpips"], hole_bins=EDGES5)
    merge, res = virtual_ranks(setup, 1)
    h = merge.extra[:, 0].cpu().numpy().astype(np.float64)
    bins = np.searchsorted(np.array(EDGES5[1:-1]), h, side="right")
    assert sorted(set(bins.tolist())) == list(range(5)), bins
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert b.count == len(idx)
        if len(idx) > 3:
            at = torch.from_numpy(idx).cuda()
            want = prdc.precision_recall_density_coverage(merge.kept[0], merge.kept[1][at])
            assert tuple(b[-4:]) == tuple(want[:4]), k
        else:
            assert all(math.isnan(v) for v in b[-4:])
    lines = printed(res)
    print("\n".join(lines))
    assert all(ln.endswith("Precision %r Recall %r Density %r Coverage %r" % tuple(b[-4:]))
               for ln, b in zip(lines[-5:], res.by_hole))
    for world in (2, 3):
        assert printed(virtual_ranks(setup, world)[1]) == lines, world


PREFIXES = ("FID:", "LPIPS:", "SSIM:", "PSNR:", "P-IDS:", "U-IDS:", "KID:", "Precision:", "Recall:", "Density:",
            "Coverage:", "HOLE ")


def test_score_results_command(data):
    from migan_b200 import score_results as S
    res = S.score(data["real"], data["results"], data["masks"], resolution=R, batch_size=BATCH,
                  inception_weights=data["inception"], lpips_weights=data["lpips"], hole_bins=(0, 0.5, 1), prdc=True,
                  kid=True)
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m", "migan_b200.score_results", "--resolution", str(R), "--results-dir",
                        str(data["results"]), "--mask-dir", str(data["masks"]), "--hole-bins", "0,0.5,1", "--kid",
                        "--prdc", "--real-dir", str(data["real"]), "--batch-size", str(BATCH),
                        "--inception-weights", str(data["files"] / "inception.pth"),
                        "--lpips-weights", str(data["files"] / "lpips.pth")],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith(PREFIXES)]
    print("\n".join(lines))
    assert lines == printed(res, kid=True) and len(lines) == 2 + 1 + 4 + 2
    assert [ln.split(":")[0] for ln in lines[2:7]] == ["KID", "Precision", "Recall", "Density", "Coverage"]

"""P-IDS and U-IDS on the GPU: `ids.inception_discriminative_scores` against the float64 finite-Newton oracle at
N = 10,000 pairs of 2048-d features, against sklearn's LinearSVC(dual=False) on the stored fixture, on InceptionV3
features of EvalPipeline outputs, bitwise repeatability, and the evaluation command's `--ids`: the same bits at
W = 1, 2 and 3 (virtual ranks in one process), at --batch-size 8 and 32 for MI-GAN, and the four printed lines."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import comodgan_oracle as C  # noqa: E402
from oracle import fid_oracle as FO  # noqa: E402
from oracle import ids_oracle as O  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "ids.npz")
# Coefficients against the oracle, max |coef - oracle| / max |oracle coef|: both are the minimiser to float64 rounding,
# reached by different sums.  Measured on an H100: 3e-12 to 3e-11 on the gamma sets, 3.0e-9 on the 40 InceptionV3
# feature pairs (a separable set with tiny weights).
COEF_REL = 1e-8


def _check_against(got, sol, what):
    scale = float(np.abs(sol.coef).max())
    err = float(np.abs(got.coef - sol.coef).max()) / scale
    print("%s: P %.6f U %.6f f %.15g (oracle %.15g) residual %.2e, %d iterations (%s; oracle %d), coef err %.2e"
          % (what, got.p_ids, got.u_ids, got.objective, sol.objective, got.residual, got.iterations, got.stop_rule,
             sol.iterations, err))
    assert got.objective <= sol.objective * (1 + 1e-12)
    assert got.p_ids == sol.p_ids and got.u_ids == sol.u_ids
    assert err <= COEF_REL
    assert abs(got.intercept - sol.intercept) <= COEF_REL * max(scale, abs(sol.intercept))
    assert got.residual <= 1e-12 or got.stop_rule == "active set"


@pytest.mark.parametrize("kind", ["overlap", "separable"])
def test_against_oracle_at_10000_pairs(lib, kind):
    from migan_b200 import ids
    real, fake = O.features(10000, 2048, kind, seed=11)
    got = ids.inception_discriminative_scores(torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda())
    _check_against(got, O.solve(real, fake), "N=10000 %s" % kind)


def test_sklearn_fixture(lib):
    from migan_b200 import ids
    g = np.load(GOLDEN)
    for name in ("overlap2048", "separable2048", "n197", "d37"):
        real, fake = g[name + "_real"] / np.float32(64), g[name + "_fake"] / np.float32(64)
        n = len(real)
        got = ids.inception_discriminative_scores(real.astype(np.float32), fake.astype(np.float32))
        print("%s: f %.15g (sklearn %.15g), U %r (%r), P %r (%r)" % (name, got.objective, g[name + "_objective"],
                                                                    got.u_ids, g[name + "_u_ids"], got.p_ids,
                                                                    g[name + "_p_ids"]))
        assert got.objective <= g[name + "_objective"] * (1 + 1e-12)
        assert abs(got.u_ids - g[name + "_u_ids"]) * 2 * n <= g[name + "_u_rows"] + 1e-9
        assert abs(got.p_ids - g[name + "_p_ids"]) * n <= g[name + "_p_rows"] + 1e-9
        _check_against(got, O.solve(real, fake), name)
        got64 = ids.inception_discriminative_scores(real.astype(np.float64), fake.astype(np.float64))
        assert got64.coef.tobytes() == got.coef.tobytes() and got64.objective == got.objective   # exact promotion


def test_bitwise_repeatable_across_calls_and_streams(lib):
    from migan_b200 import ids
    real, fake = O.features(3000, 2048, "overlap", seed=5)
    r, f = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
    a = ids.inception_discriminative_scores(r, f)
    b = ids.inception_discriminative_scores(r, f)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = ids.inception_discriminative_scores(r, f)
    for x in (b, c):
        assert x.coef.tobytes() == a.coef.tobytes()
        assert (x.p_ids, x.u_ids, x.intercept, x.objective, x.residual, x.iterations) == \
            (a.p_ids, a.u_ids, a.intercept, a.objective, a.residual, a.iterations)


def test_refusals(lib):
    from migan_b200 import ids
    x = np.zeros((4, 8), np.float32)
    with pytest.raises(ValueError, match="same shape"):
        ids.inception_discriminative_scores(x, np.zeros((5, 8), np.float32))
    with pytest.raises(ValueError, match="no rows"):
        ids.inception_discriminative_scores(x[:0], x[:0])
    with pytest.raises(ValueError, match="outside 1..4096"):
        ids.inception_discriminative_scores(np.zeros((2, 4097)), np.zeros((2, 4097)))
    bad = x.copy()
    bad[1, 2] = np.nan
    with pytest.raises(ValueError, match="fake has non-finite"):
        ids.inception_discriminative_scores(torch.from_numpy(x).cuda(), torch.from_numpy(bad).cuda())


# -- the evaluation command -----------------------------------------------------------------------------------------

R = 256
N = 40


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib):
    from PIL import Image
    root = tmp_path_factory.mktemp("idsdata")
    real, masks = root / "real", root / "masks"
    real.mkdir()
    masks.mkdir()
    rng = np.random.default_rng(17)
    sizes = [(R, R), (R + 44, R * 3 // 2), (200, 180)]
    for i in range(N):
        h, w = sizes[i % len(sizes)]
        low = rng.random((max(2, h // 32), max(2, w // 32), 3))
        img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BILINEAR), np.float64)
        img = np.clip(0.85 * img + 0.15 * rng.integers(0, 256, (h, w, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(img).save(real / ("img_%03d.png" % i))
        m = np.where(rng.random((max(1, h // 16), max(1, w // 16))) < 0.35, 0, 255).astype(np.uint8)
        Image.fromarray(m).resize((w, h), Image.NEAREST).save(masks / ("img_%03d.png" % i))
    files = root / "files"
    files.mkdir()
    weights = {"model": MO.make_state_dict(R, seed=3), "inception": FO.seeded_state_dict(0),
               "lpips": LO.seeded_state_dict(0)}
    for k, v in weights.items():
        torch.save(v, files / ("%s.pth" % k))
    return {"real": real, "masks": masks, "files": files, **weights}


def run(data, model_name="migan-256", model=None, batch_size=8, **kw):
    from migan_b200 import evaluate_fid_lpips as E
    return E.evaluate(model_name, data["model"] if model is None else model, data["real"], data["masks"],
                      batch_size=batch_size, inception_weights=data["inception"], lpips_weights=data["lpips"], **kw)


def virtual_ranks(setup, world):
    """W ranks in one process; rank 0's merge keeps the features.  Returns (result, the kept features)."""
    from migan_b200 import evaluate_fid_lpips as E
    merge = E.Merge(len(setup.images), setup.device, setup.real_features, keep_features=True)
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
    return merge.result(), [k.cpu().numpy() for k in merge.kept]


def test_ranks_give_the_same_bits_and_match_the_oracle(data):
    from migan_b200 import evaluate_fid_lpips as E
    setup = E.EvalSetup("migan-256", data["model"], data["real"], data["masks"], batch_size=8,
                        inception_weights=data["inception"], lpips_weights=data["lpips"])
    one, feats = virtual_ranks(setup, 1)
    want = run(data, ids=True)
    assert (one.fid, one.p_ids, one.u_ids) == (want.fid, want.p_ids, want.u_ids)
    for world in (2, 3):
        got, f = virtual_ranks(setup, world)
        assert (got.fid, got.lpips, got.p_ids, got.u_ids) == (one.fid, one.lpips, one.p_ids, one.u_ids)
        assert all(np.array_equal(a, b) for a, b in zip(f, feats))
    sol = O.solve(*feats)                 # InceptionV3 features of EvalPipeline outputs
    print("inception features: P %r U %r, oracle P %r U %r" % (one.p_ids, one.u_ids, sol.p_ids, sol.u_ids))
    assert (one.p_ids, one.u_ids) == (sol.p_ids, sol.u_ids)
    from migan_b200 import ids
    _check_against(ids.inception_discriminative_scores(*feats), sol, "inception features")


def test_migan_scores_do_not_depend_on_the_batch_size(data):
    a, b = run(data, batch_size=8, ids=True), run(data, batch_size=32, ids=True)
    assert (a.p_ids, a.u_ids) == (b.p_ids, b.u_ids)
    plain = run(data, batch_size=8)
    assert plain.p_ids is None and plain.u_ids is None and plain.fid == a.fid and plain.lpips == a.lpips


def test_comodgan_runs(data):
    res = run(data, "comodgan-256", C.make_state_dict(R, seed=1), ids=True)
    assert 0 <= res.p_ids <= 1 and 0 <= res.u_ids <= 1 and np.isfinite(res.fid)


def test_main_prints_four_lines(data, capsys):
    from migan_b200 import evaluate_fid_lpips as E
    argv = ["--model-name", "migan-256", "--model-path", str(data["files"] / "model.pth"), "--real-dir",
            str(data["real"]), "--mask-dir", str(data["masks"]), "--batch-size", "8",
            "--inception-weights", str(data["files"] / "inception.pth"),
            "--lpips-weights", str(data["files"] / "lpips.pth")]
    E.main(argv)
    plain = capsys.readouterr().out.splitlines()
    E.main(argv + ["--ids"])
    lines = capsys.readouterr().out.splitlines()
    assert len(plain) == 2 and len(lines) == 4
    assert lines[:2] == plain
    assert lines[2].startswith("P-IDS: ") and lines[3].startswith("U-IDS: ")
    res = run(data, ids=True)
    assert lines[2:] == ["P-IDS: %r" % res.p_ids, "U-IDS: %r" % res.u_ids]


def test_torchrun_two_gpus_prints_the_same_scores(data):
    import subprocess
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs for torchrun --nproc_per_node=2; %d visible" % torch.cuda.device_count())
    cmd = ["-m", "migan_b200.evaluate_fid_lpips", "--model-name", "migan-256", "--model-path",
           str(data["files"] / "model.pth"), "--real-dir", str(data["real"]), "--mask-dir", str(data["masks"]),
           "--batch-size", "8", "--inception-weights", str(data["files"] / "inception.pth"),
           "--lpips-weights", str(data["files"] / "lpips.pth"), "--ids"]
    env = dict(os.environ, PYTHONPATH=ROOT)
    one = subprocess.run([sys.executable] + cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    two = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2"] + cmd,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert one.returncode == 0, one.stderr
    assert two.returncode == 0, two.stderr
    lines = [ln for ln in one.stdout.splitlines() if ln.startswith(("FID:", "LPIPS:", "P-IDS:", "U-IDS:"))]
    assert len(lines) == 4
    assert [ln for ln in two.stdout.splitlines() if ln.startswith(("FID:", "LPIPS:", "P-IDS:", "U-IDS:"))] == lines

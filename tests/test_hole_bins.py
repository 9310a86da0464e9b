"""Scores by hole size in `evaluate_fid_lpips` and `score_results`, on the CPU: the refusals of --hole-bins and
--hole-range (and of `RandomMaskStream`'s hole_range) before any work, the bin of a hole fraction at and between the
edges, the HOLE line format, and rank 0's per-bin merge, also through gloo at W = 2 and 3 against W = 1.  The feature
statistics, the distance and the discriminative scores are replaced by stand-ins that record rows, since they run on
CUDA only."""
import io
import math
import os
import socket
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from migan_b200 import evaluate_fid_lpips as E
from migan_b200 import fid, ids
from migan_b200 import masks as masks_mod
from migan_b200 import score_results as S


class RowStats:
    """`fid.FeatureStatistics` stand-in: keeps its rows; its 'mean' is their column sum."""

    def __init__(self, dim=fid.FEATURES, device="cpu"):
        self.rows = []

    def add(self, feats):
        self.rows.append(feats.clone())

    def mean_cov_device(self):
        return torch.cat(self.rows).double().sum(0), None

    def frechet_distance(self, other):
        return 0.0


class BinnedRows:
    """`fid.BinnedFeatureStatistics` stand-in: keeps every (feats, bins) call."""

    def __init__(self, nbins, dim=fid.FEATURES, device="cpu"):
        self.nbins, self.calls = nbins, []

    def add(self, feats, bins):
        assert bins.dtype == torch.int32
        self.calls.append((feats.clone(), bins.clone()))

    def counts(self):
        b = torch.cat([c[1] for c in self.calls]).numpy()
        return np.bincount(b[b >= 0], minlength=self.nbins).astype(np.int64)

    def mean_cov_device(self, b, count=None):
        rows = torch.cat([f[k == b] for f, k in self.calls])
        assert count == rows.shape[0]
        return rows.double().sum(0), rows


def fake_distance(mu1, sigma1, mu2, sigma2):
    return float(torch.as_tensor(mu1).sum()) * 1e-6 + float(mu2.sum())


class FakeScores:
    def __init__(self, p, u):
        self.p_ids, self.u_ids = p, u


def fake_ids(real, fake):
    return FakeScores(float(real.double().sum()), float(fake.double().mean()))


@pytest.fixture
def stand_ins(monkeypatch):
    monkeypatch.setattr(fid, "FeatureStatistics", RowStats)
    monkeypatch.setattr(fid, "BinnedFeatureStatistics", BinnedRows)
    monkeypatch.setattr(fid, "frechet_distance", fake_distance)
    monkeypatch.setattr(ids, "inception_discriminative_scores", fake_ids)


EXTRA = ("hole_fraction", "ssim", "psnr")
EDGES = (0.0, 0.25, 3 / 7, 0.6, 1.0)


def stand_in(j, chunks, extra_values):
    a, b = chunks[j]
    idx = torch.arange(a, b, dtype=torch.float32)[:, None]
    col = torch.arange(fid.FEATURES, dtype=torch.float32)[None]
    i = idx[:, 0]
    values = {"hole_fraction": (i % 8) / 7, "ssim": torch.cos(i * 0.3) * 0.4 + 0.5, "psnr": 12 + i / 3}
    extra = torch.stack([values[v] for v in extra_values], 1)
    return E.ChunkResult(j, a, torch.sin(idx * 0.37 + col * 0.011), torch.cos(idx * 0.53 - col * 0.007) / 3,
                         torch.tanh(i / 9), extra)


def merged(n, batch, extra_values, edges, keep=True, chunk_results=None, real_stats=None):
    chunks = E.chunk_bounds(n, batch)
    merge = E.Merge(n, "cpu", True, keep_features=keep, extra_values=extra_values, hole_bins=edges)
    for c in chunk_results if chunk_results is not None else [stand_in(j, chunks, extra_values)
                                                              for j in range(len(chunks))]:
        merge.add(c)
    return merge.result(real_stats)


# -- refusals -----------------------------------------------------------------------------------------------------------

def _eval_argv(tmp_path, *extra):
    return ["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", str(tmp_path)] + list(extra)


def _score_argv(tmp_path, *extra):
    return ["--resolution", "256", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)] + list(extra)


@pytest.mark.parametrize("command,argv", [(E, _eval_argv), (S, _score_argv)], ids=["evaluate_fid_lpips", "score_results"])
@pytest.mark.parametrize("flags,match", [
    (["--hole-bins", "0,0.5"], "from 0 to 1"), (["--hole-bins", "0.1,1"], "from 0 to 1"),
    (["--hole-bins", "0,0.5,0.5,1"], "strictly"), (["--hole-bins", "0,0.6,0.5,1"], "strictly"),
    (["--hole-bins", "0,a,1"], "comma-separated"), (["--hole-bins", "1"], "edges"),
    (["--hole-bins", "0,nan,1"], "strictly|from 0 to 1"),
    (["--hole-bins", ",".join(str(k / 33) for k in range(34))], "34 edges"),
    (["--hole-range", "0.5", "0.4"], "hole_range"), (["--hole-range", "0", "1.5"], "hole_range"),
    (["--hole-range", "0.0", "0.1"], "randint"), (["--hole-range", "nan", "1"], "hole_range"),
    (["--hole-range", "0", "1", "--mask-dir", "m"], "--mask-dir"),
    (["--hole-range", "0.2", "0.4", "--mask-dir", "m"], "--mask-dir")])
def test_refusals_before_any_work(tmp_path, command, argv, flags, match):
    with pytest.raises(ValueError, match=match):                        # a CPU device would be refused later
        command.main(argv(tmp_path, *flags, "--device", "cpu"))


def test_library_refusals_before_any_work(tmp_path):
    with pytest.raises(ValueError, match="--mask-dir"):
        E.evaluate("migan-256", None, tmp_path, tmp_path, device="cpu", hole_range=(0.2, 0.4))
    with pytest.raises(ValueError, match="strictly"):
        S.score(tmp_path, tmp_path, resolution=256, device="cpu", hole_bins=(0, 1, 1))
    with pytest.raises(ValueError, match="randint"):
        masks_mod.RandomMaskStream(64, device="cpu", hole_range=(0.05, 0.1))
    with pytest.raises(ValueError, match="hole_range"):
        masks_mod.RandomMaskStream(64, device="cpu", hole_range=(0.3,))
    assert E.check_hole_args([0, 1], [0, 1], "masks") == ((0.0, 1.0), (0.0, 1.0))
    assert E.check_hole_bins([0] + [k / 32 for k in range(1, 32)] + [1]) == tuple(k / 32 for k in range(33))


def test_flags_parse(tmp_path):
    a = E.get_args(_eval_argv(tmp_path))
    assert (a.hole_bins, a.hole_range) == (None, None)
    assert E.check_hole_flags(a) == (None, (0.0, 1.0))
    a = S.get_args(_score_argv(tmp_path, "--hole-bins", "0,0.1,1", "--hole-range", "0.1", "0.3"))
    assert E.check_hole_flags(a) == ((0.0, 0.1, 1.0), (0.1, 0.3))


# -- bins and lines ---------------------------------------------------------------------------------------------------

def test_bin_of_a_hole_fraction():
    inner = torch.tensor(EDGES[1:-1], dtype=torch.float64)
    h = torch.tensor([0.0, 0.25, np.nextafter(np.float32(0.25), np.float32(0)), 0.6, 1.0, np.float32(3 / 7), 0.99],
                     dtype=torch.float32)
    got = E.hole_bin_index(h, inner)
    assert got.dtype == torch.int32
    # float32 3/7 is above the float64 edge 3/7, so it lies in the bin that edge opens
    assert float(np.float32(3 / 7)) > 3 / 7
    assert got.tolist() == [0, 1, 0, 3, 3, 2, 3]
    assert E.hole_bin_index(torch.tensor([0.0, 0.5, 1.0]), torch.zeros(0, dtype=torch.float64)).tolist() == [0, 0, 0]


def test_hole_line_format():
    b = E.HoleBin(0.0, 0.1, 812, 3.52, 0.0412)
    assert E.hole_line(b, False) == "HOLE [0.0, 0.1): images 812 FID 3.52 LPIPS 0.0412"
    b = E.HoleBin(0.6, 1.0, 1, math.nan, 0.25, 0.5, math.inf, math.nan, math.nan)
    assert E.hole_line(b, True) == "HOLE [0.6, 1.0]: images 1 FID nan LPIPS 0.25 SSIM 0.5 PSNR inf P-IDS nan U-IDS nan"
    b = E.HoleBin(0.2, 0.3, 0, math.nan, math.nan, None, 30.0)
    assert E.hole_line(b, False) == "HOLE [0.2, 0.3): images 0 FID nan LPIPS nan PSNR 30.0"


def _printed(res, *flags):
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, *flags)
    return out.getvalue().splitlines()


def test_merge_per_bin(stand_ins):
    n, batch = 29, 8
    res = merged(n, batch, EXTRA, EDGES)
    chunks = E.chunk_bounds(n, batch)
    parts = [stand_in(j, chunks, EXTRA) for j in range(len(chunks))]
    h = torch.cat([p.extra[:, 0] for p in parts]).numpy().astype(np.float64)
    bins = np.searchsorted(np.array(EDGES[1:-1]), h, side="right")
    real_sum = torch.cat([p.real for p in parts]).double().sum(0)
    fake = torch.cat([p.fake for p in parts])
    assert len(res.by_hole) == 4 and res.per_image is None
    for k, b in enumerate(res.by_hole):
        idx = np.flatnonzero(bins == k)
        assert (b.lo, b.hi, b.count) == (EDGES[k], EDGES[k + 1], len(idx))
        want_fid = float(real_sum.sum()) * 1e-6 + float(fake[idx].double().sum(0).sum())
        assert b.fid == want_fid
        assert b.lpips == float(np.mean(res.lpips_values[idx]))
        ssim = torch.cat([p.extra[:, 1] for p in parts]).numpy().astype(np.float64)
        assert b.ssim == float(np.mean(ssim[idx]))
        assert b.p_ids == fake_ids(torch.cat([p.real for p in parts])[idx], fake[idx]).p_ids
    lines = _printed(res, True, True, True)
    assert lines[:2] == ["FID: 0.0", "LPIPS:  %r" % res.lpips] and len(lines) == 6 + 4
    assert lines[6].startswith("HOLE [0.0, 0.25): images %d FID " % (bins == 0).sum())
    assert lines[-1].startswith("HOLE [0.6, 1.0]: ")
    # stored statistics: every bin against them
    res = merged(n, batch, EXTRA, EDGES, keep=False, real_stats=(np.full(4, 2.0), None))
    assert res.by_hole[0].fid == 8e-6 + float(fake[bins == 0].double().sum(0).sum())
    assert res.by_hole[0].p_ids is None


def test_small_and_empty_bins(stand_ins):
    res = merged(4, 2, ("hole_fraction",), (0.0, 0.1, 0.2, 0.3, 1.0))   # h = 0, 1/7, 2/7, 3/7
    assert [b.count for b in res.by_hole] == [1, 1, 1, 1]
    assert all(math.isnan(b.fid) and math.isnan(b.p_ids) and not math.isnan(b.lpips) for b in res.by_hole)
    assert (res.by_hole[0].ssim, res.by_hole[0].psnr) == (None, None)
    res = merged(4, 2, ("hole_fraction",), (0.0, 0.05, 0.9, 0.95, 1.0), keep=False)
    assert [b.count for b in res.by_hole] == [1, 3, 0, 0]
    assert math.isnan(res.by_hole[2].lpips) and math.isnan(res.by_hole[2].fid) and res.by_hole[2].p_ids is None
    with pytest.raises(ValueError, match="hole fraction"):
        E.Merge(4, "cpu", True, extra_values=("ssim",), hole_bins=(0, 1))


def test_without_bins_nothing_changes(stand_ins):
    res = merged(20, 8, ("hole_fraction",), None)
    assert res.by_hole is None and E.EvalResult(1.0, 0.5, np.zeros(2), 2).by_hole is None
    assert _printed(res, False) == ["FID: 0.0", "LPIPS:  %r" % res.lpips]


# -- transport over gloo --------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


CASES = [(70, 8, EXTRA, EDGES), (5, 2, ("hole_fraction",), (0.0, 1.0)), (33, 32, ("hole_fraction", "psnr"), EDGES)]


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    fid.FeatureStatistics, fid.BinnedFeatureStatistics, fid.frechet_distance = RowStats, BinnedRows, fake_distance
    ids.inception_discriminative_scores = fake_ids
    for case, (n, batch, extra_values, edges) in enumerate(CASES):
        chunks = E.chunk_bounds(n, batch)
        width = 2 * fid.FEATURES + 1 + len(extra_values)
        received = []
        for r in range(E.num_rounds(len(chunks), world)):
            j = E.round_chunk(r, rank, len(chunks), world)
            mine = None if j is None else stand_in(j, chunks, extra_values)
            received += E.gather_round(mine, r, chunks, width, "cpu", extra=len(extra_values))
        if rank == 0:
            res = merged(n, batch, extra_values, edges, chunk_results=received)
            torch.save({"lines": _printed(res, True, "ssim" in extra_values, "psnr" in extra_values),
                        "by_hole": res.by_hole}, os.path.join(out_dir, "case%d.pt" % case))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_print_the_bins_of_one_rank(tmp_path, stand_ins, world):
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for case, (n, batch, extra_values, edges) in enumerate(CASES):
        got = torch.load(tmp_path / ("case%d.pt" % case), weights_only=False)
        one = merged(n, batch, extra_values, edges)
        assert got["lines"] == _printed(one, True, "ssim" in extra_values, "psnr" in extra_values)
        assert len(got["by_hole"]) == len(edges) - 1
        for g, w in zip(got["by_hole"], one.by_hole):
            assert tuple(g) == tuple(w) or all(a == b or (a != a and b != b) for a, b in zip(g, w))


def test_generate_masks_refuses_a_range_before_any_work(tmp_path):
    from migan_b200 import generate_masks
    with pytest.raises(ValueError, match="randint"):
        generate_masks.main(["--images-dir", str(tmp_path), "--output-dir", str(tmp_path / "out"), "--resolution", "64",
                             "--hole-range", "0", "0.1"])
    assert not (tmp_path / "out").exists()

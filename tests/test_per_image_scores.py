"""Per-image scores, SSIM and PSNR in `evaluate_fid_lpips` and `score_results`, on the CPU: the flags of both commands,
the result lines and their order, rank 0's merge of the per-image values into `EvalResult` and the `--per-image` CSV
(header, sorted row order, `repr(float)`, inf PSNR), and the round transport over gloo with stand-in chunk results
(W = 2 and 3 write the CSV bytes of W = 1; without the new flags the gathered buffer keeps its width).  The feature
statistics are replaced by a stand-in that records rows, since `FeatureStatistics` runs on CUDA only."""
import csv
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
from migan_b200 import fid
from migan_b200 import score_results as S


class RowStats:
    """`fid.FeatureStatistics` stand-in: keeps the rows it is given; the distance is 0."""

    def __init__(self, dim=fid.FEATURES, device="cpu"):
        self.rows = []

    def add(self, feats):
        self.rows.append(feats.clone())

    def frechet_distance(self, other):
        return 0.0


NAMES = ["a,b.jpg", "img \"q\".png"]                      # quoting in the CSV


def names(n):
    return [NAMES[i] if i < len(NAMES) else "img_%04d.jpg" % i for i in range(n)]


def stand_in(j, chunks, real, extra_values):
    """A chunk's results as a function of its global image indices; PSNR is inf for every 7th image."""
    a, b = chunks[j]
    idx = torch.arange(a, b, dtype=torch.float32)[:, None]
    col = torch.arange(fid.FEATURES, dtype=torch.float32)[None]
    feats_r = torch.sin(idx * 0.37 + col * 0.011)
    feats_f = torch.cos(idx * 0.53 - col * 0.007) / 3
    i = idx[:, 0]
    values = {"hole_fraction": (i % 5) / 7, "ssim": torch.cos(i * 0.3) * 0.4 + 0.5,
              "psnr": torch.where(i % 7 == 0, torch.full_like(i, float("inf")), 12 + i / 3)}
    extra = torch.stack([values[v] for v in extra_values], 1) if extra_values else None
    return E.ChunkResult(j, a, feats_r if real else None, feats_f, torch.tanh(i / 9), extra)


def merged(n, batch, extra_values, per_image, chunk_results=None):
    """Rank 0's `Merge` over the stand-in chunks (W = 1 when `chunk_results` is None)."""
    chunks = E.chunk_bounds(n, batch)
    merge = E.Merge(n, "cpu", True, extra_values=extra_values, names=names(n) if per_image else None)
    for c in chunk_results if chunk_results is not None else [stand_in(j, chunks, True, extra_values)
                                                              for j in range(len(chunks))]:
        merge.add(c)
    return merge.result()


def csv_bytes(res, tmp_path, name="scores.csv"):
    path = tmp_path / name
    E.write_per_image(path, res.per_image)
    return path.read_bytes()


@pytest.fixture
def row_stats(monkeypatch):
    monkeypatch.setattr(fid, "FeatureStatistics", RowStats)


# -- flags ------------------------------------------------------------------------------------------------------------

def _eval_argv(tmp_path, *extra):
    return ["--model-name", "migan-256", "--model-path", "m.pt", "--real-dir", str(tmp_path)] + list(extra)


def _score_argv(tmp_path, *extra):
    return ["--resolution", "256", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)] + list(extra)


@pytest.mark.parametrize("command,argv", [(E, _eval_argv), (S, _score_argv)], ids=["evaluate_fid_lpips", "score_results"])
def test_flags_parse(tmp_path, command, argv):
    a = command.get_args(argv(tmp_path))
    assert (a.ssim, a.psnr, a.per_image) == (False, False, None)
    a = command.get_args(argv(tmp_path, "--ssim", "--psnr", "--per-image", "out/scores.csv"))
    assert (a.ssim, a.psnr, str(a.per_image)) == (True, True, "out/scores.csv")
    a = command.get_args(argv(tmp_path, "--psnr"))
    assert (a.ssim, a.psnr, a.per_image) == (False, True, None)


@pytest.mark.parametrize("command,argv", [(E, _eval_argv), (S, _score_argv)], ids=["evaluate_fid_lpips", "score_results"])
def test_refusals(tmp_path, command, argv):
    with pytest.raises(ValueError, match="--per-image"):                 # before any device work
        command.main(argv(tmp_path, "--per-image", str(tmp_path / "missing" / "x.csv"), "--device", "cpu"))
    # --per-image with stored statistics is allowed: the refusal that follows is the device's, not the arguments'
    with pytest.raises(RuntimeError, match="CUDA"):
        command.main(argv(tmp_path, "--real-stats", "r.npz", "--per-image", str(tmp_path / "x.csv"), "--ssim",
                          "--psnr", "--device", "cpu"))
    with pytest.raises(ValueError, match="--ids"):                       # the existing refusals stand
        command.main(argv(tmp_path, "--real-stats", "r.npz", "--ids", "--per-image", str(tmp_path / "x.csv")))
    assert not (tmp_path / "x.csv").exists()


# -- the result and its lines ---------------------------------------------------------------------------------------

def test_result_tuple_is_unchanged_and_extras_ride_outside_it():
    res = E.EvalResult(1.5, 0.25, np.zeros(3), 3)
    assert len(res) == 8 and res._fields == ("fid", "lpips", "lpips_values", "count", "decode_wait_s", "seconds",
                                             "p_ids", "u_ids")
    assert (res.ssim, res.psnr, res.per_image) == (None, None, None)
    fid_, lp, vals, count, *_ = res
    assert (fid_, lp, count) == (1.5, 0.25, 3)
    res.ssim, res.per_image = 0.5, {"name": ["x"]}
    again = res._replace(seconds=2.0)
    assert again.seconds == 2.0 and again.ssim == 0.5 and again.per_image == {"name": ["x"]} and again.psnr is None
    assert len(again) == 8 and tuple(again)[:2] == (1.5, 0.25)


def _printed(res, *flags):
    out = io.StringIO()
    with redirect_stdout(out):
        E.print_result(res, *flags)
    return out.getvalue().splitlines()


def test_lines_and_their_order(row_stats):
    res = merged(20, 8, ("ssim", "psnr"), False)
    res = res._replace(p_ids=0.125, u_ids=0.375)
    base = ["FID: %r" % res.fid, "LPIPS:  %r" % res.lpips]
    assert _printed(res, False) == base
    assert _printed(res, False, False, False) == base
    assert _printed(res, True, True, True) == base + ["SSIM: %r" % res.ssim, "PSNR: inf", "P-IDS: 0.125",
                                                      "U-IDS: 0.375"]
    assert _printed(res, False, False, True) == base + ["PSNR: inf"]
    assert _printed(None, True, True, True) == []


# -- rank 0's merge and the CSV ---------------------------------------------------------------------------------------

def test_merge_without_new_values_is_unchanged(row_stats):
    n, batch = 20, 8
    res = merged(n, batch, (), False)
    chunks = E.chunk_bounds(n, batch)
    want = torch.cat([stand_in(j, chunks, True, ()).lpips for j in range(len(chunks))]).numpy().astype(np.float64)
    assert res.count == n and res.lpips_values.dtype == np.float64 and np.array_equal(res.lpips_values, want)
    assert res.lpips == float(np.mean(want)) and res.fid == 0.0
    assert (res.ssim, res.psnr, res.per_image) == (None, None, None)
    merge = E.Merge(n, "cpu", True)
    assert merge.extra is None and merge.names is None
    with pytest.raises(ValueError):
        E.Merge(n, "cpu", True, extra_values=("lpips",))


def test_csv_header_order_and_repr(row_stats, tmp_path):
    n = 20
    res = merged(n, 8, E.EXTRA_VALUES, True)
    chunks = E.chunk_bounds(n, 8)
    parts = [stand_in(j, chunks, True, E.EXTRA_VALUES) for j in range(len(chunks))]
    want = {v: torch.cat([p.extra[:, k] for p in parts]).numpy().astype(np.float64)
            for k, v in enumerate(E.EXTRA_VALUES)}
    assert list(res.per_image) == ["name", "hole_fraction", "lpips", "ssim", "psnr"]
    assert res.per_image["name"] == names(n)
    for v in E.EXTRA_VALUES:
        assert res.per_image[v].dtype == np.float64 and np.array_equal(res.per_image[v], want[v])
    assert res.per_image["lpips"] is res.lpips_values
    assert res.ssim == float(np.mean(want["ssim"]))
    text = csv_bytes(res, tmp_path).decode("utf-8")
    lines = text.split("\n")
    assert lines[0] == "name,hole_fraction,lpips,ssim,psnr" and lines[-1] == "" and len(lines) == n + 2
    assert lines[1].startswith('"a,b.jpg",') and lines[2].startswith('"img ""q"".png",')
    rows = list(csv.reader(io.StringIO(text)))[1:]
    assert [r[0] for r in rows] == names(n)
    for i, r in enumerate(rows):
        assert r[1:] == [repr(float(res.per_image[k][i])) for k in ("hole_fraction", "lpips", "ssim", "psnr")]
    assert rows[3][1] == repr(float(np.float32(3 / 7)))                 # float32 value, float64 repr
    assert not list(tmp_path.glob(".*.tmp"))                             # the temporary name is gone


def test_inf_psnr_is_written_and_averaged(row_stats, tmp_path):
    res = merged(20, 8, ("hole_fraction", "psnr"), True)
    psnr = res.per_image["psnr"]
    assert np.isinf(psnr[0]) and np.isinf(psnr[7]) and np.isinf(psnr[14]) and np.isfinite(psnr[1])
    assert res.psnr == math.inf and res.ssim is None
    rows = list(csv.reader(io.StringIO(csv_bytes(res, tmp_path).decode())))
    assert rows[0] == ["name", "hole_fraction", "lpips", "psnr"]
    assert [r[3] for r in rows[1:] if r[3] == "inf"] == ["inf"] * 3 and rows[1][3] == "inf"
    merge = E.Merge(5, "cpu", True, extra_values=("psnr",))
    merge.add(stand_in(0, [(1, 6)], True, ("psnr",))._replace(start=0))  # images 1..5: no inf, a finite mean
    res = merge.result()
    assert res.per_image is None and math.isfinite(res.psnr)


def test_csv_replaces_an_existing_file(row_stats, tmp_path):
    path = tmp_path / "scores.csv"
    path.write_text("old contents that are longer than nothing\n" * 100)
    res = merged(5, 2, ("hole_fraction",), True)
    E.write_per_image(path, res.per_image)
    assert path.read_text().split("\n")[0] == "name,hole_fraction,lpips" and len(path.read_text().split("\n")) == 7


# -- transport over gloo --------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


CASES = [(70, 8, ()), (70, 8, E.EXTRA_VALUES), (5, 2, ("hole_fraction", "psnr")), (33, 32, ("hole_fraction",))]


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    fid.FeatureStatistics = RowStats
    widths = []
    gather = dist.gather

    def recording(buf, *a, **k):
        widths.append(tuple(buf.shape))
        return gather(buf, *a, **k)

    E.dist.gather = recording
    for case, (n, batch, extra_values) in enumerate(CASES):
        chunks = E.chunk_bounds(n, batch)
        width = 2 * fid.FEATURES + 1 + len(extra_values)
        received = []
        for r in range(E.num_rounds(len(chunks), world)):
            j = E.round_chunk(r, rank, len(chunks), world)
            mine = None if j is None else stand_in(j, chunks, True, extra_values)
            received += E.gather_round(mine, r, chunks, width, "cpu", extra=len(extra_values))
        assert set(widths) == {(batch, width)}
        widths.clear()
        if rank == 0:
            res = merged(n, batch, extra_values, bool(extra_values), received)
            torch.save({"chunks": [tuple(c) for c in received], "fid": res.fid, "lpips": res.lpips,
                        "lpips_values": res.lpips_values, "ssim": res.ssim, "psnr": res.psnr},
                       os.path.join(out_dir, "case%d.pt" % case))
            if extra_values:
                E.write_per_image(os.path.join(out_dir, "case%d.csv" % case), res.per_image)
        else:
            assert received == []
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_write_the_csv_bytes_of_one_rank(tmp_path, row_stats, world):
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for case, (n, batch, extra_values) in enumerate(CASES):
        chunks = E.chunk_bounds(n, batch)
        got = torch.load(tmp_path / ("case%d.pt" % case), weights_only=False)
        want = [stand_in(j, chunks, True, extra_values) for j in range(len(chunks))]
        assert len(got["chunks"]) == len(chunks)
        for g, w in zip(got["chunks"], want):
            g = E.ChunkResult(*g)
            assert (g.index, g.start) == (w.index, w.start)
            assert torch.equal(g.real, w.real) and torch.equal(g.fake, w.fake) and torch.equal(g.lpips, w.lpips)
            assert (g.extra is None) == (not extra_values)
            if extra_values:
                assert torch.equal(g.extra, w.extra)
        one = merged(n, batch, extra_values, bool(extra_values))
        assert (got["fid"], got["lpips"], got["ssim"], got["psnr"]) == (one.fid, one.lpips, one.ssim, one.psnr)
        assert np.array_equal(got["lpips_values"], one.lpips_values)
        if extra_values:
            assert (tmp_path / ("case%d.csv" % case)).read_bytes() == csv_bytes(one, tmp_path, "one%d.csv" % case)

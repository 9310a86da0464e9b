"""pytorch_fid's command line on the GPU: FID between two image folders (or stored statistics), on one GPU or all the
GPUs of a box, with KID and precision / recall / density / coverage on request.

    python -m migan_b200.fid_score PATH PATH [--batch-size 50] [--num-workers N] [--dims 2048] [--save-stats]
                                             [--device cuda] [--inception-weights FILE] [--kid] [--prdc]
    torchrun --nproc_per_node=8 -m migan_b200.fid_score PATH PATH ...

pytorch_fid 0.3's `fid_score.main`, restated:

* a PATH is a directory or an `.npz` holding `mu` and `sigma` (pytorch_fid's statistics file); a path that does not
  exist is refused with its name;
* a directory's images are its top-level files matching `*.<ext>` for ext in bmp, jpg, jpeg, pgm, png, ppm, tif, tiff,
  webp (case-sensitive, as `Path.glob` is on Linux), sorted by path; fewer than 2 is refused, because the covariance
  needs two;
* each image is decoded with `Image.open(p).convert("RGB")` on a host thread pool and goes through the network at its
  own size (pytorch_fid's `ToTensor`, then InceptionV3's bilinear resize to 299 x 299).  Before any GPU work one
  planning pass opens every file and raises one `demo_command.PlanError` naming each unreadable one;
* it prints `FID:  <value>` as pytorch_fid does;
* `--save-stats PATH OUT` writes the folder's `mu` and `sigma` (float64) with `np.savez_compressed` and refuses to
  overwrite an existing file.

Differences from pytorch_fid:

* the photos go to the device as uint8, packed into one buffer per batch, and a batch may mix sizes
  (`fid.InceptionV3.features_u8`); pytorch_fid uploads float32 and fails on a batch of two sizes;
* `--batch-size` sets the chunking and nothing else: the features, and every printed number, are the same bytes for
  any batch size and any number of GPUs.  The feature statistics are summed in groups of `STATS_ROWS` rows in listing
  order, whatever the chunking;
* FID is computed on the GPU: `FeatureStatistics.frechet_distance` for two folders, `fid.frechet_distance` against an
  `.npz`'s `mu` and `sigma`.  `--dims` takes 2048 only (`fid.InceptionV3` builds block 3 alone);
* `--kid` prints `KID: <repr>` (`kid.kernel_inception_distance`) and `--prdc` prints `Precision:`, `Recall:`,
  `Density:` and `Coverage:` (`prdc.precision_recall_density_coverage`, k = 3), as the evaluation command does, with
  the first folder as real and the second as fake.  Both need two directories;
* `--inception-weights` takes a state_dict file; without it the cached weight file is read, as `fid.InceptionV3()`
  does.  Nothing is downloaded.

Sharding: a folder's sorted list is cut into chunks of `--batch-size` images and chunk j runs on rank j % W
(`evaluate_fid_lpips.chunk_bounds` / `round_chunk`); each round's features reach rank 0 in one gather
(`evaluate_fid_lpips.gather_round`), where they are kept in listing order.
"""
from __future__ import annotations

import argparse
import os
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist

from . import evaluate_fid_lpips as E
from . import fid
from . import kid as kid_metric
from . import prdc as prdc_metric
from .demo_command import PlanError, _header

IMAGE_EXTENSIONS = ("bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp")
DIMS = (2048,)
BATCH_SIZE = 50
STATS_ROWS = 4096               # feature rows per FeatureStatistics.add, independent of the chunking


def default_num_workers() -> int:
    """pytorch_fid's default: the CPUs this process may run on, at most 8."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    return min(n, 8)


# -- paths ----------------------------------------------------------------------------------------------------------

def is_stats_file(path) -> bool:
    """pytorch_fid's rule: a path ending in `.npz` holds statistics, any other is a directory of images."""
    return str(path).endswith(".npz")


def list_images(path) -> List[Path]:
    """The top-level files of directory `path` matching `*.<ext>` for ext in IMAGE_EXTENSIONS, sorted by path."""
    path = Path(path)
    return sorted(f for ext in IMAGE_EXTENSIONS for f in path.glob("*.{}".format(ext)))


def load_stats(path) -> Tuple[np.ndarray, np.ndarray]:
    """(mu, sigma) of a pytorch_fid `.npz`, as float64."""
    with np.load(path) as f:
        return np.asarray(f["mu"], dtype=np.float64), np.asarray(f["sigma"], dtype=np.float64)


def save_stats(path, mu: np.ndarray, sigma: np.ndarray) -> None:
    """pytorch_fid's `--save-stats` file: np.savez_compressed(path, mu=mu, sigma=sigma) in float64."""
    np.savez_compressed(path, mu=np.asarray(mu, dtype=np.float64), sigma=np.asarray(sigma, dtype=np.float64))


def check_paths(paths: Sequence, save_stats: bool = False, kid: bool = False, prdc: bool = False) -> None:
    """The refusals of the command line, before any file is read."""
    if len(paths) != 2:
        raise ValueError("expected two paths, got %d" % len(paths))
    if save_stats:
        if kid or prdc:
            raise ValueError("--kid and --prdc compare two folders; --save-stats writes one folder's statistics")
        if not os.path.exists(paths[0]):
            raise RuntimeError("Invalid path: %s" % paths[0])
        if is_stats_file(paths[0]) or not os.path.isdir(paths[0]):
            raise ValueError("--save-stats: the first path must be a directory of images, got %s" % paths[0])
        if os.path.exists(paths[1]):
            raise RuntimeError("Existing output file: %s" % paths[1])
        return
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError("Invalid path: %s" % p)
    for p in paths:
        if (kid or prdc) and is_stats_file(p):
            raise ValueError("--%s needs the images' features, which a statistics file (%s) does not carry"
                             % ("kid" if kid else "prdc", p))


def plan_folder(path, num_workers: int = 1) -> List[Path]:
    """The sorted image list of directory `path`, each file opened once (its header: no pixels are decoded).  Fewer than
    2 images raise ValueError; unreadable files raise one `PlanError` naming each."""
    if not os.path.isdir(path):
        raise ValueError("%s is neither a directory nor an .npz file" % path)
    files = list_images(path)
    if len(files) < 2:
        raise ValueError("%s holds %d images; the covariance needs at least 2" % (path, len(files)))

    def look(f: Path) -> Optional[str]:
        try:
            _header(f)
        except Exception as e:  # noqa: BLE001 -- any unreadable file is reported with the others
            return "%s: cannot be read (%s)" % (f, e)
        return None

    with ThreadPoolExecutor(max_workers=max(1, int(num_workers))) as pool:
        problems = [p for p in pool.map(look, files) if p is not None]
    if problems:
        raise PlanError(problems)
    return files


# -- features -------------------------------------------------------------------------------------------------------

class FolderFeatures(NamedTuple):
    """Rank 0's features of a folder in listing order (float32 [n, 2048] on the device; None on the other ranks) and the
    host time this rank spent waiting for decoded photos."""
    features: Optional[torch.Tensor]
    decode_wait_s: float


def folder_features(files: Sequence[Path], model: fid.InceptionV3, batch_size: int = BATCH_SIZE, device="cuda",
                    num_workers: int = 1) -> FolderFeatures:
    """The features of `files` (a `plan_folder` list), chunked by `batch_size`: alone, or in an initialised process
    group as one rank of the round-robin sharding, gathered to rank 0.  `model` is called as
    `model.features_u8(photos, device)` once per chunk."""
    if batch_size < 1:
        raise ValueError("--batch-size must be >= 1, got %d" % batch_size)
    device = torch.device(device)
    distributed = dist.is_available() and dist.is_initialized()
    world, rank = (dist.get_world_size(), dist.get_rank()) if distributed else (1, 0)
    chunks = E.chunk_bounds(len(files), int(batch_size))
    own = list(range(rank, len(chunks), world))
    out = torch.empty((len(files), fid.FEATURES), dtype=torch.float32, device=device) if rank == 0 else None
    wait = 0.0
    with ThreadPoolExecutor(max_workers=max(1, int(num_workers))) as pool:
        pending = deque()

        def submit():
            while len(pending) < E.PREFETCH and own:
                a, b = chunks[own.pop(0)]
                pending.append([pool.submit(E.decode_photo, f) for f in files[a:b]])

        for r in range(E.num_rounds(len(chunks), world)):
            j = E.round_chunk(r, rank, len(chunks), world)
            got = None
            if j is not None:
                submit()
                futs = pending.popleft()
                t = time.perf_counter()
                photos = [f.result() for f in futs]
                wait += time.perf_counter() - t
                submit()                 # keep PREFETCH chunks decoding while the GPU works
                got = E.ChunkResult(j, chunks[j][0], None, model.features_u8(photos, device), None)
            got = E.gather_round(got, r, chunks, fid.FEATURES, device, lpips=False) if distributed else [got]
            for c in got:
                out[c.start:c.start + c.fake.shape[0]] = c.fake
    return FolderFeatures(out, wait)


def feature_statistics(features: torch.Tensor) -> fid.FeatureStatistics:
    """FeatureStatistics of the rows in order, added STATS_ROWS at a time (so the sums do not depend on the chunking)."""
    stats = fid.FeatureStatistics(device=features.device)
    for a in range(0, features.shape[0], STATS_ROWS):
        stats.add(features[a:a + STATS_ROWS])
    return stats


def _model(model, inception_weights) -> fid.InceptionV3:
    if model is None:
        return fid.InceptionV3(weights=inception_weights)
    if not isinstance(model, fid.InceptionV3):
        raise TypeError("model must be a migan_b200.fid.InceptionV3")
    return model


def folder_statistics(path, model: Optional[fid.InceptionV3] = None, batch_size: int = BATCH_SIZE, device="cuda",
                      num_workers: int = 1, inception_weights=None) -> Optional[Tuple[np.ndarray, np.ndarray]]:
    """pytorch_fid's `compute_statistics_of_path`: (mu, sigma) as float64 numpy arrays of an `.npz` or of a directory's
    images.  In an initialised process group rank 0 returns them and the other ranks None."""
    if is_stats_file(path):
        return load_stats(path)
    files = plan_folder(path, num_workers)
    feats = folder_features(files, _model(model, inception_weights), batch_size, device, num_workers).features
    if feats is None:
        return None
    mu, sigma = feature_statistics(feats).mean_cov_device()
    return mu.cpu().numpy(), sigma.cpu().numpy()


class FidScores(NamedTuple):
    """What the command prints: `fid`, and with --kid / --prdc `kid` (a float) and `prdc` (a PRDCResult)."""
    fid: float
    kid: Optional[float] = None
    prdc: Optional[prdc_metric.PRDCResult] = None
    decode_wait_s: float = 0.0
    seconds: float = 0.0


def score_paths(paths: Sequence, batch_size: int = BATCH_SIZE, device="cuda", num_workers: int = 1,
                inception_weights=None, kid: bool = False, prdc: bool = False,
                model: Optional[fid.InceptionV3] = None) -> Optional[FidScores]:
    """The FID of paths[0] against paths[1] (directories or `.npz` files), and the KID and manifold metrics of the second
    folder ("fake") against the first ("real") when asked for.  Every refusal and the planning pass of every folder come
    before any GPU work.  In an initialised process group rank 0 returns the scores and the other ranks None."""
    check_paths(paths, kid=kid, prdc=prdc)
    t0 = time.perf_counter()
    files, problems = [], []
    for p in paths:
        try:
            files.append(None if is_stats_file(p) else plan_folder(p, num_workers))
        except PlanError as e:
            problems += e.problems
    if problems:
        raise PlanError(problems)
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("fid_score runs on CUDA devices only (there is no CPU path); got %s" % device)
    net = _model(model, inception_weights) if any(f is not None for f in files) else None
    feats, wait = [], 0.0
    for f in files:
        got = None if f is None else folder_features(f, net, batch_size, device, num_workers)
        feats.append(None if got is None else got.features)
        wait += 0.0 if got is None else got.decode_wait_s
    if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
        return None
    with torch.cuda.device(device):
        stats = [None if x is None else feature_statistics(x) for x in feats]
        if stats[0] is not None and stats[1] is not None:
            value = stats[0].frechet_distance(stats[1])
        else:
            terms = [load_stats(p) if s is None else s.mean_cov_device() for p, s in zip(paths, stats)]
            value = fid.frechet_distance(*terms[0], *terms[1])
        res = FidScores(float(value))
        if kid:
            res = res._replace(kid=float(kid_metric.kernel_inception_distance(feats[0], feats[1]).kid))
        if prdc:
            res = res._replace(prdc=prdc_metric.precision_recall_density_coverage(feats[0], feats[1], k=E.PRDC_K))
        torch.cuda.synchronize(device)
    return res._replace(decode_wait_s=wait, seconds=time.perf_counter() - t0)


def calculate_fid_given_paths(paths: Sequence, batch_size: int, device, dims: int, num_workers: int = 1) -> float:
    """pytorch_fid's `calculate_fid_given_paths`: the FID of two paths (directories or `.npz` files)."""
    check_dims(dims)
    res = score_paths(paths, batch_size, device, num_workers)
    return None if res is None else res.fid


def save_fid_stats(paths: Sequence, batch_size: int, device, dims: int, num_workers: int = 1,
                   inception_weights=None) -> None:
    """pytorch_fid's `save_fid_stats`: the statistics of directory paths[0] written to paths[1] (on rank 0)."""
    check_dims(dims)
    check_paths(paths, save_stats=True)
    got = folder_statistics(paths[0], None, batch_size, device, num_workers, inception_weights)
    if got is not None:
        save_stats(paths[1], *got)


def check_dims(dims: int) -> None:
    if dims not in DIMS:
        raise ValueError("--dims %r: fid.InceptionV3 builds the 2048-d pool3 block only" % (dims,))


# -- command --------------------------------------------------------------------------------------------------------

def get_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m migan_b200.fid_score")
    parser.add_argument("--batch-size", type=int, default=BATCH_SIZE, help="Batch size to use")
    parser.add_argument("--num-workers", type=int, default=None,
                        help="Number of processes to use for data loading. Defaults to `min(8, num_cpus)`")
    parser.add_argument("--device", type=str, default="cuda", help="Device to use. Like cuda, cuda:0 (CUDA only)")
    parser.add_argument("--dims", type=int, default=2048, choices=list(DIMS),
                        help="Dimensionality of Inception features to use.")
    parser.add_argument("--save-stats", action="store_true",
                        help="Generate an npz archive from a directory of samples. The first path is used as input "
                             "and the second as output.")
    parser.add_argument("--inception-weights", type=Path, default=None, help="FID Inception state_dict file.")
    E.add_kid_arg(parser)
    E.add_prdc_arg(parser)
    parser.add_argument("path", type=str, nargs=2, help="Paths to the generated images or to .npz statistic files")
    return parser.parse_args(argv)


def print_scores(res: Optional[FidScores], kid: bool = False, prdc: bool = False) -> None:
    """`FID:  <value>` as pytorch_fid prints it, then the evaluation command's `KID:` and manifold-metric lines."""
    if res is None:
        return
    print("FID: ", res.fid)
    if kid:
        print("KID: %r" % float(res.kid))
    if prdc:
        for name in ("precision", "recall", "density", "coverage"):
            print("%s: %r" % (name.capitalize(), float(getattr(res.prdc, name))))


def main(argv=None) -> None:
    args = get_args(argv)
    check_paths(args.path, args.save_stats, args.kid, args.prdc)
    workers = default_num_workers() if args.num_workers is None else args.num_workers
    if args.save_stats:
        E.run_command(args.device, lambda device: save_fid_stats(args.path, args.batch_size, device, args.dims, workers,
                                                                 args.inception_weights), "fid_score")
        return
    res = E.run_command(args.device, lambda device: score_paths(
        args.path, args.batch_size, device, workers, args.inception_weights, args.kid, args.prdc), "fid_score")
    print_scores(res, args.kid, args.prdc)


if __name__ == "__main__":
    main()

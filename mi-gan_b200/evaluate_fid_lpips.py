"""scripts/evaluate_fid_lpips.py on the GPU: the same command line and the same two result lines, on one GPU or all the
GPUs of a box, with results that do not depend on how many.

    python -m migan_b200.evaluate_fid_lpips --model-name migan-512 --model-path M.pt --real-dir DIR [--mask-dir MASKS]
    torchrun --nproc_per_node=8 -m migan_b200.evaluate_fid_lpips --model-name migan-512 ...

Differences from the reference script:

* the images are the top-level files of `--real-dir` with a suffix in {.jpg, .jpeg, .JPG, .JPEG, .png, .PNG}, **sorted
  by name** (the script takes `Path.iterdir()`'s order, which is not reproducible).  For a flat directory with lowercase
  suffixes this is the order `generate_masks` uses, so generated masks pair with images as in the files it writes;
* `--batch-size` defaults to 32 (one `EvalPipeline` pass) instead of 8.  It sets the chunk, the unit of work; results
  depend on it at rounding level (the feature sums are grouped by chunk), not on the number of GPUs;
* Co-Mod-GAN draws its noise from seeded streams: image k gets seed `noise_seed * 2**32 + k` (`--noise-seed`, default 0);
* `--real-stats PATH` scores against stored real-image statistics (pytorch_fid's `.npz` with `mu` and `sigma`) and skips
  Inception on the real images; `--save-real-stats PATH` writes them;
* `--inception-weights` and `--lpips-weights` take state_dict files; without them the cached weight files are read, as
  `fid.InceptionV3()` and `lpips.LPIPS()` do.  Nothing is downloaded;
* FID is computed on the GPU (`FeatureStatistics.frechet_distance`), not with scipy's `sqrtm`.  Only CUDA devices run;
* `--ids` also prints Co-Mod-GAN's paired and unpaired Inception discriminative scores (`P-IDS:`, `U-IDS:`) after the two
  lines, from the real and composed features of every image (`ids.inception_discriminative_scores`).  Rank 0 keeps
  those features on the device (16 KiB per image), so `--ids` does not combine with `--real-stats`;
* `--kid` also prints the kernel Inception distance (`KID:`) after all the lines above, from the same kept features:
  `kid.kernel_inception_distance(real, composed)` with 100 subsets of min(n, 1000) images and seed 0, StyleGAN2-ADA's
  unbiased estimator on pytorch_fid's features.  Like `--ids` it does not combine with `--real-stats`;
* `--prdc` also prints `Precision:`, `Recall:`, `Density:` and `Coverage:` after all the lines above (after `KID:`),
  from the same kept features: `prdc.precision_recall_density_coverage(real, composed)` with k = 3, the k-nearest-
  neighbour manifold metrics of StyleGAN2-ADA's `pr50k3` and of Naeem et al. on pytorch_fid's features.  Like `--ids`
  it does not combine with `--real-stats`;
* `--ssim` and `--psnr` also print `SSIM:` and `PSNR:` after the two lines: the means of the per-image
  `metrics.compute_ssim(real, composed, window_size=11, size_average=False)` and `metrics.compute_psnr(composed, real,
  for_dataset=None)` (rgb_range 1, nothing shaved; an image whose composite equals the photo has PSNR inf, and so does
  the mean), the reference's `eva_ssim` / `eva_psnr` on the tensors LPIPS sees;
* `--per-image PATH` writes one CSV row per image in the sorted order: `name` (the photo's path relative to
  `--real-dir`), `hole_fraction` (the share of hole pixels in its R x R mask), `lpips`, then `ssim` and `psnr` when
  asked for, every number as `repr(float)` of the float64 value.  The file is written under a temporary name and moved
  into place;
* `--hole-bins EDGES` (comma-separated, strictly increasing, from 0 to 1, 2 to 33 edges) also prints one `HOLE` line per
  bin of hole fraction h, image i in bin j when e_j <= h_i < e_{j+1} (the last bin also takes h = 1): its image count,
  the FID of its composed images against the real statistics of *all* images (or `--real-stats`), and the means of its
  per-image LPIPS, SSIM and PSNR values, with `--ids` its P-IDS and U-IDS, with `--kid` the KID of its composed
  images against the real images of all images (a fresh RandomState(0) per bin), and with `--prdc` the precision,
  recall, density and coverage of its composed images against the real images of all images (the real radii computed
  once); `nan` where a bin has too few images;
* `--hole-range LO HI` draws the generated masks from RandomMask(R, [LO, HI]) (`RandomMaskStream(R, 0, hole_range)`)
  instead of [0, 1]; it does not combine with `--mask-dir`.

Sharding: the sorted list is cut into chunks of `--batch-size` consecutive images and chunk j runs on rank j % W.  A chunk
is always one `EvalPipeline.forward_batch` call (`ResultsPipeline.forward_batch` when `python -m
migan_b200.score_results` scores result files instead), one LPIPS call and one Inception call on (real, composed), so its
outputs are the same bytes on any rank at any W.  Per round of W chunks every rank sends its chunk's features and LPIPS
values to rank 0 in one fixed-size gather (a rank without a chunk sends padding), and rank 0 adds them to the feature
statistics in chunk order, one `FeatureStatistics.add` per chunk, so the sums see the same rows in the same groups at
every W; with `--ids`, `--kid` or `--prdc` it also keeps them in dataset order, so the scores are the same bits at every W.  The optional
per-image values (hole fraction, SSIM, PSNR) travel as extra columns of the same gather and are kept at their global
index as the LPIPS values are, so their means and the CSV are the same bytes at every W.  Generated
masks come from one sequential stream: every rank advances its own stream through all chunks and
keeps the masks of its own.  With `--hole-bins` the hole fraction travels in the gather too, rank 0 computes each
chunk's bins on the device and adds its composed features to one `BinnedFeatureStatistics` in chunk order, so the bins
see the same rows in the same groups at every W.
"""
from __future__ import annotations

import argparse
import csv
import math
import os
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist

from . import _abi, comodgan, fid, ids, lpips, metrics
from . import kid as kid_metric
from . import prdc as prdc_metric
from ._request_path import load_generator
from .evaluate import EvalPipeline, ResultsPipeline
from .masks import check_hole_range

MODELS = {"migan-256": ("migan", 256), "migan-512": ("migan", 512),
          "comodgan-256": ("comodgan", 256), "comodgan-512": ("comodgan", 512)}
IMG_EXTENSIONS = {".jpg", ".jpeg", ".JPG", ".JPEG", ".png", ".PNG"}
BATCH_SIZE = _abi.PIPE_MAX_BATCH
PREFETCH = 2                    # chunks decoded ahead of the one the GPU works on
MASK_SKIP = 256                 # generated masks skipped per RandomMaskStream.next call
EXTRA_VALUES = ("hole_fraction", "ssim", "psnr")    # optional per-image values, in their gather-column order
PER_IMAGE_COLUMNS = ("name", "hole_fraction", "lpips", "ssim", "psnr")   # the per-image table's column order
FULL_RANGE = (0.0, 1.0)         # RandomMask's default hole_range
PRDC_K = 3                      # the neighbourhood size of --prdc: StyleGAN2-ADA's pr50k3


def resolution(model_name: str) -> int:
    if model_name not in MODELS:
        raise Exception("Unsupported model name.")
    return MODELS[model_name][1]


# -- dataset --------------------------------------------------------------------------------------------------------

def list_images(real_dir) -> List[Path]:
    """The top-level image files of `real_dir` (InferenceDataset's suffixes), sorted by name."""
    return sorted((p for p in Path(real_dir).iterdir() if p.suffix in IMG_EXTENSIONS and p.is_file()),
                  key=lambda p: p.name)


def stem_pngs(images: Sequence[Path], directory) -> List[Path]:
    """`<directory>/<stem>.png` of every image (a.b.jpg -> a.b.png), whether it exists or not."""
    return [Path(directory) / ("%s.png" % p.stem) for p in images]


def list_masks(images: Sequence[Path], mask_dir) -> List[Path]:
    """`<mask_dir>/<stem>.png` of every image; FileNotFoundError names the first that is missing."""
    masks = stem_pngs(images, mask_dir)
    for m, p in zip(masks, images):
        if not m.is_file():
            raise FileNotFoundError("no mask %s for image %s" % (m, p.name))
    return masks


def decode_photo(path) -> np.ndarray:
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im.convert("RGB"))


def decode_mask(path) -> np.ndarray:
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im.convert("L"))


# -- chunks ---------------------------------------------------------------------------------------------------------

def chunk_bounds(n: int, batch_size: int) -> List[Tuple[int, int]]:
    """[start, end) of each chunk: `batch_size` consecutive images, the last one possibly short."""
    if n < 0 or batch_size < 1:
        raise ValueError("bad chunking (%d images, batch size %d)" % (n, batch_size))
    return [(a, min(a + batch_size, n)) for a in range(0, n, batch_size)]


def num_rounds(n_chunks: int, world_size: int) -> int:
    """Rounds every rank joins: round r holds chunks r*W ... r*W + W - 1."""
    return -(-n_chunks // world_size)


def round_chunk(r: int, rank: int, n_chunks: int, world_size: int) -> Optional[int]:
    """The chunk rank `rank` runs in round r (chunk j runs on rank j % W), or None when it has none left."""
    j = r * world_size + rank
    return j if j < n_chunks else None


# -- per-rank work --------------------------------------------------------------------------------------------------

class ChunkResult(NamedTuple):
    """What a chunk sends to rank 0: float32 features [c, 2048] (`real` None when the real statistics are loaded from a
    file), LPIPS values [c] and, when the setup asks for any, the extra per-image values [c, len(extra_values)] in
    `EvalSetup.extra_values` order."""
    index: int
    start: int
    real: Optional[torch.Tensor]
    fake: torch.Tensor
    lpips: torch.Tensor
    extra: Optional[torch.Tensor] = None


class EvalSetup:
    """What every rank of one evaluation shares: the file lists, the chunking and the networks, on `device`.

    The composite's fill-in comes from one of two sources.  A generator: `model_name` and `model`.  Or a method's result
    files: `results`, the result file of each image of `list_images(real_dir)` in that order, with `model_name` and
    `model` None and `res` the resolution R (`score_results` plans and checks these lists).

    `ssim` / `psnr`: every chunk also computes each image's SSIM / PSNR; `per_image`: each image's hole fraction too, and
    rank 0's result keeps the per-image table (`EvalResult.per_image`).  `hole_bins`: the edges of the hole-fraction
    bins rank 0 scores (`EvalResult.by_hole`; the hole fraction is then computed too); `hole_range`: RandomMask's
    hole_range for the generated masks."""

    def __init__(self, model_name: Optional[str], model, real_dir, mask_dir=None, *, device="cuda",
                 batch_size: int = BATCH_SIZE, num_workers: int = 2, noise_seed: int = 0, real_features: bool = True,
                 inception_weights=None, lpips_weights=None, results: Optional[Sequence] = None,
                 res: Optional[int] = None, ssim: bool = False, psnr: bool = False, per_image: bool = False,
                 hole_bins: Optional[Sequence[float]] = None, hole_range: Sequence[float] = FULL_RANGE):
        self.hole_bins, self.hole_range = check_hole_args(hole_bins, hole_range, mask_dir)
        if results is None:
            self.res = resolution(model_name)
        elif model_name is not None or model is not None or res is None:
            raise ValueError("EvalSetup: result files take the place of the generator: pass model_name=None, "
                             "model=None and res=R")
        else:
            self.res = int(res)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("evaluate_fid_lpips runs on a CUDA device (there is no CPU path); got %s" % self.device)
        if batch_size < 1:
            raise ValueError("--batch-size must be >= 1, got %d" % batch_size)
        self.real_dir = Path(real_dir)
        self.images = list_images(real_dir)
        if len(self.images) < 2:
            raise ValueError("%s holds %d images; FID needs at least 2" % (real_dir, len(self.images)))
        self.results = None if results is None else [Path(r) for r in results]
        if self.results is not None and len(self.results) != len(self.images):
            raise ValueError("EvalSetup: %d result files for %d images" % (len(self.results), len(self.images)))
        self.masks = None if mask_dir is None else list_masks(self.images, mask_dir)
        self.chunks = chunk_bounds(len(self.images), int(batch_size))
        self.num_workers = max(1, int(num_workers))
        self.noise_seed = int(noise_seed)
        self.real_features = bool(real_features)
        self.per_image = bool(per_image)
        holes = per_image or self.hole_bins is not None
        self.extra_values = tuple(v for v, on in zip(EXTRA_VALUES, (holes, ssim, psnr)) if on)
        if self.results is not None:
            self.model = None
        elif MODELS[model_name][0] == "comodgan":
            self.model = comodgan.load(model, self.res).to(self.device)
        else:
            self.model = load_generator(self, model, self.res, self.device)
        self.inception = fid.InceptionV3(weights=inception_weights)
        self.lpips = lpips.LPIPS(net="alex", weights=lpips_weights).to(self.device)

    @property
    def feature_width(self) -> int:
        """Floats per image in a round's gather buffer: the features, the LPIPS value, then the extra values."""
        return (2 if self.real_features else 1) * fid.FEATURES + 1 + len(self.extra_values)

    @property
    def names(self) -> List[str]:
        """Each image's path relative to `real_dir`, with POSIX separators, in the sorted order."""
        return [p.relative_to(self.real_dir).as_posix() for p in self.images]


class RankWorker:
    """Rank `rank` of `world_size`: its own `EvalPipeline`, or `ResultsPipeline` for result files (and the pipeline's
    mask stream), and its host decode pool.  `run_round(r)`
    runs this rank's chunk of round r; call it for r = 0, 1, ... in order.  Usable as a context manager (`close()` stops
    the decode threads)."""

    def __init__(self, setup: EvalSetup, rank: int, world_size: int):
        if world_size < 1 or not 0 <= rank < world_size:
            raise ValueError("bad rank %d of %d" % (rank, world_size))
        self.setup, self.rank, self.world_size = setup, rank, world_size
        if setup.results is None:
            self.pipe = EvalPipeline(setup.model, setup.res, device=setup.device, seed=0, noise_seed=setup.noise_seed,
                                     hole_range=setup.hole_range)
        else:
            self.pipe = ResultsPipeline(setup.res, device=setup.device, seed=0, hole_range=setup.hole_range)
        self.rounds = num_rounds(len(setup.chunks), world_size)
        self.own = [j for j in range(rank, len(setup.chunks), world_size)]
        self._pool = ThreadPoolExecutor(max_workers=setup.num_workers)
        self._pending = deque()          # (chunk, [futures]) decoding ahead, in chunk order
        self._next = 0                   # index into self.own of the next chunk to submit for decoding
        self._mask_pos = 0               # images whose generated masks this rank's stream has passed
        self.decode_wait_s = 0.0         # host time spent waiting for decoded chunks

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self) -> None:
        for _, futs in self._pending:
            for f in futs:
                f.cancel()
        self._pending.clear()
        self._pool.shutdown(wait=True)

    def _submit(self) -> None:
        while len(self._pending) < PREFETCH and self._next < len(self.own):
            j = self.own[self._next]
            self._next += 1
            a, b = self.setup.chunks[j]
            futs = [self._pool.submit(decode_photo, p) for p in self.setup.images[a:b]]
            if self.setup.results is not None:
                futs += [self._pool.submit(decode_photo, p) for p in self.setup.results[a:b]]
            if self.setup.masks is not None:
                futs += [self._pool.submit(decode_mask, p) for p in self.setup.masks[a:b]]
            self._pending.append((j, futs))

    def _decoded(self, j: int):
        self._submit()
        got, futs = self._pending.popleft()
        assert got == j, "chunks must be run in round order"
        t = time.perf_counter()
        arrays = [f.result() for f in futs]
        self.decode_wait_s += time.perf_counter() - t
        self._submit()                   # keep PREFETCH chunks decoding while the GPU works
        a, b = self.setup.chunks[j]
        c = b - a
        photos = arrays[:c]
        results = None if self.setup.results is None else arrays[c:2 * c]
        masks = None if self.setup.masks is None else arrays[-c:]
        return photos, results, masks

    def _skip_masks(self, upto: int) -> None:
        """Advance the generated-mask stream to image `upto`: the masks of other ranks' chunks are drawn and dropped."""
        while self._mask_pos < upto:
            k = min(MASK_SKIP, upto - self._mask_pos)
            self.pipe.masks.next(k)
            self._mask_pos += k

    @torch.no_grad()
    def run_chunk(self, j: int) -> ChunkResult:
        setup = self.setup
        a, b = setup.chunks[j]
        photos, results, masks = self._decoded(j)
        if masks is None:
            self._skip_masks(a)
            self._mask_pos = b
        holes = "hole_fraction" in setup.extra_values
        if results is None:
            self.pipe.noise_index = a
            got = self.pipe.forward_batch(photos, masks, hole_fraction=holes)
        else:
            got = self.pipe.forward_batch(photos, results, masks, hole_fraction=holes)
        real, composed = got[0], got[1]
        values = setup.lpips(real, composed, normalize=True).view(-1)
        extra = [got[2]] if holes else []
        if "ssim" in setup.extra_values:
            extra.append(metrics.compute_ssim(real, composed, window_size=11, size_average=False))
        if "psnr" in setup.extra_values:
            extra.append(metrics.compute_psnr(composed, real, for_dataset=None))
        extra = torch.stack(extra, 1) if extra else None
        c = b - a
        if setup.real_features:
            feats = setup.inception(torch.cat([real, composed]))[0].view(2 * c, fid.FEATURES)
            return ChunkResult(j, a, feats[:c], feats[c:], values, extra)
        return ChunkResult(j, a, None, setup.inception(composed)[0].view(c, fid.FEATURES), values, extra)

    def run_round(self, r: int) -> Optional[ChunkResult]:
        j = round_chunk(r, self.rank, len(self.setup.chunks), self.world_size)
        return None if j is None else self.run_chunk(j)


# -- transport and merge --------------------------------------------------------------------------------------------

def gather_round(result: Optional[ChunkResult], r: int, chunks: Sequence[Tuple[int, int]], width: int, device,
                 group=None, extra: int = 0, lpips: bool = True) -> List[ChunkResult]:
    """One round's chunk results on rank 0, in chunk order ([] on the other ranks).  Every rank of `group` calls it
    once per round, with its chunk's result or None: it sends one [batch, width] float32 buffer (features, the LPIPS
    value, then `extra` per-image values; zero rows pad a short or absent chunk) in one gather.  `width` is
    2 * 2048 + 1 + extra, or 2048 + 1 + extra without real features.  With `lpips` False the chunks carry features
    alone (`lpips` None) and there is no LPIPS column: `width` is then 2048 (+ extra), as `fid_score` sends."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    batch = chunks[0][1] - chunks[0][0]
    F = fid.FEATURES
    nl = 1 if lpips else 0
    lpips_at = width - nl - extra                         # the LPIPS column, when sent; the extra values follow it
    fake_at = lpips_at - F                                # real features, when sent, occupy [0, F)
    buf = torch.zeros((batch, width), dtype=torch.float32, device=device)
    if result is not None:
        c = result.fake.shape[0]
        if fake_at:
            buf[:c, :F] = result.real
        buf[:c, fake_at:lpips_at] = result.fake
        if lpips:
            buf[:c, lpips_at] = result.lpips
        if extra:
            buf[:c, lpips_at + nl:] = result.extra
    bufs = [torch.empty_like(buf) for _ in range(world)] if rank == 0 else None
    dist.gather(buf, bufs, dst=0, group=group)
    if rank != 0:
        return []
    out = []
    for k, got in enumerate(bufs):
        j = round_chunk(r, k, len(chunks), world)
        if j is not None:
            a, b = chunks[j]
            c = b - a
            out.append(ChunkResult(j, a, got[:c, :F] if fake_at else None, got[:c, fake_at:lpips_at],
                                   got[:c, lpips_at] if lpips else None, got[:c, lpips_at + nl:] if extra else None))
    return out


class _EvalFields(NamedTuple):
    fid: float
    lpips: float                      # np.mean of lpips_values, the script's reduction
    lpips_values: np.ndarray          # float64 [count], dataset (sorted) order
    count: int
    decode_wait_s: float = 0.0        # rank 0's host time waiting for decoded chunks
    seconds: float = 0.0              # rank 0's wall time of the chunk loop and the distance
    p_ids: Optional[float] = None     # with ids=True: the paired and unpaired Inception discriminative scores
    u_ids: Optional[float] = None


class HoleBin(NamedTuple):
    """The scores of the images whose hole fraction h lies in [lo, hi) ([lo, hi] for the last bin).  `fid`: the bin's
    composed images against the real statistics of all images; `lpips`, `ssim`, `psnr`: np.mean of the bin's per-image
    values; `kid`: the KID of the bin's composed features against the real features of all images; `precision`,
    `recall`, `density`, `coverage`: those of the bin's composed features against the real features of all images
    (k = 3).  nan where the bin has too few images (2 for FID, the discriminative scores and KID, k + 1 = 4 for the
    four manifold metrics, 1 for the means); None where the value was not asked for."""
    lo: float
    hi: float
    count: int
    fid: float
    lpips: float
    ssim: Optional[float] = None
    psnr: Optional[float] = None
    p_ids: Optional[float] = None
    u_ids: Optional[float] = None
    kid: Optional[float] = None
    precision: Optional[float] = None
    recall: Optional[float] = None
    density: Optional[float] = None
    coverage: Optional[float] = None


class EvalResult(_EvalFields):
    """The evaluation's result: a tuple of the eight fields above.  The attributes below are kept outside the tuple, so
    its length, unpacking and equality stay those of the fields; each is None unless asked for.

    * `ssim` / `psnr`: `np.mean` of the per-image SSIM / PSNR values (inf when an image's PSNR is inf);
    * `per_image`: {column: values} in `PER_IMAGE_COLUMNS` order: "name" (list of str), then float64 [count] arrays
      "hole_fraction", "lpips" and, when computed, "ssim" and "psnr", all in dataset (sorted) order;
    * `by_hole`: with hole bins, one `HoleBin` per bin in edge order;
    * `kid`: the kernel Inception distance of the composed features against the real ones (`kid_metric.KIDResult.kid`);
    * `prdc`: precision, recall, density and coverage of the composed features against the real ones, k = 3
      (`prdc_metric.PRDCResult`)."""
    ssim: Optional[float] = None
    psnr: Optional[float] = None
    per_image: Optional[Dict[str, Union[List[str], np.ndarray]]] = None
    by_hole: Optional[Tuple[HoleBin, ...]] = None
    kid: Optional[float] = None
    prdc: Optional[prdc_metric.PRDCResult] = None

    def _replace(self, **fields) -> "EvalResult":
        out = super()._replace(**fields)
        out.__dict__.update(self.__dict__)
        return out


class Merge:
    """Rank 0's ordered merge: `add` the chunk results in chunk order, then `result()`.  With `keep_features` it also
    keeps every real and composed feature row in dataset order on the device, for the discriminative scores; with `kid`
    it keeps them too, for the kernel Inception distance, and with `prdc` for precision, recall, density and coverage
    (the real radii computed once for the overall value and every bin).
    `extra_values`: the names of the chunks' extra per-image values (`EvalSetup.extra_values`), kept at their global
    index as the LPIPS values are; `names`: each image's name, for the per-image table of the result; `hole_bins`: the
    edges of the hole-fraction bins (the extra values then hold "hole_fraction"): each chunk's composed features also
    go to one `BinnedFeatureStatistics` by their bins, computed on the device."""

    def __init__(self, n: int, device, real_features: bool = True, keep_features: bool = False,
                 extra_values: Sequence[str] = (), names: Optional[Sequence[str]] = None,
                 hole_bins: Optional[Sequence[float]] = None, kid: bool = False, prdc: bool = False):
        self.n, self.device = n, torch.device(device)
        self.real = fid.FeatureStatistics(device=self.device) if real_features else None
        self.fake = fid.FeatureStatistics(device=self.device)
        if (keep_features or kid or prdc) and not real_features:
            raise ValueError("the discriminative scores, KID and the manifold metrics need the real features")
        self.ids, self.kid, self.prdc = bool(keep_features), bool(kid), bool(prdc)
        self.kept = None
        if keep_features or kid or prdc:
            self.kept = [torch.empty((n, fid.FEATURES), dtype=torch.float32, device=self.device) for _ in range(2)]
        self.values = torch.empty(n, dtype=torch.float32, device=self.device)
        self.extra_values = tuple(extra_values)
        if any(v not in EXTRA_VALUES for v in self.extra_values):
            raise ValueError("extra per-image values are among %s; got %s" % (EXTRA_VALUES, self.extra_values))
        self.extra = None
        if self.extra_values:
            self.extra = torch.empty((n, len(self.extra_values)), dtype=torch.float32, device=self.device)
        if names is not None and len(names) != n:
            raise ValueError("%d names for %d images" % (len(names), n))
        self.names = None if names is None else list(names)
        self.hole_bins = self.binned = None
        if hole_bins is not None:
            if "hole_fraction" not in self.extra_values:
                raise ValueError("hole bins need the hole fraction among the extra per-image values")
            self.hole_bins = tuple(float(e) for e in hole_bins)
            self.inner_edges = torch.tensor(self.hole_bins[1:-1], dtype=torch.float64, device=self.device)
            self.binned = fid.BinnedFeatureStatistics(len(self.hole_bins) - 1, device=self.device)
        self.next_chunk = 0
        self.count = 0

    def add(self, chunk: ChunkResult) -> None:
        if chunk.index != self.next_chunk:
            raise RuntimeError("chunk %d merged before chunk %d" % (chunk.index, self.next_chunk))
        c = chunk.fake.shape[0]
        if self.real is not None:
            self.real.add(chunk.real)
        self.fake.add(chunk.fake)
        if self.binned is not None:
            hole = chunk.extra[:, self.extra_values.index("hole_fraction")].to(self.device)
            self.binned.add(chunk.fake, hole_bin_index(hole, self.inner_edges))
        self.values[chunk.start:chunk.start + c] = chunk.lpips.to(self.device)
        if self.extra is not None:
            self.extra[chunk.start:chunk.start + c] = chunk.extra.to(self.device)
        if self.kept is not None:
            self.kept[0][chunk.start:chunk.start + c] = chunk.real
            self.kept[1][chunk.start:chunk.start + c] = chunk.fake
        self.next_chunk += 1
        self.count += c

    def real_statistics(self) -> Tuple[np.ndarray, np.ndarray]:
        """(mu, sigma) of the real features as float64 numpy arrays, from `mean_cov_device()`."""
        mu, sigma = self.real.mean_cov_device()
        return mu.cpu().numpy(), sigma.cpu().numpy()

    def result(self, real_stats=None) -> EvalResult:
        """The FID against the merged real statistics, or against `real_stats` = (mu, sigma) when given."""
        if self.count != self.n:
            raise RuntimeError("merged %d of %d images" % (self.count, self.n))
        if real_stats is None:
            value = self.real.frechet_distance(self.fake)
        else:
            value = fid.frechet_distance(real_stats[0], real_stats[1], *self.fake.mean_cov_device())
        values = self.values.cpu().numpy().astype(np.float64)
        res = EvalResult(float(value), float(np.mean(values)), values, self.n)
        if self.ids:
            scores = ids.inception_discriminative_scores(*self.kept)
            res = res._replace(p_ids=scores.p_ids, u_ids=scores.u_ids)
        if self.kid:
            res.kid = kid_metric.kernel_inception_distance(*self.kept).kid
        radii = None
        if self.prdc:
            radii = prdc_metric.RealRadii(self.kept[0], PRDC_K, max_fake=self.n)
            res.prdc = prdc_metric.precision_recall_density_coverage(radii, self.kept[1])
        columns = {"lpips": values}
        if self.extra is not None:
            extra = self.extra.cpu().numpy().astype(np.float64)
            columns.update((v, extra[:, k]) for k, v in enumerate(self.extra_values))
        if "ssim" in columns:
            res.ssim = float(np.mean(columns["ssim"]))
        if "psnr" in columns:
            res.psnr = float(np.mean(columns["psnr"]))
        if self.names is not None:
            columns["name"] = self.names
            res.per_image = {k: columns[k] for k in PER_IMAGE_COLUMNS if k in columns}
        if self.binned is not None:
            res.by_hole = self.hole_results(columns, real_stats, radii)
        return res

    def hole_results(self, columns, real_stats=None, radii=None) -> Tuple[HoleBin, ...]:
        """One `HoleBin` per bin: the bins of the merged hole fractions, the binned composed statistics against the
        real ones of all images (or `real_stats`), and the per-image columns' means over each bin; with `radii`
        (`prdc_metric.RealRadii` of all real features) each bin's composed features against them."""
        bins = hole_bin_index(torch.from_numpy(columns["hole_fraction"]), self.inner_edges.cpu()).numpy()
        counts = self.binned.counts()
        want = np.bincount(bins, minlength=len(counts))
        if not np.array_equal(counts, want):
            raise RuntimeError("binned feature counts %s differ from the hole fractions' %s" % (counts, want))
        real = real_stats if real_stats is not None else self.real.mean_cov_device()
        out = []
        for b, (lo, hi) in enumerate(zip(self.hole_bins[:-1], self.hole_bins[1:])):
            idx = np.flatnonzero(bins == b)
            n = len(idx)
            fid_b = fid.frechet_distance(*real, *self.binned.mean_cov_device(b, n)) if n >= 2 else math.nan
            means = {k: float(np.mean(columns[k][idx])) if n else math.nan for k in ("lpips", "ssim", "psnr")
                     if k in columns}
            p_ids = u_ids = kid = None
            at = torch.from_numpy(idx).to(self.device) if n >= 2 and self.kept is not None else None
            if self.ids:
                p_ids = u_ids = math.nan
                if at is not None:
                    scores = ids.inception_discriminative_scores(self.kept[0][at], self.kept[1][at])
                    p_ids, u_ids = scores.p_ids, scores.u_ids
            if self.kid:
                kid = math.nan
                if at is not None:
                    kid = kid_metric.kernel_inception_distance(self.kept[0], self.kept[1][at]).kid
            manifold = (None,) * 4
            if self.prdc:
                manifold = (math.nan,) * 4
                if n > PRDC_K:
                    manifold = tuple(prdc_metric.precision_recall_density_coverage(radii, self.kept[1][at])[:4])
            out.append(HoleBin(lo, hi, n, float(fid_b), means["lpips"], means.get("ssim"), means.get("psnr"), p_ids,
                               u_ids, kid, *manifold))
        return tuple(out)


def hole_bin_index(hole: torch.Tensor, inner_edges: torch.Tensor) -> torch.Tensor:
    """int32 bin of each hole fraction (float32, compared as float64) among the bins of edges 0, *inner_edges, 1: bin j
    when e_j <= h < e_{j+1}, and the last bin also takes h = 1.  On the tensors' device."""
    return torch.searchsorted(inner_edges, hole.to(torch.float64).contiguous(), right=True).to(torch.int32)


def parse_hole_bins(text: str) -> Tuple[float, ...]:
    """--hole-bins EDGES: comma-separated edges, checked as `check_hole_bins` does."""
    try:
        edges = [float(v) for v in text.split(",")]
    except ValueError:
        raise ValueError("--hole-bins %r: a comma-separated list of numbers, e.g. 0,0.2,0.4,1" % text) from None
    return check_hole_bins(edges)


def check_hole_bins(edges: Sequence[float]) -> Tuple[float, ...]:
    """2 to 33 finite, strictly increasing edges from 0 to 1 (1 to 32 bins)."""
    edges = tuple(float(e) for e in edges)
    if not 2 <= len(edges) <= fid.MAX_BINS + 1:
        raise ValueError("--hole-bins: %d edges (2 to %d: 1 to %d bins)" % (len(edges), fid.MAX_BINS + 1, fid.MAX_BINS))
    if edges[0] != 0.0 or edges[-1] != 1.0 or not all(math.isfinite(e) for e in edges):
        raise ValueError("--hole-bins %s: the edges run from 0 to 1" % ",".join(map(repr, edges)))
    if any(b <= a for a, b in zip(edges, edges[1:])):
        raise ValueError("--hole-bins %s: the edges must increase strictly" % ",".join(map(repr, edges)))
    return edges


def check_hole_args(hole_bins, hole_range, mask_dir) -> Tuple[Optional[Tuple[float, ...]], Tuple[float, float]]:
    """The refusals of --hole-bins and --hole-range, before any work: (edges or None, (lo, hi))."""
    edges = None if hole_bins is None else check_hole_bins(hole_bins)
    lo_hi = check_hole_range(hole_range, "--hole-range")
    if lo_hi != FULL_RANGE and mask_dir is not None:
        raise ValueError("--hole-range draws the generated masks; it does not combine with --mask-dir")
    return edges, lo_hi


def write_per_image(path, per_image) -> None:
    """`per_image` (`EvalResult.per_image`) as a CSV file at `path`: a header of its columns, then one row per image,
    each number as `repr(float)` (so inf is written `inf`).  It is written to a temporary name in the same directory
    and moved into place with `os.replace`, so `path` never holds a partial table."""
    path = Path(path)
    columns = list(per_image)
    tmp = path.with_name(".%s.%d.tmp" % (path.name, os.getpid()))
    try:
        with open(tmp, "w", newline="", encoding="utf-8") as f:
            w = csv.writer(f, lineterminator="\n")
            w.writerow(columns)
            for i, name in enumerate(per_image["name"]):
                w.writerow([name] + [repr(float(per_image[k][i])) for k in columns[1:]])
        os.replace(tmp, path)
    except BaseException:
        tmp.unlink(missing_ok=True)
        raise


def load_real_stats(path) -> Tuple[np.ndarray, np.ndarray]:
    with np.load(path) as f:
        return np.asarray(f["mu"], dtype=np.float64), np.asarray(f["sigma"], dtype=np.float64)


def save_real_stats(path, mu: np.ndarray, sigma: np.ndarray) -> None:
    """pytorch_fid's layout: an .npz with `mu` and `sigma`, written to `path` as given."""
    with open(path, "wb") as f:
        np.savez(f, mu=mu, sigma=sigma)


# -- entry points ---------------------------------------------------------------------------------------------------

def evaluate(model_name: str, model, real_dir, mask_dir=None, *, device="cuda", batch_size: int = BATCH_SIZE,
             num_workers: int = 2, noise_seed: int = 0, real_stats=None, save_real_stats_to=None,
             inception_weights=None, lpips_weights=None, ids: bool = False, ssim: bool = False, psnr: bool = False,
             per_image: bool = False, hole_bins: Optional[Sequence[float]] = None,
             hole_range: Sequence[float] = FULL_RANGE, kid: bool = False, prdc: bool = False) -> Optional[EvalResult]:
    """FID and LPIPS of `model` over `real_dir`, as the command prints them.  `model`: a state_dict, a path to one, or a
    generator object (MI-GAN `Generator`, or `comodgan.Generator` for the comodgan names).  `real_stats`: a path to an
    .npz with `mu` and `sigma` (or such a pair); `save_real_stats_to`: where to write the real statistics.
    `inception_weights` / `lpips_weights`: state_dicts or paths instead of the cached weight files.  `ids`: also the
    paired and unpaired Inception discriminative scores (`p_ids`, `u_ids`); it needs the real features, so it excludes
    `real_stats`.  `ssim` / `psnr`: also the mean SSIM / PSNR (`EvalResult.ssim` / `.psnr`); `per_image`: also the
    per-image table (`EvalResult.per_image`).  `hole_bins`: the edges of hole-fraction bins, scored one by one
    (`EvalResult.by_hole`); `hole_range`: RandomMask's hole_range for the generated masks (not with `mask_dir`).
    `kid`: also the kernel Inception distance (`EvalResult.kid`, and per bin); like `ids` it excludes `real_stats`.
    `prdc`: also precision, recall, density and coverage (`EvalResult.prdc`, and per bin); it excludes `real_stats` too.

    In an initialised process group (one process per GPU, `device` this rank's), the chunks are sharded round-robin and
    rank 0 returns the result; the other ranks return None."""
    check_stats_args(real_stats, save_real_stats_to, ids, kid, prdc)
    check_hole_args(hole_bins, hole_range, mask_dir)
    if real_stats is not None and not isinstance(real_stats, tuple):
        real_stats = load_real_stats(real_stats)
    setup = EvalSetup(model_name, model, real_dir, mask_dir, device=device, batch_size=batch_size,
                      num_workers=num_workers, noise_seed=noise_seed, real_features=real_stats is None,
                      inception_weights=inception_weights, lpips_weights=lpips_weights, ssim=ssim, psnr=psnr,
                      per_image=per_image, hole_bins=hole_bins, hole_range=hole_range)
    return run_setup(setup, real_stats, save_real_stats_to, ids, kid, prdc)


def check_stats_args(real_stats, save_real_stats_to, ids: bool, kid: bool = False, prdc: bool = False) -> None:
    """The refusals of --real-stats, --save-real-stats, --ids, --kid and --prdc, before any work."""
    if real_stats is not None and save_real_stats_to is not None:
        raise ValueError("--real-stats and --save-real-stats exclude each other: with stored statistics the real images "
                         "are not scored")
    if ids and real_stats is not None:
        raise ValueError("--ids needs the real images' features, which stored statistics (--real-stats) do not carry")
    if kid and real_stats is not None:
        raise ValueError("--kid needs the real images' features, which stored statistics (--real-stats) do not carry")
    if prdc and real_stats is not None:
        raise ValueError("--prdc needs the real images' features, which stored statistics (--real-stats) do not carry")


def run_setup(setup: EvalSetup, real_stats=None, save_real_stats_to=None, ids: bool = False,
              kid: bool = False, prdc: bool = False) -> Optional[EvalResult]:
    """Every round of `setup`'s chunks on this rank, merged on rank 0 in chunk order (see `evaluate`); `real_stats`: a
    loaded (mu, sigma) pair or None.  The setup's `ssim`, `psnr` and `per_image` choices fill the result's attributes of
    those names; `kid` fills `EvalResult.kid` (and each bin's), `prdc` fills `EvalResult.prdc` (and each bin's four)."""
    distributed = dist.is_available() and dist.is_initialized()
    world, rank = (dist.get_world_size(), dist.get_rank()) if distributed else (1, 0)
    merge = None
    if rank == 0:
        merge = Merge(len(setup.images), setup.device, setup.real_features, keep_features=ids,
                      extra_values=setup.extra_values, names=setup.names if setup.per_image else None,
                      hole_bins=setup.hole_bins, kid=kid, prdc=prdc)
    t0 = time.perf_counter()
    with torch.cuda.device(setup.device), RankWorker(setup, rank, world) as worker:
        for r in range(worker.rounds):
            got = worker.run_round(r)
            if distributed:
                got = gather_round(got, r, setup.chunks, setup.feature_width, setup.device,
                                   extra=len(setup.extra_values))
            else:
                got = [got]
            for chunk in got:
                merge.add(chunk)
        if merge is None:
            return None
        if save_real_stats_to is not None:
            save_real_stats(save_real_stats_to, *merge.real_statistics())
        res = merge.result(real_stats)
        torch.cuda.synchronize(setup.device)
    return res._replace(decode_wait_s=worker.decode_wait_s, seconds=time.perf_counter() - t0)


def get_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m migan_b200.evaluate_fid_lpips")
    parser.add_argument("--model-name", type=str, help="One of [migan-256, migan-512, comodgan-256, comodgan-512]")
    parser.add_argument("--model-path", type=Path, help="Saved model path.", required=True)
    parser.add_argument("--real-dir", type=Path, help="Real dataset directory path.", required=True)
    parser.add_argument("--mask-dir", type=Path, help="Pre-generated mask directory path.", required=False)
    parser.add_argument("--device", type=str, help="Device to use (CUDA only).", required=False, default="cuda")
    parser.add_argument("--batch-size", type=int, help="Images per chunk (the unit of work).", required=False,
                        default=BATCH_SIZE)
    parser.add_argument("--num-workers", type=int, help="Host decode threads.", required=False, default=2)
    parser.add_argument("--noise-seed", type=int, default=0, help="Co-Mod-GAN: image k gets noise seed "
                        "noise_seed * 2**32 + k.")
    parser.add_argument("--save-real-stats", type=Path, default=None, help="Write the real images' mu and sigma (.npz).")
    parser.add_argument("--real-stats", type=Path, default=None, help="Score against stored real mu and sigma (.npz).")
    parser.add_argument("--inception-weights", type=Path, default=None, help="FID Inception state_dict file.")
    parser.add_argument("--lpips-weights", type=Path, default=None, help="LPIPS (alex) state_dict file.")
    parser.add_argument("--ids", action="store_true", help="Also print P-IDS and U-IDS (Co-Mod-GAN's Inception "
                        "discriminative scores).")
    add_kid_arg(parser)
    add_prdc_arg(parser)
    add_per_image_args(parser)
    return parser.parse_args(argv)


def add_kid_arg(parser: argparse.ArgumentParser) -> None:
    """--kid, shared with score_results."""
    parser.add_argument("--kid", action="store_true", help="Also print the kernel Inception distance (KID: 100 subsets "
                        "of min(n, 1000) images, seed 0).")


def add_prdc_arg(parser: argparse.ArgumentParser) -> None:
    """--prdc, shared with score_results."""
    parser.add_argument("--prdc", action="store_true", help="Also print precision, recall, density and coverage "
                        "(k-nearest-neighbour manifold metrics, k = 3).")


def add_per_image_args(parser: argparse.ArgumentParser) -> None:
    """--ssim, --psnr, --per-image, --hole-bins and --hole-range, shared with score_results."""
    parser.add_argument("--ssim", action="store_true", help="Also print the mean SSIM (window 11).")
    parser.add_argument("--psnr", action="store_true", help="Also print the mean PSNR (rgb_range 1, nothing shaved).")
    parser.add_argument("--per-image", type=Path, default=None, metavar="PATH",
                        help="Write one CSV row per image: name, hole_fraction, lpips[, ssim][, psnr].")
    parser.add_argument("--hole-bins", type=str, default=None, metavar="EDGES",
                        help="Also print the scores per bin of hole fraction, e.g. 0,0.1,0.2,0.3,0.4,0.5,0.6,1.")
    parser.add_argument("--hole-range", type=float, nargs=2, default=None, metavar=("LO", "HI"),
                        help="Draw the generated masks from RandomMask(R, [LO, HI]) (not with --mask-dir).")


def check_hole_flags(args) -> Tuple[Optional[Tuple[float, ...]], Tuple[float, float]]:
    """--hole-bins and --hole-range of a parsed command line, checked before any work: (edges or None, (lo, hi))."""
    if args.hole_range is not None and args.mask_dir is not None:
        raise ValueError("--hole-range draws the generated masks; it does not combine with --mask-dir")
    edges = None if args.hole_bins is None else parse_hole_bins(args.hole_bins)
    return check_hole_args(edges, FULL_RANGE if args.hole_range is None else args.hole_range, args.mask_dir)


def check_per_image_path(path) -> None:
    """Refuse a --per-image file whose directory does not exist, before any work."""
    if path is not None and not Path(path).parent.is_dir():
        raise ValueError("--per-image %s: the directory %s does not exist" % (path, Path(path).parent))


def device_for(requested: str, world_size: int, local_rank: int, command: str = "evaluate_fid_lpips") -> torch.device:
    """The CUDA device of this process: `requested` alone, `cuda:LOCAL_RANK` under torchrun."""
    dev = torch.device(requested)
    if dev.type != "cuda":
        raise RuntimeError("%s runs on CUDA devices only (there is no CPU path); got --device %s" % (command, requested))
    if world_size > 1:
        if dev.index is not None:
            raise ValueError("--device %s: with several processes each one uses cuda:LOCAL_RANK; pass --device cuda"
                             % requested)
        return torch.device("cuda", local_rank)
    return dev


def run_command(requested_device: str, call, command: str = "evaluate_fid_lpips") -> Optional[EvalResult]:
    """`call(device)` in this process: alone, or under torchrun (WORLD_SIZE > 1) as one rank of an NCCL process group
    that lives for the call."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = device_for(requested_device, world, local_rank, command)
    if world > 1:
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=device)
    try:
        return call(device)
    finally:
        if world > 1:
            dist.destroy_process_group()


def hole_line(b: HoleBin, last: bool) -> str:
    """`HOLE [lo, hi): images n FID f LPIPS l[ SSIM s][ PSNR p][ P-IDS a U-IDS u][ KID k][ Precision p Recall r
    Density d Coverage c]`, every number repr(float); the last bin is closed, `[lo, 1.0]`."""
    line = "HOLE [%r, %r%s: images %d FID %r LPIPS %r" % (float(b.lo), float(b.hi), "]" if last else ")", b.count,
                                                          float(b.fid), float(b.lpips))
    for name, v in (("SSIM", b.ssim), ("PSNR", b.psnr), ("P-IDS", b.p_ids), ("U-IDS", b.u_ids), ("KID", b.kid),
                    ("Precision", b.precision), ("Recall", b.recall), ("Density", b.density),
                    ("Coverage", b.coverage)):
        if v is not None:
            line += " %s %r" % (name, float(v))
    return line


def print_result(res: Optional[EvalResult], ids: bool, ssim: bool = False, psnr: bool = False,
                 kid: bool = False, prdc: bool = False) -> None:
    """The script's two result lines on rank 0, then the mean SSIM and PSNR with `ssim` / `psnr`, then the
    discriminative scores' two with `ids`, then `KID: <repr>` with `kid`, then `Precision: <repr>`, `Recall: <repr>`,
    `Density: <repr>` and `Coverage: <repr>` with `prdc`, then one `hole_line` per bin with hole bins."""
    if res is not None:
        print("FID:", res.fid)
        print("LPIPS: ", res.lpips)
        if ssim:
            print("SSIM:", res.ssim)
        if psnr:
            print("PSNR:", res.psnr)
        if ids:
            print("P-IDS:", res.p_ids)
            print("U-IDS:", res.u_ids)
        if kid:
            print("KID: %r" % float(res.kid))
        if prdc:
            for name in ("precision", "recall", "density", "coverage"):
                print("%s: %r" % (name.capitalize(), float(getattr(res.prdc, name))))
        if res.by_hole is not None:
            for k, b in enumerate(res.by_hole):
                print(hole_line(b, k == len(res.by_hole) - 1))


def finish_command(res: Optional[EvalResult], args) -> None:
    """Rank 0's output: the result lines, and the --per-image file."""
    print_result(res, args.ids, args.ssim, args.psnr, args.kid, args.prdc)
    if res is not None and args.per_image is not None:
        write_per_image(args.per_image, res.per_image)


def main(argv=None) -> None:
    args = get_args(argv)
    resolution(args.model_name)
    check_per_image_path(args.per_image)
    hole_bins, hole_range = check_hole_flags(args)
    res = run_command(args.device, lambda device: evaluate(
        args.model_name, args.model_path, args.real_dir, args.mask_dir, device=device, batch_size=args.batch_size,
        num_workers=args.num_workers, noise_seed=args.noise_seed, real_stats=args.real_stats,
        save_real_stats_to=args.save_real_stats, inception_weights=args.inception_weights,
        lpips_weights=args.lpips_weights, ids=args.ids, ssim=args.ssim, psnr=args.psnr,
        per_image=args.per_image is not None, hole_bins=hole_bins, hole_range=hole_range, kid=args.kid,
        prdc=args.prdc))
    finish_command(res, args)


if __name__ == "__main__":
    main()

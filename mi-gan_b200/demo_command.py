"""scripts/demo.py on the GPU: the same command line and the same files, on one GPU or all the GPUs of a box.

    python -m migan_b200.demo --model-name migan-512 --model-path M.pt --images-dir I --masks-dir M --output-dir O
    torchrun --standalone --nproc_per_node=8 -m migan_b200.demo --model-name migan-512 ...

The files follow scripts/demo.py:115-142:

* photos: `glob(images_dir/**/*{ext}, recursive=True)` for .jpg, .jpeg and .png (case-sensitive, subdirectories
  included), `sorted`;
* the mask of photo p: `masks_dir / ("".join(basename(p).split(".")[:-1]) + ".png")` (inner dots dropped: a.b.jpg takes
  ab.png); its output: `output_dir / (Path(p).stem + ".png")` (dots kept: a.b.jpg writes a.b.png);
* photos are decoded with `Image.open(p).convert("RGB")`, masks with `np.array(Image.open(m))` as they are (any mode that
  decodes to uint8 with 1 to 4 channels: L, P, LA, RGB, RGBA, CMYK, ...), and results are written with
  `Image.fromarray(out).save(path)`, so with `--pipeline demo` a file is byte for byte the one demo.py writes;
* when several photos map to one output name, demo.py leaves the file of the last in sorted order: only that photo is
  processed, and it keeps its index k in the full sorted list.

Differences from the script:

* one planning pass reads every photo and mask header (size and mode, no pixels) before any GPU work and raises one
  `PlanError` naming every missing mask, every mask mode that does not decode to uint8 with 1 to 4 channels and every
  photo / mask pair the pipeline refuses by size.  Nothing is written then; the script stops at the first bad file,
  after writing the files before it;
* `--batch-size` photos (default 32) form a chunk, one `forward_batch`; `--num-workers` host threads decode and encode;
* Co-Mod-GAN draws its noise from seeded streams: image k gets seed `noise_seed * 2**32 + k` (`--noise-seed`).  Its
  style RMS is taken over the generator's batch (DESIGN §8), so its files depend on `--batch-size`, not on the GPU count;
* `--pipeline fullres` / `holewindow` write `FullResPipeline` / `HoleWindowPipeline` results at the photo's own size
  (MI-GAN only; the mask must have the photo's size).  Only CUDA devices run.

The loop: a thread pool decodes photos and masks into pinned host tensors up to `PREFETCH` chunks ahead of the chunk on
the GPU; each chunk is one `forward_batch(..., wait=False)`, whose results come back by asynchronous copies into pinned
buffers; the same pool PNG-encodes and writes them behind the GPU.  At most `INFLIGHT` chunks of photos and `INFLIGHT`
chunks of outputs are held in pinned memory, so `--batch-size` sets the bound: about 3 x batch x (largest photo +
largest output) bytes, 0.8 GB of photos for a chunk of 32 4K photos.  PyTorch's pinned-memory cache rounds blocks up to
a power of two and keeps them, so the process may hold up to twice that.

Sharding: under `torchrun` (WORLD_SIZE, RANK, LOCAL_RANK), chunk j of the planned list runs on rank j % W and each rank
writes its own files.  No process group is made.  A chunk is the same `forward_batch` call on any rank, so the files do
not depend on W.
"""
from __future__ import annotations

import argparse
import os
import sys
import time
import types
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from glob import glob
from pathlib import Path
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import comodgan
from ._request_path import load_generator
from .demo import DemoPipeline
from .evaluate_fid_lpips import MODELS, chunk_bounds, device_for, num_rounds, resolution, round_chunk
from .fullres import FullResPipeline
from .holewin import HoleWindowPipeline

IMG_EXTENSIONS = (".jpg", ".jpeg", ".png")      # demo.py:115; glob matches them case-sensitively
PIPELINES = {"demo": DemoPipeline, "fullres": FullResPipeline, "holewindow": HoleWindowPipeline}
BATCH_SIZE = 32
PREFETCH = 2                    # chunks decoded ahead of the one the GPU works on
INFLIGHT = 3                    # chunks of photos (and of outputs) held in pinned memory at most


# -- file rules -----------------------------------------------------------------------------------------------------

def list_photos(images_dir) -> List[str]:
    """demo.py:115-120: the .jpg, .jpeg and .png files under `images_dir`, subdirectories included, sorted."""
    paths = []
    for ext in IMG_EXTENSIONS:
        paths += glob(os.path.join(images_dir, "**", "*" + ext), recursive=True)
    return sorted(paths)


def mask_path(masks_dir, photo) -> Path:
    """demo.py:123: the inner dots of the photo's name are dropped (a.b.jpg -> ab.png)."""
    return Path(os.path.join(masks_dir, "".join(os.path.basename(photo).split(".")[:-1]) + ".png"))


def output_name(photo) -> str:
    """demo.py:142: the stem keeps its dots (a.b.jpg -> a.b.png)."""
    return Path(photo).stem + ".png"


class Item(NamedTuple):
    """A photo that is processed.  `index`: its position in the full sorted list (Co-Mod-GAN's seed is
    noise_seed * 2**32 + index); `output`: the file name it writes in the output directory."""
    index: int
    photo: str
    mask: Path
    output: str


def plan_items(photos: Sequence[str], masks_dir) -> List[Item]:
    """The photos to process, in sorted order: of the photos with one output name only the last, whose file demo.py
    leaves behind."""
    last = {output_name(p): k for k, p in enumerate(photos)}
    return [Item(k, p, mask_path(masks_dir, p), output_name(p)) for k, p in enumerate(photos)
            if last[output_name(p)] == k]


def mask_mode_supported(mode: str) -> bool:
    """Whether `np.array(Image.open(m))` of a mask in this mode is uint8 with 1 to 4 channels, as `read_mask` and the
    pipelines take it (L, P, LA, PA, RGB, RGBA, CMYK, ...; not 1, I, I;16 or F)."""
    from PIL import ImageMode
    try:
        m = ImageMode.getmode(mode)
    except KeyError:
        return False
    return m.typestr == "|u1" and 1 <= len(m.bands) <= 4


def _header(path):
    """(size (w, h), mode, bands) from the file's header; PIL decodes no pixels for this."""
    from PIL import Image
    with Image.open(path) as im:
        return im.size, im.mode, len(im.getbands())


def _size_check(pipeline: str, res: int):
    """The pipeline's own `_check_mask_size` on header sizes: it reads only `res`, its name and the two shapes, so it
    runs on a stand-in and zero-byte arrays of those shapes instead of a pipeline on the GPU."""
    cls = PIPELINES[pipeline]
    stand_in = types.SimpleNamespace(res=res, _name=cls._name)

    def check(photo_size, mask_size, mask_bands) -> None:
        (W, H), (Wm, Hm) = photo_size, mask_size
        img = np.broadcast_to(np.uint8(0), (H, W, 3))
        mask = np.broadcast_to(np.uint8(0), (Hm, Wm, mask_bands))
        cls._check_mask_size(stand_in, 0, img, mask)
    return check


class PlanError(ValueError):
    """Every file the command cannot process, found before anything is written: `problems` has one line per file."""

    def __init__(self, problems: Sequence[str]):
        self.problems = list(problems)
        super().__init__("%d file(s) cannot be processed; nothing was written:\n  %s"
                         % (len(self.problems), "\n  ".join(self.problems)))


def check_items(items: Sequence[Item], pipeline: str, res: int, num_workers: int = 2) -> None:
    """Read every photo and mask header; raise one `PlanError` naming every missing mask, unsupported mask mode and
    photo / mask pair the pipeline refuses by size."""
    check = _size_check(pipeline, res)

    def look(item: Item) -> Optional[str]:
        try:
            psize, _, _ = _header(item.photo)
        except Exception as e:  # noqa: BLE001 -- any unreadable photo is reported with the others
            return "photo %s: cannot be read (%s)" % (item.photo, e)
        if not item.mask.is_file():
            return "photo %s: no mask %s" % (item.photo, item.mask)
        try:
            msize, mode, bands = _header(item.mask)
        except Exception as e:  # noqa: BLE001
            return "mask %s: cannot be read (%s)" % (item.mask, e)
        if not mask_mode_supported(mode):
            return "mask %s: mode %s is not supported; masks must decode to uint8 with 1 to 4 channels (L, P, LA, RGB, " \
                   "RGBA, CMYK)" % (item.mask, mode)
        try:
            check(psize, msize, bands)
        except ValueError as e:
            return "photo %s (%dx%d), mask %s (%dx%d): %s" % (item.photo, psize[0], psize[1], item.mask, msize[0],
                                                              msize[1], e)
        return None

    with ThreadPoolExecutor(max_workers=max(1, int(num_workers))) as pool:
        problems = [p for p in pool.map(look, items) if p is not None]
    if problems:
        raise PlanError(problems)


# -- host decode and encode -----------------------------------------------------------------------------------------

def _pinned(a: np.ndarray) -> torch.Tensor:
    t = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    t.numpy()[...] = a
    return t


def decode_photo(path) -> torch.Tensor:
    """`Image.open(p).convert("RGB")` in a pinned uint8 tensor [H, W, 3]."""
    from PIL import Image
    with Image.open(path) as im:
        return _pinned(np.asarray(im.convert("RGB")))


def decode_mask(path) -> torch.Tensor:
    """`np.array(Image.open(m))`, unconverted, in a pinned uint8 tensor [H, W] or [H, W, C]; ValueError naming the file
    and its mode when that is not uint8 with 1 to 4 channels."""
    from PIL import Image
    with Image.open(path) as im:
        mode = im.mode
        a = np.array(im)
    if a.dtype != np.uint8 or not (a.ndim == 2 or (a.ndim == 3 and 1 <= a.shape[2] <= 4)):
        raise ValueError("mask %s: mode %s decodes to %s %s, not uint8 with 1 to 4 channels" % (path, mode, a.dtype,
                                                                                                 a.shape))
    return _pinned(a)


def encode(out: torch.Tensor, path) -> None:
    """demo.py:141-142: `Image.fromarray(out).save(path)` with PIL's PNG defaults."""
    from PIL import Image
    Image.fromarray(out.numpy()).save(path)


# -- setup and per-rank loop ----------------------------------------------------------------------------------------

def rank_chunks(n_chunks: int, rank: int, world_size: int) -> List[int]:
    """The chunks rank `rank` of `world_size` runs, in order: chunk j runs on rank j % W."""
    ran = (round_chunk(r, rank, n_chunks, world_size) for r in range(num_rounds(n_chunks, world_size)))
    return [j for j in ran if j is not None]


class DemoSetup:
    """What every rank of one run shares: the planned items, the chunking and the generator on `device`.  The plan and
    its checks (`PlanError`) come before the generator is loaded, so a bad data set costs no GPU work."""

    def __init__(self, model_name: str, model, images_dir, masks_dir, output_dir, *, invert_mask: bool = False,
                 device="cuda", batch_size: int = BATCH_SIZE, num_workers: int = 2, noise_seed: int = 0,
                 pipeline: str = "demo", margin: Optional[int] = None):
        self.res = resolution(model_name)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("migan_b200.demo runs on CUDA devices only (there is no CPU path); got --device %s" % device)
        if pipeline not in PIPELINES:
            raise ValueError("--pipeline %s: one of %s" % (pipeline, ", ".join(PIPELINES)))
        self.comodgan = MODELS[model_name][0] == "comodgan"
        if self.comodgan and pipeline != "demo":
            raise ValueError("--pipeline %s runs MI-GAN only; %s runs with --pipeline demo" % (pipeline, model_name))
        if margin is not None and pipeline != "holewindow":
            raise ValueError("--margin applies to --pipeline holewindow only")
        if int(batch_size) < 1:
            raise ValueError("--batch-size must be >= 1, got %d" % batch_size)
        if not 0 <= int(noise_seed) < 1 << 32:
            raise ValueError("--noise-seed must lie in [0, 2**32), got %d" % noise_seed)
        self.pipeline, self.margin = pipeline, 1 if margin is None else int(margin)
        self.invert_mask, self.noise_seed = bool(invert_mask), int(noise_seed)
        self.num_workers = max(1, int(num_workers))
        self.output_dir = Path(output_dir)
        self.photos = list_photos(images_dir)
        self.items = plan_items(self.photos, masks_dir)
        check_items(self.items, pipeline, self.res, self.num_workers)
        self.chunks = chunk_bounds(len(self.items), int(batch_size))
        if self.comodgan:
            self.model = comodgan.load(model, self.res).to(self.device)
        else:
            self.model = load_generator(self, model, self.res, self.device)

    def make_pipeline(self):
        if self.pipeline == "demo":
            return DemoPipeline(self.model, self.res, device=self.device, noise_seed=self.noise_seed)
        if self.pipeline == "fullres":
            return FullResPipeline(self.model, self.res, device=self.device)
        return HoleWindowPipeline(self.model, self.res, margin=self.margin, device=self.device)

    def seeds(self, j: int) -> Optional[np.ndarray]:
        """Chunk j's Co-Mod-GAN seeds, noise_seed * 2**32 + k for each image's index k in the full sorted list (None
        for MI-GAN)."""
        if not self.comodgan:
            return None
        a, b = self.chunks[j]
        return np.array([(self.noise_seed << 32) + it.index for it in self.items[a:b]], dtype=np.uint64)


class RunStats(NamedTuple):
    images: int                 # files this rank wrote
    seconds: float              # wall time of this rank's chunk loop, the last file written included
    decode_wait_s: float        # host time waiting for decoded chunks
    gpu_wait_s: float           # host time waiting for a chunk's results
    encode_wait_s: float        # host time waiting for encodes (bounded pinned memory, and the last chunks)


def run_rank(setup: DemoSetup, rank: int = 0, world_size: int = 1, progress: bool = False) -> RunStats:
    """Run and write the chunks of rank `rank` of `world_size` (all of them at W = 1)."""
    if world_size < 1 or not 0 <= rank < world_size:
        raise ValueError("bad rank %d of %d" % (rank, world_size))
    own = rank_chunks(len(setup.chunks), rank, world_size)
    setup.output_dir.mkdir(parents=True, exist_ok=True)
    pipe = setup.make_pipeline()
    dev = setup.device if setup.device.index is not None else torch.device("cuda", torch.cuda.current_device())
    decoding = deque()          # (j, photo futures, mask futures), in chunk order
    on_gpu = deque()            # (j, outputs): enqueued, not yet waited for
    encoding = deque()          # encode futures of one chunk each
    waits = {"decode": 0.0, "gpu": 0.0, "encode": 0.0}
    t0 = time.perf_counter()
    nxt = 0
    done_images = 0

    def timed(what, fn):
        t = time.perf_counter()
        out = fn()
        waits[what] += time.perf_counter() - t
        return out

    pool = ThreadPoolExecutor(max_workers=setup.num_workers, initializer=torch.cuda.set_device, initargs=(dev,))
    try:
        def submit_decodes():
            nonlocal nxt
            while nxt < len(own) and len(decoding) < PREFETCH and len(decoding) + len(on_gpu) < INFLIGHT:
                a, b = setup.chunks[own[nxt]]
                items = setup.items[a:b]
                decoding.append((own[nxt], [pool.submit(decode_photo, it.photo) for it in items],
                                 [pool.submit(decode_mask, it.mask) for it in items]))
                nxt += 1

        def finish_oldest():
            nonlocal done_images
            j, outs = on_gpu.popleft()
            timed("gpu", lambda: pipe.wait(1))
            while encoding:                      # one chunk encoding at a time: INFLIGHT chunks of outputs at most
                futs = encoding.popleft()
                timed("encode", lambda: [f.result() for f in futs])
            a, b = setup.chunks[j]
            encoding.append([pool.submit(encode, out, setup.output_dir / it.output)
                             for out, it in zip(outs, setup.items[a:b])])
            done_images += b - a
            if progress and rank == 0:
                el = time.perf_counter() - t0
                print("migan_b200.demo: chunk %d of %d done (images %d-%d); rank 0: %d images in %.1f s"
                      % (j + 1, len(setup.chunks), a, b - 1, done_images, el), file=sys.stderr, flush=True)

        with torch.cuda.device(dev):
            for j in own:
                submit_decodes()
                got, photo_futs, mask_futs = decoding.popleft()
                assert got == j
                photos = timed("decode", lambda: [f.result() for f in photo_futs])
                masks = timed("decode", lambda: [f.result() for f in mask_futs])
                if setup.pipeline == "demo":
                    outs = pipe.forward_batch(photos, masks, setup.invert_mask, wait=False, seeds=setup.seeds(j))
                else:
                    outs = pipe.forward_batch(photos, masks, setup.invert_mask, wait=False)
                del photos, masks                # the pipeline keeps them until the chunk is waited for
                on_gpu.append((j, outs))
                if len(on_gpu) > 1:
                    finish_oldest()              # the chunk before this one, while this one runs
                submit_decodes()
            while on_gpu:
                finish_oldest()
            while encoding:
                futs = encoding.popleft()
                timed("encode", lambda: [f.result() for f in futs])
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    return RunStats(done_images, time.perf_counter() - t0, waits["decode"], waits["gpu"], waits["encode"])


# -- entry points ---------------------------------------------------------------------------------------------------

def demo(model_name: str, model, images_dir, masks_dir, output_dir, *, invert_mask: bool = False, device="cuda",
         batch_size: int = BATCH_SIZE, num_workers: int = 2, noise_seed: int = 0, pipeline: str = "demo",
         margin: Optional[int] = None, rank: int = 0, world_size: int = 1, progress: bool = False) -> RunStats:
    """Write the command's files: plan and check every file, load `model` (a state_dict, a path to one, or a generator
    object: MI-GAN `Generator`, or `comodgan.Generator` for the comodgan names) and run the chunks of rank `rank` of
    `world_size`."""
    setup = DemoSetup(model_name, model, images_dir, masks_dir, output_dir, invert_mask=invert_mask, device=device,
                      batch_size=batch_size, num_workers=num_workers, noise_seed=noise_seed, pipeline=pipeline,
                      margin=margin)
    return run_rank(setup, rank, world_size, progress)


def get_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m migan_b200.demo")
    parser.add_argument("--model-name", type=str, help="One of [migan-256, migan-512, comodgan-256, comodgan-512]",
                        required=True)
    parser.add_argument("--model-path", type=str, help="Saved model path.", required=True)
    parser.add_argument("--images-dir", type=Path, help="Path to images directory.", required=True)
    parser.add_argument("--masks-dir", type=Path, help="Path to masks directory.", required=True)
    parser.add_argument("--invert-mask", action="store_true", help="Invert mask? (make 0-known, 1-hole)")
    parser.add_argument("--output-dir", type=Path, help="Output directory.", required=True)
    parser.add_argument("--device", type=str, help="Device (CUDA only).", default="cuda")
    parser.add_argument("--batch-size", type=int, default=BATCH_SIZE,
                        help="Photos per chunk: one forward_batch, and the unit of sharding.")
    parser.add_argument("--num-workers", type=int, default=2, help="Host threads for decoding and encoding.")
    parser.add_argument("--noise-seed", type=int, default=0,
                        help="Co-Mod-GAN: image k of the sorted list gets noise seed noise_seed * 2**32 + k.")
    parser.add_argument("--pipeline", choices=sorted(PIPELINES), default="demo",
                        help="demo: demo.py's files; fullres / holewindow: MI-GAN at the photo's own size.")
    parser.add_argument("--margin", type=int, default=None, help="holewindow: cells of context around the holes "
                        "(default 1).")
    return parser.parse_args(argv)


def main(argv=None) -> None:
    args = get_args(argv)
    resolution(args.model_name)
    if torch.device(args.device).type != "cuda":
        raise RuntimeError("migan_b200.demo runs on CUDA devices only (there is no CPU path); got --device %s"
                           % args.device)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = device_for(args.device, world, local_rank)
    if world > 1:
        torch.cuda.set_device(device)
    stats = demo(args.model_name, args.model_path, args.images_dir, args.masks_dir, args.output_dir,
                 invert_mask=args.invert_mask, device=device, batch_size=args.batch_size, num_workers=args.num_workers,
                 noise_seed=args.noise_seed, pipeline=args.pipeline, margin=args.margin, rank=rank, world_size=world,
                 progress=True)
    if rank == 0:
        print("migan_b200.demo: rank 0 of %d wrote %d files to %s in %.1f s"
              % (world, stats.images, args.output_dir, stats.seconds), file=sys.stderr, flush=True)


if __name__ == "__main__":
    main()

"""scripts/create_onnx_pipeline.py's sample loop on the GPU: the crop pipeline's result for every photo of a directory.

    python -m migan_b200.crop_results --resolution 512 --model-path M.pt --images-dir I --masks-dir M --output-dir O
    torchrun --standalone --nproc_per_node=8 -m migan_b200.crop_results --resolution 512 ...

The reference script exports `MIGAN_Pipeline` to ONNX and then, for every photo, decodes it, reads its mask with its
`read_mask`, runs the pipeline and writes `sample_results/<stem>.png` (:323-344).  This command runs that loop without the
export, through `CropPipeline` in batched passes:

* photos: `glob(images_dir/**/*{ext}, recursive=True)` for .jpg, .jpeg and .png, sorted; the mask of photo p is
  `masks_dir / ("".join(basename(p).split(".")[:-1]) + ".png")` (inner dots dropped); the output is
  `output_dir / "sample_results" / (Path(p).stem + ".png")`.  When several photos map to one output name, only the last in
  sorted order is processed, the one whose file the script leaves (the demo command's rules, `demo_command.py`);
* photos are decoded with `Image.open(p).convert("RGB")` at their own size, masks with `np.array(Image.open(m))`
  unconverted; the mask may have any size and 1 to 4 channels (`read_mask` of :27-45 and the NEAREST resize to the
  photo's size run on the GPU); results are written with `Image.fromarray(out).save(path)`.

With MI-GAN (`--generator migan`, the default) every file is byte for byte what the reference loop writes when its
pipeline call is this project's `MIGAN_Pipeline`, one photo at a time; the stored reference vectors of the reference's
own class are reproduced exactly.  Against the reference's torch `MIGAN_Pipeline` on the CPU (its commented-out line
:339) the files can differ: the anti-aliased crop resize rounds like torch's CPU resize except at rare values next to a
rounding boundary, where it lands one uint8 level away (on a seeded 569 x 405 photo, one element of the model input is
140 where torch gives 139), and that changes the generator's output for the photo.  ONNX Runtime's own arithmetic is
not reproduced either, so the files the script writes through its ONNX session may differ from these.

`--generator comodgan` runs a Co-Mod-GAN checkpoint of that resolution in the same pipeline.  Its noise comes from seeded
streams (image k of the sorted list gets seed `noise_seed * 2**32 + k`) and its style RMS is taken over the generator's
batch (DESIGN §8), so its files depend on `--batch-size`, not on the GPU count.  MI-GAN's files depend on neither.

The rest is the demo command's machinery (`demo_command.py`): one planning pass that reads every header and raises one
`PlanError` naming every missing mask, unsupported mask mode and photo under 3 x 3 before anything is written; thread-pool
decode and encode around `forward_batch(..., wait=False)` with bounded pinned memory; and under `torchrun` chunk j of the
planned list on rank j % W.  Only CUDA devices run.
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import torch

from . import comodgan
from ._request_path import load_generator
from .demo_command import BATCH_SIZE, DemoSetup, RunStats, check_items, list_photos, plan_items, run_rank
from .evaluate_fid_lpips import MODELS, chunk_bounds, device_for
from .pipeline import CropPipeline

GENERATORS = ("migan", "comodgan")
COMODGAN_RESOLUTIONS = tuple(sorted(r for kind, r in MODELS.values() if kind == "comodgan"))
PADDING = 128                   # MIGAN_Pipeline's default (create_onnx_pipeline.py:123)
RESULTS = "sample_results"      # the subdirectory the reference writes its files to (:329)


def check_options(resolution: int, generator: str, padding: int, device, batch_size: int, noise_seed: int) -> None:
    """Every refusal that needs no file and no GPU."""
    if generator not in GENERATORS:
        raise ValueError("--generator %s: one of %s" % (generator, ", ".join(GENERATORS)))
    if int(resolution) < 3:
        raise ValueError("--resolution must be >= 3, got %d" % resolution)
    if generator == "comodgan" and int(resolution) not in COMODGAN_RESOLUTIONS:
        raise ValueError("--generator comodgan runs at resolution %s, got --resolution %d"
                         % (" or ".join(map(str, COMODGAN_RESOLUTIONS)), resolution))
    if int(padding) < 0:
        raise ValueError("--padding must be >= 0, got %d" % padding)
    if torch.device(device).type != "cuda":
        raise RuntimeError("migan_b200.crop_results runs on CUDA devices only (there is no CPU path); got --device %s"
                           % device)
    if int(batch_size) < 1:
        raise ValueError("--batch-size must be >= 1, got %d" % batch_size)
    if not 0 <= int(noise_seed) < 1 << 32:
        raise ValueError("--noise-seed must lie in [0, 2**32), got %d" % noise_seed)


class CropSetup(DemoSetup):
    """What every rank of one run shares: the planned items, the chunking and the generator on `device`.  The checks
    and the plan (`PlanError`) come before the generator is loaded, so a bad data set costs no GPU work."""

    prog = "migan_b200.crop_results"

    def __init__(self, model, resolution: int, images_dir, masks_dir, output_dir, *, generator: str = "migan",
                 padding: int = PADDING, invert_mask: bool = False, device="cuda", batch_size: int = BATCH_SIZE,
                 num_workers: int = 2, noise_seed: int = 0):
        check_options(resolution, generator, padding, device, batch_size, noise_seed)
        self.res, self.padding = int(resolution), int(padding)
        self.device = torch.device(device)
        self.pipeline = "crop"
        self.comodgan = generator == "comodgan"
        self.invert_mask, self.noise_seed = bool(invert_mask), int(noise_seed)
        self.num_workers = max(1, int(num_workers))
        self.output_dir = Path(output_dir) / RESULTS
        self.photos = list_photos(images_dir)
        self.items = plan_items(self.photos, masks_dir)
        check_items(self.items, CropPipeline, self.res, self.num_workers)
        self.chunks = chunk_bounds(len(self.items), int(batch_size))
        if self.comodgan:
            self.model = comodgan.load(model, self.res).to(self.device)
        else:
            self.model = load_generator(self, model, self.res, self.device)

    def make_pipeline(self):
        return CropPipeline(self.model, self.res, self.padding, device=self.device, noise_seed=self.noise_seed)

    def forward(self, pipe, j: int, photos, masks) -> list:
        return pipe.forward_batch(photos, masks, self.invert_mask, wait=False, seeds=self.seeds(j))


def crop_results(model, resolution: int, images_dir, masks_dir, output_dir, *, generator: str = "migan",
                 padding: int = PADDING, invert_mask: bool = False, device="cuda", batch_size: int = BATCH_SIZE,
                 num_workers: int = 2, noise_seed: int = 0, rank: int = 0, world_size: int = 1,
                 progress: bool = False) -> RunStats:
    """Write the command's files: plan and check every file, load `model` (a state_dict, a path to one, or a generator
    object: MI-GAN `Generator`, or `comodgan.Generator` with generator="comodgan") and run the chunks of rank `rank` of
    `world_size`."""
    setup = CropSetup(model, resolution, images_dir, masks_dir, output_dir, generator=generator, padding=padding,
                      invert_mask=invert_mask, device=device, batch_size=batch_size, num_workers=num_workers,
                      noise_seed=noise_seed)
    return run_rank(setup, rank, world_size, progress)


def get_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m migan_b200.crop_results")
    parser.add_argument("--resolution", type=int, help="256 or 512", required=True)
    parser.add_argument("--model-path", type=str, help="Saved .pt model path.", required=True)
    parser.add_argument("--images-dir", type=Path, help="Path to images directory.", required=True)
    parser.add_argument("--masks-dir", type=Path, help="Path to masks directory.", required=True)
    parser.add_argument("--invert-mask", action="store_true", help="Invert mask? (make 0-known, 1-hole)")
    parser.add_argument("--output-dir", type=Path, help="Output directory.", required=True)
    parser.add_argument("--device", type=str, help="Device (CUDA only).", default="cuda")
    parser.add_argument("--generator", choices=GENERATORS, default="migan",
                        help="migan: an exported MI-GAN state_dict; comodgan: a Co-Mod-GAN checkpoint of --resolution.")
    parser.add_argument("--padding", type=int, default=PADDING, help="Context around the holes' bounding box (>= 0).")
    parser.add_argument("--batch-size", type=int, default=BATCH_SIZE,
                        help="Photos per chunk: one forward_batch, and the unit of sharding.")
    parser.add_argument("--num-workers", type=int, default=2, help="Host threads for decoding and encoding.")
    parser.add_argument("--noise-seed", type=int, default=0,
                        help="Co-Mod-GAN: image k of the sorted list gets noise seed noise_seed * 2**32 + k.")
    return parser.parse_args(argv)


def main(argv=None) -> None:
    args = get_args(argv)
    check_options(args.resolution, args.generator, args.padding, args.device, args.batch_size, args.noise_seed)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = device_for(args.device, world, local_rank, "migan_b200.crop_results")
    if world > 1:
        torch.cuda.set_device(device)
    stats = crop_results(args.model_path, args.resolution, args.images_dir, args.masks_dir, args.output_dir,
                         generator=args.generator, padding=args.padding, invert_mask=args.invert_mask, device=device,
                         batch_size=args.batch_size, num_workers=args.num_workers, noise_seed=args.noise_seed,
                         rank=rank, world_size=world, progress=True)
    if rank == 0:
        print("migan_b200.crop_results: rank 0 of %d wrote %d files to %s in %.1f s"
              % (world, stats.images, Path(args.output_dir) / RESULTS, stats.seconds), file=sys.stderr, flush=True)


if __name__ == "__main__":
    main()

"""migan_b200 -- H100-native (sm_90a) implementation of the MI-GAN generator forward pass.

Public surface (mirrors the reference's for this path):
    Generator(resolution)            drop-in for lib.model_zoo.migan_inference.Generator
    ops.upfirdn2d / ops.bias_act ... drop-ins for torch_utils.ops.{upfirdn2d,bias_act,conv2d_resample}
    pipeline.MIGAN_Pipeline          drop-in for scripts/create_onnx_pipeline.py:MIGAN_Pipeline (any-size image + mask -> in-place result)
    pipeline.CropPipeline            the same crop pipeline on decoded photos [H,W,3] and raw masks of any size
    demo.DemoPipeline                scripts/demo.py's request path at any photo size (PIL / OpenCV resizes on the GPU)
    fullres.FullResPipeline          photos of any size inpainted at their own resolution (reflect padding on the GPU)
    holewin.HoleWindowPipeline       the same, but only on windows around the holes; the rest of the photo is untouched
    masks.RandomMaskStream           scripts/generate_masks.py's RandomMask(s) on the GPU: same bytes, same numpy stream
    evaluate.EvalPipeline            evaluate_fid_lpips.py's batch around the generator: resizes, composite, normalisations
    evaluate.ResultsPipeline         the same batch around another method's result images in place of the generator
    fid.InceptionV3 / fid.FeatureStatistics / fid.calculate_frechet_distance
                                     pytorch_fid's FID features, statistics and distance (InceptionV3 on tensor cores)
    fid.frechet_distance / FeatureStatistics.frechet_distance
                                     the Frechet distance on the GPU (fp64 block-Jacobi eigensolver, deterministic)
    ids.inception_discriminative_scores
                                     Co-Mod-GAN's P-IDS and U-IDS (LinearSVC(dual=False) solved on the GPU, fp64 Newton)
    kid.kernel_inception_distance    the kernel Inception distance (StyleGAN2-ADA's KID, fp64 tensor-core kernel sums)
    prdc.precision_recall_density_coverage
                                      k-NN precision, recall, density and coverage (fp64 tensor-core distances)
    lpips.LPIPS                      drop-in for lpips.LPIPS(net="alex"): the script's LPIPS distance (AlexNet on tensor cores)
    metrics.compute_ssim / metrics.SSIM / metrics.compute_psnr
                                     the reference's SSIM (pytorch-ssim) and PSNR evaluators' arithmetic, in double
    generate_masks                   python -m migan_b200.generate_masks: the reference script's CLI and files
    evaluate_fid_lpips               python -m migan_b200.evaluate_fid_lpips: the evaluation script's CLI, sharded over GPUs
    score_results                    python -m migan_b200.score_results: the evaluation protocol over a directory of any
                                     method's result images, sharded over GPUs
    demo (python -m)                 python -m migan_b200.demo: scripts/demo.py's CLI and files, sharded over GPUs
    crop_results                     python -m migan_b200.crop_results: create_onnx_pipeline.py's sample loop, sharded over GPUs
    export.copy_weights              drop-in for scripts/export_inference_model.py:copy_weights (filters computed on the GPU)
    parallel.ShardedGenerator        batch sharding over the GPUs of one box + one all-gather of the outputs
    build.build()                    compile the C-ABI library (nvcc, sm_90a)

The directory is named `mi-gan_b200`; import it as `migan_b200` (repo-root shim `migan_b200.py`).
"""
import warnings as _warnings

# `python -m migan_b200.demo` runs demo.py as __main__ after this package has imported it as `migan_b200.demo`.  Its
# __main__ block only calls demo_command.main, so runpy's warning about the module's second copy does not apply.
_warnings.filterwarnings("ignore", message=r"'migan_b200\.demo' found in sys\.modules", category=RuntimeWarning)

from . import arch, build, demo, evaluate, export, fid, fullres, holewin, ids, kid, lpips, masks, metrics, ops, parallel, pipeline, prdc, synthetic  # noqa: F401
from .fullres import FullResPipeline  # noqa: F401
from .holewin import HoleWindowPipeline  # noqa: F401
from .evaluate import EvalPipeline, ResultsPipeline  # noqa: F401
from .masks import RandomMaskStream  # noqa: F401
from .generator import Generator  # noqa: F401

__all__ = ["EvalPipeline", "FullResPipeline", "Generator", "HoleWindowPipeline", "RandomMaskStream", "ResultsPipeline", "arch", "build", "demo", "evaluate", "export", "fid", "fullres", "holewin", "ids", "kid", "lpips", "masks", "metrics", "ops", "parallel", "pipeline", "prdc", "synthetic"]
__version__ = "0.1.0"

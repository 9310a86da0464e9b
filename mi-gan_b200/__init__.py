"""migan_b200 -- H100-native (sm_90a) implementation of the MI-GAN generator forward pass.

Public surface (mirrors the reference's for this path):
    Generator(resolution)            drop-in for lib.model_zoo.migan_inference.Generator
    ops.upfirdn2d / ops.bias_act ... drop-ins for torch_utils.ops.{upfirdn2d,bias_act,conv2d_resample}
    pipeline.MIGAN_Pipeline          drop-in for scripts/create_onnx_pipeline.py:MIGAN_Pipeline (any-size image + mask -> in-place result)
    demo.DemoPipeline                scripts/demo.py's request path at any photo size (PIL / OpenCV resizes on the GPU)
    fullres.FullResPipeline          photos of any size inpainted at their own resolution (reflect padding on the GPU)
    holewin.HoleWindowPipeline       the same, but only on windows around the holes; the rest of the photo is untouched
    masks.RandomMaskStream           scripts/generate_masks.py's RandomMask(s) on the GPU: same bytes, same numpy stream
    evaluate.EvalPipeline            evaluate_fid_lpips.py's batch around the generator: resizes, composite, normalisations
    fid.InceptionV3 / fid.FeatureStatistics / fid.calculate_frechet_distance
                                     pytorch_fid's FID features, statistics and distance (InceptionV3 on tensor cores)
    lpips.LPIPS                      drop-in for lpips.LPIPS(net="alex"): the script's LPIPS distance (AlexNet on tensor cores)
    generate_masks                   python -m migan_b200.generate_masks: the reference script's CLI and files
    export.copy_weights              drop-in for scripts/export_inference_model.py:copy_weights (filters computed on the GPU)
    parallel.ShardedGenerator        batch sharding over the GPUs of one box + one all-gather of the outputs
    build.build()                    compile the C-ABI library (nvcc, sm_90a)

The directory is named `mi-gan_b200`; import it as `migan_b200` (repo-root shim `migan_b200.py`).
"""
from . import arch, build, demo, evaluate, export, fid, fullres, holewin, lpips, masks, ops, parallel, pipeline, synthetic  # noqa: F401
from .fullres import FullResPipeline  # noqa: F401
from .holewin import HoleWindowPipeline  # noqa: F401
from .evaluate import EvalPipeline  # noqa: F401
from .masks import RandomMaskStream  # noqa: F401
from .generator import Generator  # noqa: F401

__all__ = ["EvalPipeline", "FullResPipeline", "Generator", "HoleWindowPipeline", "RandomMaskStream", "arch", "build", "demo", "evaluate", "export", "fid", "fullres", "holewin", "lpips", "masks", "ops", "parallel", "pipeline", "synthetic"]
__version__ = "0.1.0"

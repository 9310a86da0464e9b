"""migan_b200 -- H100-native (sm_90a) implementation of the MI-GAN generator forward pass.

Public surface (mirrors the reference's for this path):
    Generator(resolution)            drop-in for lib.model_zoo.migan_inference.Generator
    ops.upfirdn2d / ops.bias_act ... drop-ins for torch_utils.ops.{upfirdn2d,bias_act,conv2d_resample}
    pipeline.MIGAN_Pipeline          drop-in for scripts/create_onnx_pipeline.py:MIGAN_Pipeline (any-size image + mask -> in-place result)
    export.copy_weights              drop-in for scripts/export_inference_model.py:copy_weights (filters computed on the GPU)
    parallel.ShardedGenerator        batch sharding over the GPUs of one box + one all-gather of the outputs
    build.build()                    compile the C-ABI library (nvcc, sm_90a)

The directory is named `mi-gan_b200`; import it as `migan_b200` (repo-root shim `migan_b200.py`).
"""
from . import arch, build, export, ops, parallel, pipeline, synthetic  # noqa: F401
from .generator import Generator  # noqa: F401

__all__ = ["Generator", "arch", "build", "export", "ops", "parallel", "pipeline", "synthetic"]
__version__ = "0.1.0"

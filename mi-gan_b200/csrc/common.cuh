// Shared device helpers for the MI-GAN generator kernels (sm_90a only).
//
// Activation semantics follow lrelu_agc in the reference,
// lib/model_zoo/migan_inference.py:20-28 with the constants every block passes
// (alpha=0.2, gain=sqrt(2), clamp=256; :179,:210,:255,:289,:325).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace migan {

constexpr float kLreluAlpha = 0.2f;
constexpr float kActGain = 1.41421356237309515f;  // float(np.sqrt(2)) as torch casts it to fp32
constexpr float kActClamp = 256.0f;

// Power-of-two scales applied before the fp16 hi/lo split of the pointwise-conv
// operands (undone exactly in the epilogue).  Activations are clamped to +-256 before
// every 1x1 conv, so 2^6 keeps them < 65504; weights are unit-L2-norm rows (|w| <= 1)
// in released checkpoints, the scale is chosen per layer on the host from max|w|.
constexpr float kActSplitScale = 64.0f;

__device__ __forceinline__ float lrelu_agc(float v) {
    v = v < 0.0f ? v * kLreluAlpha : v;
    v = v * kActGain;
    return fminf(fmaxf(v, -kActClamp), kActClamp);
}

__device__ __forceinline__ float4 lrelu_agc4(float4 v) {
    v.x = lrelu_agc(v.x); v.y = lrelu_agc(v.y); v.z = lrelu_agc(v.z); v.w = lrelu_agc(v.w);
    return v;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void stg4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

__device__ __forceinline__ void fma4(float4& acc, const float4 w, const float4 v) {
    acc.x = fmaf(w.x, v.x, acc.x); acc.y = fmaf(w.y, v.y, acc.y);
    acc.z = fmaf(w.z, v.z, acc.z); acc.w = fmaf(w.w, v.w, acc.w);
}

// fp32 -> (hi, lo) fp16 pair with v*scale ~= hi + lo (22-23 significant bits).
__device__ __forceinline__ void split_f16(float v, float scale, __half& hi, __half& lo) {
    float s = v * scale;
    hi = __float2half_rn(s);
    lo = __float2half_rn(s - __half2float(hi));
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may start while
// its predecessor in the stream is still draining; everything before pdl_wait() (barrier setup, weight-table loads --
// nothing the predecessor writes) overlaps the predecessor's tail, everything after it sees the predecessor's memory.
// pdl_trigger() lets the successor's blocks start launching as soon as every block of this grid has passed it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Host: kernel launch with the PDL attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace migan

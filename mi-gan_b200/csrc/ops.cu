// Standalone sm_90a versions of the reference's two CUDA plugin ops (forward only):
//   upfirdn2d : torch_utils/ops/upfirdn2d.cpp:16-94 + upfirdn2d.cu:29-200
//   bias_act  : torch_utils/ops/bias_act.cpp:32-90  + bias_act.cu:23-147
// Both are pure HBM streaming ops on NCHW fp32 tensors (the plugin's public layout).
#include "common.cuh"
#include "kernels.h"

namespace migan {

// --------------------------------------------------------------------------------------
// upfirdn2d: zero-insert up-sample, pad/crop, FIR, decimate.  One thread = 4 consecutive
// outputs along x of one (n, c, oy) row -> 128-bit coalesced stores; only the polyphase taps
// that meet a non-zero sample of the zero-inserted signal are visited.
//   out[oy][ox] = gain * sum_{fy,fx} F[fy][fx] * U[oy*downy + fy - pady0][ox*downx + fx - padx0]
//   F = f flipped unless flip_filter (true convolution, upfirdn2d.py:198-200 / .cu:125-126)
// --------------------------------------------------------------------------------------
constexpr int kMaxTaps = 32 * 32;
__global__ void __launch_bounds__(256)
upfirdn2d_kernel(const float* __restrict__ x, const float* __restrict__ f, float* __restrict__ y,
                 int64_t rows /* n*c*oh */, int h, int w, int oh, int ow, int fh, int fw,
                 int upx, int upy, int downx, int downy, int padx0, int pady0, int flip, float gain) {
    extern __shared__ float sf[];  // fh*fw taps, already flipped + gain-scaled
    for (int i = threadIdx.x; i < fh * fw; i += blockDim.x) {
        const int fy = i / fw, fx = i % fw;
        const int sy = flip ? fy : fh - 1 - fy, sx = flip ? fx : fw - 1 - fx;
        sf[i] = __ldg(f + sy * fw + sx) * gain;
    }
    __syncthreads();
    const int ow4 = (ow + 3) >> 2;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * ow4) return;
    const int ox0 = (int)(idx % ow4) * 4;
    const int64_t row = idx / ow4;
    const int oy = (int)(row % oh);
    const int64_t nc = row / oh;
    const float* xp = x + nc * (int64_t)h * w;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    // first tap index whose upsampled coordinate is a multiple of upy
    const int uy0 = oy * downy - pady0;
    int fy0 = (-uy0) % upy; if (fy0 < 0) fy0 += upy;
    for (int fy = fy0; fy < fh; fy += upy) {
        const int uy = uy0 + fy;
        if (uy < 0) continue;
        const int iy = uy / upy;
        if (iy >= h) break;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int ox = ox0 + j;
            if (ox >= ow) break;
            const int ux0 = ox * downx - padx0;
            int fx0 = (-ux0) % upx; if (fx0 < 0) fx0 += upx;
            for (int fx = fx0; fx < fw; fx += upx) {
                const int ux = ux0 + fx;
                if (ux < 0) continue;
                const int ix = ux / upx;
                if (ix >= w) break;
                acc[j] = fmaf(sf[fy * fw + fx], __ldg(xp + (int64_t)iy * w + ix), acc[j]);
            }
        }
    }
    float* yp = y + row * ow + ox0;
    if (ox0 + 3 < ow && (((uintptr_t)yp) & 15) == 0) {
        *reinterpret_cast<float4*>(yp) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    } else {
        for (int j = 0; j < 4 && ox0 + j < ow; ++j) yp[j] = acc[j];
    }
}

cudaError_t launch_upfirdn2d(const float* x, const float* f, float* y, int n, int c, int h, int w,
                             int fh, int fw, int upx, int upy, int downx, int downy,
                             int padx0, int padx1, int pady0, int pady1, int flip, float gain,
                             int oh, int ow, cudaStream_t s) {
    (void)padx1; (void)pady1;
    if (fh * fw > kMaxTaps || fh < 1 || fw < 1) return cudaErrorInvalidValue;
    const int64_t rows = (int64_t)n * c * oh;
    const int64_t items = rows * ((ow + 3) / 4);
    if (items == 0) return cudaSuccess;
    upfirdn2d_kernel<<<(unsigned)((items + 255) / 256), 256, fh * fw * sizeof(float), s>>>(
        x, f, y, rows, h, w, oh, ow, fh, fw, upx, upy, downx, downy, padx0, pady0, flip, gain);
    return cudaGetLastError();
}

// --------------------------------------------------------------------------------------
// bias_act: y = clamp(gain * act(x + b[(i / step_b) % size_b]))   (bias_act.cu:23-147, grad = 0)
// act index follows the plugin's cuda_idx (bias_act.py:22-32):
//   1 linear 2 relu 3 lrelu 4 tanh 5 sigmoid 6 elu 7 selu 8 softplus 9 swish
// --------------------------------------------------------------------------------------
__device__ __forceinline__ float apply_act(float v, int act, float alpha) {
    switch (act) {
        default:
        case 1: return v;
        case 2: return v > 0.f ? v : 0.f;
        case 3: return v > 0.f ? v : v * alpha;
        case 4: return tanhf(v);
        case 5: return 1.0f / (1.0f + expf(-v));
        case 6: return v > 0.f ? v : expm1f(v);
        case 7: return v > 0.f ? 1.0507009873554804934193349852946f * v
                               : 1.0507009873554804934193349852946f * 1.6732632423543772848170429916717f * expm1f(v);
        case 8: return v > 20.f ? v : log1pf(expf(v));  // torch softplus threshold = 20
        case 9: return v / (1.0f + expf(-v));
    }
}

__global__ void __launch_bounds__(256)
bias_act_kernel(const float* __restrict__ x, const float* __restrict__ b, float* __restrict__ y,
                int64_t numel, int64_t step_b, int size_b, int act, float alpha, float gain, float clamp) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i0 >= numel) return;
    const bool vec = (i0 + 3 < numel) && ((((uintptr_t)(x + i0)) | ((uintptr_t)(y + i0))) & 15) == 0;
    float v[4];
    if (vec) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(x + i0));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        for (int j = 0; j < 4; ++j) v[j] = (i0 + j < numel) ? __ldg(x + i0 + j) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float t = v[j];
        if (b) t += __ldg(b + ((i0 + j) / step_b) % size_b);
        t = apply_act(t, act, alpha) * gain;
        if (clamp >= 0.f) t = fminf(fmaxf(t, -clamp), clamp);
        v[j] = t;
    }
    if (vec) {
        *reinterpret_cast<float4*>(y + i0) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
        for (int j = 0; j < 4 && i0 + j < numel; ++j) y[i0 + j] = v[j];
    }
}

cudaError_t launch_bias_act(const float* x, const float* b, float* y, int64_t numel, int64_t step_b, int size_b,
                            int act, float alpha, float gain, float clamp, cudaStream_t s) {
    if (numel == 0) return cudaSuccess;
    if (act < 1 || act > 9) return cudaErrorInvalidValue;
    if (b && (step_b < 1 || size_b < 1)) return cudaErrorInvalidValue;
    const int64_t items = (numel + 3) / 4;
    bias_act_kernel<<<(unsigned)((items + 255) / 256), 256, 0, s>>>(x, b, y, numel, step_b, size_b, act, alpha, gain, clamp);
    return cudaGetLastError();
}

}  // namespace migan

// Item kernels of the LPIPS forward (lpips_abi.cu), in the style of inception_kernels.cuh: each functor produces item i
// from global memory only and launches through ck_launch(), so the same code runs as a host loop in the emulation build.
// The convolutions and pools are the FID network's (inception.cu, incep::PoolK).
//
// Batch: the n image pairs run through AlexNet as one batch of 2n images, image i from in0 and image n + i from in1.
// No atomics, every sum in a fixed order: the value of pair i depends only on its two images.  LPIPS(a, b) and
// LPIPS(b, a) evaluate the same expressions with the roles swapped, so they are bitwise equal, and LPIPS(x, x) == 0.
#pragma once
#include "comod_kernels.cuh"

namespace lpips {

using comod::f4;
using comod::ld4;
using comod::st4;

// NCHW [n][3][H][W] of in0 then in1 -> NHWC [2n][H][W][4]: v = normalize ? 2x - 1 : x, then (v - shift) / scale
// (lpips' ScalingLayer); channel 3 zero (the first convolution reads 4-channel pixels).
struct InputK {        // items = 2n*H*W
    const float* in0; const float* in1; float* out;
    int n, HW, normalize;
    float shift[3], scale[3];
    CK_HD void operator()(int64_t i) const {
        const int64_t img = i / HW, p = i - img * HW;
        const float* src = img < n ? in0 + img * 3 * HW : in1 + (img - n) * 3 * HW;
        float v[3];
        for (int c = 0; c < 3; ++c) {
            float x = src[c * (int64_t)HW + p];
            if (normalize) x = 2.f * x - 1.f;
            v[c] = (x - shift[c]) / scale[c];
        }
        st4(out + i * 4, f4{v[0], v[1], v[2], 0.f});
    }
};

// One tapped layer's per-pixel distance of pair i: f0 = pixel p of image i, f1 = the same pixel of image n + i,
// C channels (a multiple of 4).  Each is divided by (its L2 norm over the channels + 1e-10), and
// d = sum_c w[c] * (f0/|f0| - f1/|f1|)^2 (lpips' normalize_tensor, squared difference, 1 x 1 `lin` without bias).
struct DistanceK {     // items = n*HW
    const float* f; const float* w; float* out;
    int n, HW, C;
    CK_HD void operator()(int64_t i) const {
        const int64_t pair = i / HW, p = i - pair * HW;
        const float* a = f + (pair * HW + p) * C;
        const float* b = f + ((pair + n) * HW + p) * C;
        float sa = 0.f, sb = 0.f;
        for (int c = 0; c < C; c += 4) {
            const f4 u = ld4(a + c), v = ld4(b + c);
            sa += u.x * u.x; sa += u.y * u.y; sa += u.z * u.z; sa += u.w * u.w;
            sb += v.x * v.x; sb += v.y * v.y; sb += v.z * v.z; sb += v.w * v.w;
        }
        const float na = sqrtf(sa) + 1e-10f, nb = sqrtf(sb) + 1e-10f;
        float d = 0.f;
        for (int c = 0; c < C; c += 4) {
            const f4 u = ld4(a + c), v = ld4(b + c), g = ld4(w + c);
            float t;
            t = u.x / na - v.x / nb; t = t * t; d += g.x * t;
            t = u.y / na - v.y / nb; t = t * t; d += g.y * t;
            t = u.z / na - v.z / nb; t = t * t; d += g.z * t;
            t = u.w / na - v.w / nb; t = t * t; d += g.w * t;
        }
        out[i] = d;
    }
};

// The final reduction, one block of kReduceThreads per pair (lpips_abi.cu: one body over portable.cuh's block layer,
// with its shared-memory tree).  For each layer k, thread t sums pixels t, t + 256, ... of
// pair i in double (partial()), the block adds the 256 partial sums in a fixed tree (stride 128, 64, ..., 1), and the
// spatial mean rounded to fp32 is the layer term; the total adds the five terms in order, as lpips does
// (val = 0; val += res[k]).  px: layer k's per-pixel values [n][hw[k]] at px + off[k].
constexpr int kReduceThreads = 256;
struct ReduceArgs {
    static constexpr int kLayers = 5;
    const float* px; float* out; float* per_layer;   // per_layer [5][n] or null
    int n;
    int hw[kLayers];
    int64_t off[kLayers];
    CK_HD double partial(int64_t i, int k, int t) const {
        const float* q = px + off[k] + i * hw[k];
        double s = 0.0;
        for (int p = t; p < hw[k]; p += kReduceThreads) s += (double)q[p];
        return s;
    }
    // thread 0, with layer k's tree result in s0
    CK_HD float layer_term(int64_t i, int k, double s0) const {
        const float m = (float)(s0 / hw[k]);
        if (per_layer) per_layer[k * (int64_t)n + i] = m;
        return m;
    }
};

}  // namespace lpips

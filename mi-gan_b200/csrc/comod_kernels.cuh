// Item kernels of the Co-Mod-GAN / conv2d_resample path (comodgan_abi.cu).
//
// Every kernel here is a functor whose operator()(i) produces output element (or float4) number i from global
// memory only -- no shared memory, no warp collectives -- launched through ck_launch() as one thread per item.
// That restriction is deliberate: the same functors compile as plain C++ (-DMIGAN_EMULATE, tests/emul/) where
// ck_launch() is a host loop, so the index math, the padding bookkeeping and the whole host-side plan are checked
// against the oracle on a machine without a GPU.  The emulation build is TEST INFRASTRUCTURE: the package never
// loads it, and the product library is compiled without MIGAN_EMULATE (no host loop exists in it).
//
// The arithmetic-heavy part (the GEMM the convolutions are lowered to) is NOT here: it is launch_pw_gemm_simt
// (gemm_simt.cu, fp32 CUDA-core FMA).
//
// Layout: activations NHWC fp32 [n][H][W][C]; GEMM operands row-major; all indices 64-bit.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef MIGAN_EMULATE
#define CK_HD inline
typedef void* ck_stream_t;
#else
#include <cuda_runtime.h>
#define CK_HD __host__ __device__ __forceinline__
typedef cudaStream_t ck_stream_t;
#endif

#ifdef MIGAN_EMULATE
typedef _Float16 ck_half;                       // IEEE binary16, round-to-nearest-even conversions (GCC, x86-64)
CK_HD ck_half ck_f2h(float v) { return (ck_half)v; }
CK_HD float ck_h2f(ck_half h) { return (float)h; }
#else
#include <cuda_fp16.h>
typedef __half ck_half;
CK_HD ck_half ck_f2h(float v) { return __float2half_rn(v); }
CK_HD float ck_h2f(ck_half h) { return __half2float(h); }
#endif

namespace comod {

struct alignas(16) f4 { float x, y, z, w; };
struct alignas(8) h4 { ck_half x, y, z, w; };
CK_HD f4 ld4(const float* p) { return *reinterpret_cast<const f4*>(p); }
CK_HD void st4(float* p, const f4& v) { *reinterpret_cast<f4*>(p) = v; }

#ifdef MIGAN_EMULATE
template <class F>
inline int ck_launch(const F& f, int64_t items, ck_stream_t) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < items; ++i) f(i);
    return 0;
}
#else
template <class F>
__global__ void __launch_bounds__(256) ck_items_kernel(const F f, const int64_t items) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < items) f(i);
}
template <class F>
inline cudaError_t ck_launch(const F& f, int64_t items, ck_stream_t s) {
    if (items <= 0) return cudaSuccess;
    ck_items_kernel<F><<<(unsigned)((items + 255) / 256), 256, 0, s>>>(f, items);
    return cudaGetLastError();
}
#endif

// ---- layout changes at the NCHW boundary ------------------------------------------------------------------------
struct NchwToNhwcK {   // items = n*H*W*C (output order)
    const float* in; float* out; int H, W, C;
    CK_HD void operator()(int64_t i) const {
        const int c = (int)(i % C); int64_t t = i / C;
        const int x = (int)(t % W); t /= W;
        const int y = (int)(t % H); const int64_t n = t / H;
        out[i] = in[((n * C + c) * H + y) * (int64_t)W + x];
    }
};
struct NhwcToNchwK {   // items = n*C*H*W (output order); reads channel c0 + c of a Ct-channel NHWC tensor
    const float* in; float* out; int H, W, C, Ct, c0;
    CK_HD void operator()(int64_t i) const {
        const int x = (int)(i % W); int64_t t = i / W;
        const int y = (int)(t % H); t /= H;
        const int c = (int)(t % C); const int64_t n = t / C;
        out[i] = in[((n * H + y) * (int64_t)W + x) * Ct + c0 + c];
    }
};

// ---- im2col: NHWC input -> GEMM A operand [P = n*OH*OW][KP], column k = (ky*kw + kx)*Cg + c, zero padded to KP ----
// Reads channels [c0, c0+Cg) of a Ct-channel tensor (grouped convolutions) and multiplies by scale[n][c] when given
// (the modulation of stylegan.py:173, "scale the activations" form).  iy = oy*stride + ky - pad_y.
struct Im2colK {       // items = P*KP (one element each); any Cg
    const float* in; const float* scale; float* out;
    int H, W, Ct, c0, Cg, kh, kw, stride, pad_y, pad_x, OH, OW, KP;
    CK_HD void operator()(int64_t i) const {
        const int k = (int)(i % KP); const int64_t p = i / KP;
        const int ox = (int)(p % OW); const int64_t t = p / OW;
        const int oy = (int)(t % OH); const int64_t n = t / OH;
        float v = 0.f;
        if (k < kh * kw * Cg) {
            const int tap = k / Cg, c = k - tap * Cg;
            const int ky = tap / kw, kx = tap - ky * kw;
            const int iy = oy * stride + ky - pad_y, ix = ox * stride + kx - pad_x;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
                v = in[((n * H + iy) * (int64_t)W + ix) * Ct + c0 + c];
                if (scale) v *= scale[n * Cg + c];
            }
        }
        out[i] = v;
    }
};
struct Im2col4K {      // items = P*KP/4 (one float4 each); needs Cg, c0, Ct multiples of 4
    const float* in; const float* scale; float* out;
    int H, W, Ct, c0, Cg, kh, kw, stride, pad_y, pad_x, OH, OW, KP;
    CK_HD void operator()(int64_t i) const {
        const int kq = KP >> 2;
        const int k = (int)(i % kq) * 4; const int64_t p = i / kq;
        const int ox = (int)(p % OW); const int64_t t = p / OW;
        const int oy = (int)(t % OH); const int64_t n = t / OH;
        f4 v = {0.f, 0.f, 0.f, 0.f};
        if (k < kh * kw * Cg) {
            const int tap = k / Cg, c = k - tap * Cg;
            const int ky = tap / kw, kx = tap - ky * kw;
            const int iy = oy * stride + ky - pad_y, ix = ox * stride + kx - pad_x;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
                v = ld4(in + ((n * H + iy) * (int64_t)W + ix) * Ct + c0 + c);
                if (scale) {
                    const f4 s = ld4(scale + n * Cg + c);
                    v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
                }
            }
        }
        st4(out + p * KP + k, v);
    }
};

// Same gather, written as the fp16 hi / lo pair of v * a_scale (v*a_scale ~= hi + lo, 22 significant bits): the A operand
// of the wgmma GEMM (sepconv_tc.cu, A_TMA mode), K-major rows of KP halves (KP a multiple of 64).
struct Im2colSplit4K { // items = P*KP/4; needs Cg, c0, Ct multiples of 4
    const float* in; const float* scale; ck_half* hi; ck_half* lo; float a_scale;
    int H, W, Ct, c0, Cg, kh, kw, stride, pad_y, pad_x, OH, OW, KP;
    CK_HD void operator()(int64_t i) const {
        const int kq = KP >> 2;
        const int k = (int)(i % kq) * 4; const int64_t p = i / kq;
        const int ox = (int)(p % OW); const int64_t t = p / OW;
        const int oy = (int)(t % OH); const int64_t n = t / OH;
        f4 v = {0.f, 0.f, 0.f, 0.f};
        if (k < kh * kw * Cg) {
            const int tap = k / Cg, c = k - tap * Cg;
            const int ky = tap / kw, kx = tap - ky * kw;
            const int iy = oy * stride + ky - pad_y, ix = ox * stride + kx - pad_x;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
                v = ld4(in + ((n * H + iy) * (int64_t)W + ix) * Ct + c0 + c);
                if (scale) {
                    const f4 s = ld4(scale + n * Cg + c);
                    v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
                }
            }
        }
        v.x *= a_scale; v.y *= a_scale; v.z *= a_scale; v.w *= a_scale;
        h4 h = {ck_f2h(v.x), ck_f2h(v.y), ck_f2h(v.z), ck_f2h(v.w)};
        h4 l = {ck_f2h(v.x - ck_h2f(h.x)), ck_f2h(v.y - ck_h2f(h.y)), ck_f2h(v.z - ck_h2f(h.z)), ck_f2h(v.w - ck_h2f(h.w))};
        *reinterpret_cast<h4*>(hi + p * KP + k) = h;
        *reinterpret_cast<h4*>(lo + p * KP + k) = l;
    }
};

// ---- transposed convolution, second half: gather the per-input-pixel products G[p_in][(ky*kw+kx)*Cout + co] -------
// (G = X * Bt, one GEMM with no wasted MACs -- or one GEMM per tap, see tap_stride) into out[n][y][x][co],
// y = iy*stride + ky - pt  (F.conv_transpose2d).
struct Col2imTK {      // items = n*OH*OW*Cout
    const float* g; float* out;
    int64_t tap_stride;   // elements between the products of consecutive taps: Cout (one GEMM, columns (tap, co)) or rows*NP (one GEMM per tap)
    int H, W, Cout, NP, kh, kw, stride, pt_y, pt_x, OH, OW, Ct, c0;   // out has Ct channels, this group writes [c0, c0+Cout)
    CK_HD void operator()(int64_t i) const {
        const int co = (int)(i % Cout); int64_t t = i / Cout;
        const int x = (int)(t % OW); t /= OW;
        const int y = (int)(t % OH); const int64_t n = t / OH;
        float acc = 0.f;
        for (int ky = 0; ky < kh; ++ky) {
            const int Y = y + pt_y - ky;
            if (Y < 0 || Y % stride) continue;
            const int iy = Y / stride;
            if (iy >= H) continue;
            for (int kx = 0; kx < kw; ++kx) {
                const int X = x + pt_x - kx;
                if (X < 0 || X % stride) continue;
                const int ix = X / stride;
                if (ix >= W) continue;
                acc += g[((n * H + iy) * (int64_t)W + ix) * NP + (ky * kw + kx) * tap_stride + co];
            }
        }
        out[((n * OH + y) * (int64_t)OW + x) * Ct + c0 + co] = acc;
    }
};

// ---- upfirdn2d on NHWC data (torch_utils/ops/upfirdn2d.py:169-208 semantics) -------------------------------------
// out[oy][ox] = sum f[fy][fx] * xpad[oy*down + fy][ox*down + fx]; xpad = zero-inserted (x up) input shifted by the
// (possibly negative) padding.  f is passed ALREADY flipped (true convolution) and multiplied by the gain.
struct UpfirdnNhwcK {  // items = n*OH*OW*C
    const float* in; float* out; const float* add;   // add (nullable): same shape as out, summed in
    float f[64]; int fh, fw;
    int H, W, C, up, down, pad_y0, pad_x0, OH, OW;
    CK_HD void operator()(int64_t i) const {
        const int c = (int)(i % C); int64_t t = i / C;
        const int ox = (int)(t % OW); t /= OW;
        const int oy = (int)(t % OH); const int64_t n = t / OH;
        float acc = 0.f;
        for (int fy = 0; fy < fh; ++fy) {
            const int Y = oy * down + fy - pad_y0;
            if (Y < 0 || Y % up) continue;
            const int iy = Y / up;
            if (iy >= H) continue;
            for (int fx = 0; fx < fw; ++fx) {
                const int X = ox * down + fx - pad_x0;
                if (X < 0 || X % up) continue;
                const int ix = X / up;
                if (ix >= W) continue;
                acc += f[fy * fw + fx] * in[((n * H + iy) * (int64_t)W + ix) * C + c];
            }
        }
        if (add) acc += add[i];
        out[i] = acc;
    }
};

// ---- GEMM epilogue: demodulation, noise, bias, lrelu_agc(gain), skip add -----------------------------------------
// v = g[p][o] (* dcoef[n][o]) (+ noise[n*noise_stride_n + hw] * noise_strength) (+ bias[o]);
// act: v = leaky_relu(v, alpha);  v *= gain;  clamp >= 0: v = clamp(v, +-clamp);  (+ add[p][o])     (stylegan.py:300-310,
// common/utils.py:114-122).  out may alias g when NP == Cout and the channel window is the whole tensor.
struct EpilogueK {     // items = P*Cout
    const float* g; float* out; const float* dcoef; const float* noise; const float* bias; const float* add;
    int64_t noise_stride_n; float noise_strength;
    int HW, Cout, NP, Ct, c0;     // out has Ct channels; this call writes [c0, c0+Cout)
    int act; float alpha, gain, clamp;
    CK_HD void operator()(int64_t i) const {
        const int o = (int)(i % Cout); const int64_t p = i / Cout;
        const int64_t n = p / HW; const int hw = (int)(p % HW);
        float v = g[p * NP + o];
        if (dcoef) v *= dcoef[n * Cout + o];
        if (noise) v += noise[n * noise_stride_n + hw] * noise_strength;
        if (bias) v += bias[o];
        if (act) v = v < 0.f ? v * alpha : v;
        v *= gain;
        if (clamp >= 0.f) v = fminf(fmaxf(v, -clamp), clamp);
        const int64_t oi = p * Ct + c0 + o;
        if (add) v += add[oi];
        out[oi] = v;
    }
};

// ---- weight packing (device side, so the op-level entry point can take device OIHW weights) ----------------------
// Bt[k][o], k = (ky*kw + kx)*Cg + ci, o < Cout_g:  w[o0 + o][ci][ky'][kx'] * oscale[o0 + o] * gain,
// (ky', kx') mirrored when flip (true convolution, conv2d_resample.py:34-35); zero in the K / N padding.
struct PackWeightK {   // items = KP*NP
    const float* w; const float* oscale; float* out;
    int Cg, kh, kw, o0, Cout_g, KP, NP, flip; float gain;
    CK_HD void operator()(int64_t i) const {
        const int o = (int)(i % NP); const int k = (int)(i / NP);
        float v = 0.f;
        if (o < Cout_g && k < kh * kw * Cg) {
            const int tap = k / Cg, ci = k - tap * Cg;
            int ky = tap / kw, kx = tap - ky * kw;
            if (flip) { ky = kh - 1 - ky; kx = kw - 1 - kx; }
            v = w[(((int64_t)(o0 + o) * Cg + ci) * kh + ky) * kw + kx] * gain;
            if (oscale) v *= oscale[o0 + o];
        }
        out[i] = v;
    }
};
// Transposed-convolution operand: Bt[ci][(ky*kw + kx)*Cout_g + co] = w[o0 + co][ci][ky'][kx'] * oscale * gain.
struct PackWeightTK {  // items = KP*NP, KP >= Cg, NP >= kh*kw*Cout_g
    const float* w; const float* oscale; float* out;
    int Cg, kh, kw, o0, Cout_g, KP, NP, flip; float gain;
    CK_HD void operator()(int64_t i) const {
        const int j = (int)(i % NP); const int ci = (int)(i / NP);
        float v = 0.f;
        if (ci < Cg && j < kh * kw * Cout_g) {
            const int tap = j / Cout_g, co = j - tap * Cout_g;
            int ky = tap / kw, kx = tap - ky * kw;
            if (flip) { ky = kh - 1 - ky; kx = kw - 1 - kx; }
            v = w[(((int64_t)(o0 + co) * Cg + ci) * kh + ky) * kw + kx] * gain;
            if (oscale) v *= oscale[o0 + co];
        }
        out[i] = v;
    }
};

// ---- small per-sample vectors (mapping network, styles, demodulation) --------------------------------------------
struct RowRmsNormK {   // items = n: out[n][:] = x[n][:] * rsqrt(mean(x[n][:]^2) + eps)       (stylegan.py:351-352)
    const float* in; float* out; int D; float eps;
    CK_HD void operator()(int64_t n) const {
        float s = 0.f;
        for (int d = 0; d < D; ++d) { const float v = in[n * D + d]; s += v * v; }
        const float r = 1.f / sqrtf(s / (float)D + eps);
        for (int d = 0; d < D; ++d) out[n * D + d] = in[n * D + d] * r;
    }
};
struct InvRmsAllK {    // items = 1: out[0] = rsqrt(mean(x^2)) over count elements              (stylegan.py:146)
    const float* in; float* out; int64_t count;
    CK_HD void operator()(int64_t) const {
        float s = 0.f;
        for (int64_t j = 0; j < count; ++j) s += in[j] * in[j];
        out[0] = 1.f / sqrtf(s / (float)count);
    }
};
struct ScaleK {        // items = count: out = in * mul * (norm ? norm[0] : 1)
    const float* in; const float* norm; float* out; float mul;
    CK_HD void operator()(int64_t i) const { out[i] = in[i] * mul * (norm ? norm[0] : 1.f); }
};
struct DcoefK {        // items = n*O: d[n][o] = rsqrt(sum_i s[n][i]^2 * wsq[i][o] + 1e-8)       (stylegan.py:154)
    const float* s; const float* wsq; float* out; int I, O;
    CK_HD void operator()(int64_t i) const {
        const int o = (int)(i % O); const int64_t n = i / O;
        float acc = 0.f;
        for (int c = 0; c < I; ++c) { const float v = s[n * I + c]; acc += v * v * wsq[(int64_t)c * O + o]; }
        out[i] = 1.f / sqrtf(acc + 1e-8f);
    }
};
struct LerpK {         // items = n*D: out = avg + psi * (w - avg)                               (stylegan.py:433-437)
    const float* w; const float* avg; float* out; int D; float psi;
    CK_HD void operator()(int64_t i) const { const float a = avg[i % D]; out[i] = a + psi * (w[i] - a); }
};
struct ConcatK {       // items = n*(Da+Db): out[n] = [a[n] | b[n]]                              (comodgan.py:252,325)
    const float* a; const float* b; float* out; int Da, Db;
    CK_HD void operator()(int64_t i) const {
        const int D = Da + Db; const int d = (int)(i % D); const int64_t n = i / D;
        out[i] = d < Da ? a[n * Da + d] : b[n * Db + d - Da];
    }
};

}  // namespace comod

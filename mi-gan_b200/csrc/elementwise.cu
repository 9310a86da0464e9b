// CUDA-core kernels of the MI-GAN generator forward (sm_90a): everything that is not the
// 1x1 pointwise contraction.  All are HBM-bound streaming kernels: NHWC fp32, one 128-bit
// vector of 4 channels per thread so that a warp touches whole 128-byte lines.
//
// Reference semantics (lib/model_zoo/migan_inference.py):
//   stem      : EncoderBlock.fromrgb + activation                       :193-196
//   dw3x3     : SeparableConv2d.conv1 (depthwise, pad 1) + activation    :155-157
//   dw3x3_down: the same followed by Downsample2d (4x4, stride 2, pad 1) :159-160, :62-76
//   up2       : Upsample2d (zero insertion, pad (2,1,2,1), 4x4 FIR) + noise + activation,
//               then the decoder skip add                                :98-103, :165-169, :304-305
//   torgb     : SynthesisBlock torgb 1x1 + Upsample2d of the image + add :308-313
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace migan {

static inline unsigned blocks_for(int64_t items, int threads) {
    return (unsigned)((items + threads - 1) / threads);
}

// --------------------------------------------------------------------------------------
// stem: x NCHW [n,4,H,W] -> NHWC [n,H,W,C0]
// --------------------------------------------------------------------------------------
// All spatial sizes and channel counts are powers of two: index math is 32-bit shifts/masks
// (64-bit div/mod costs ~100 instructions per thread and dominated these kernels otherwise).
__device__ __forceinline__ int ilog2(int v) { return 31 - __clz(v); }

// Thread = (4 output channels, 4 adjacent pixels): the 4x4 weights + bias stay in registers, x is read as one
// 128-bit load per input plane, and the thread writes four 128-bit vectors (each warp instruction covers whole
// 256-byte pixel rows).  Re-loading the weights per output vector would saturate the L1 instead of HBM.
__global__ void __launch_bounds__(256)
stem_fromrgb_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                    float* __restrict__ out, uint32_t items, int lhw, int lcv) {
    pdl_trigger();
    pdl_wait();
    const uint32_t idx = blockIdx.x * 256u + threadIdx.x;     // over (pixel quads) x (channel quads)
    if (idx >= items) return;
    const uint32_t c4 = idx & ((1u << lcv) - 1);
    const uint32_t pq = idx >> lcv;                           // pixel-quad index over the image group
    const uint32_t p = pq << 2;
    const uint32_t q = p & ((1u << lhw) - 1);
    const uint32_t img = p >> lhw;
    const size_t HW = (size_t)1 << lhw;
    const float* xp = x + (size_t)img * 4 * HW + q;
    const float4 x0 = ldg4(xp), x1 = ldg4(xp + HW), x2 = ldg4(xp + 2 * HW), x3 = ldg4(xp + 3 * HW);
    float4 wc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) wc[j] = ldg4(w + (c4 * 4 + j) * 4);
    const float4 bv = ldg4(b + c4 * 4);
    const float bj[4] = {bv.x, bv.y, bv.z, bv.w};
    const float px[4][4] = {{x0.x, x1.x, x2.x, x3.x}, {x0.y, x1.y, x2.y, x3.y}, {x0.z, x1.z, x2.z, x3.z}, {x0.w, x1.w, x2.w, x3.w}};
    float* op = out + ((size_t)p << (lcv + 2)) + c4 * 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v = wc[j].x * px[i][0];
            v = fmaf(wc[j].y, px[i][1], v);
            v = fmaf(wc[j].z, px[i][2], v);
            v = fmaf(wc[j].w, px[i][3], v);
            o[j] = lrelu_agc(v + bj[j]);
        }
        stg4(op + ((size_t)i << (lcv + 2)), make_float4(o[0], o[1], o[2], o[3]));
    }
}

// Launch helper: split the batch so that one launch indexes < 2^31 work items.
template <typename F>
static cudaError_t for_image_groups(int n, size_t items_per_image, F&& launch) {
    const int max_imgs = (int)std::max<size_t>(1, ((size_t)1 << 31) / std::max<size_t>(items_per_image, 1));
    for (int i0 = 0; i0 < n; i0 += max_imgs) {
        launch(i0, std::min(max_imgs, n - i0));
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

static inline int host_log2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

cudaError_t launch_stem(const float* x, const float* w, const float* b, float* out,
                        int n, int H, int W, int C0, cudaStream_t s) {
    const size_t per_img = (size_t)H * W / 4 * (C0 / 4);
    return for_image_groups(n, per_img, [&](int i0, int cnt) {
        const uint32_t items = (uint32_t)(per_img * cnt);
        launch_pdl(stem_fromrgb_kernel, dim3((items + 255) / 256), dim3(256), 0, s, x + (size_t)i0 * 4 * H * W, w, b, out + (size_t)i0 * H * W * C0,
                   items, host_log2(H * W), host_log2(C0 / 4));
    });
}

// --------------------------------------------------------------------------------------
// depthwise 3x3 + bias + act, NHWC -> NHWC (used by the CUDA-core path; the wgmma path
// fuses this stage into the GEMM prologue)
// --------------------------------------------------------------------------------------
typedef unsigned long long u64;
__device__ __forceinline__ u64 pk2(float lo, float hi) {
    u64 d;
    asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(__float_as_uint(lo)), "r"(__float_as_uint(hi)));
    return d;
}
__device__ __forceinline__ float2 unpk2(u64 v) {
    uint32_t lo, hi;
    asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
    return make_float2(__uint_as_float(lo), __uint_as_float(hi));
}
__device__ __forceinline__ u64 ffma2(u64 a, u64 b, u64 c) {
    const float2 x = unpk2(a), y = unpk2(b), z = unpk2(c);
    return pk2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ u64 ldg2(const float* p) { return __ldg(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ u64 fmul2(u64 a, u64 b) {
    const float2 x = unpk2(a), y = unpk2(b);
    return pk2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
// lrelu_agc on a channel pair, bit-identical to the scalar form: max(v, 0.2 v) == leaky_relu(v) exactly,
// then * sqrt2 and clamp.
__device__ __forceinline__ u64 lrelu_agc2(u64 v) {
    const float2 a = unpk2(v), b = unpk2(fmul2(v, pk2(kLreluAlpha, kLreluAlpha)));
    const float2 m = unpk2(fmul2(pk2(fmaxf(a.x, b.x), fmaxf(a.y, b.y)), pk2(kActGain, kActGain)));
    return pk2(fminf(fmaxf(m.x, -kActClamp), kActClamp), fminf(fmaxf(m.y, -kActClamp), kActClamp));
}

// Thread = (channel PAIR, PAIR of adjacent columns x0 = 2*xp, x0 + 1, strip of RS rows): the 9 taps + bias stay in
// registers, a 3-row x 4-column window slides down the strip (4 L1-served 64-bit loads per row feed 2 outputs),
// all MACs are FFMAs on channel pairs, and the next row is fetched one iteration ahead.
template <int RS>
__global__ void __launch_bounds__(256)
dw3x3_act_kernel(const float* __restrict__ in, const float* __restrict__ w9, const float* __restrict__ bias,
                 float* __restrict__ out, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                 uint32_t items, int lw, int lh, int lcp, int lstrips) {
    pdl_trigger();
    pdl_wait();
    const uint32_t idx = blockIdx.x * 256u + threadIdx.x;
    if (idx >= items) return;
    const int W = 1 << lw, H = 1 << lh, C = 2 << lcp;
    const int c = (int)(idx & ((1u << lcp) - 1)) * 2;
    uint32_t t = idx >> lcp;
    const int x0 = (int)(t & ((W >> 1) - 1)) * 2;
    t >>= (lw - 1);
    const int strip = (int)(t & ((1u << lstrips) - 1));
    const size_t img = t >> lstrips;
    const int y0 = strip * RS;
    u64 w[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) w[k] = ldg2(w9 + k * C + c);
    const u64 bv = ldg2(bias + c);
    const float* base = in + img * (size_t)H * W * C + c;
    const bool okl = x0 > 0, okr = x0 + 2 < W;
    auto load_row = [&](int y, u64 (&r)[4]) {
        if (y < 0 || y >= H) { r[0] = r[1] = r[2] = r[3] = 0ull; return; }
        const float* p = base + ((size_t)y * W + x0) * C;
        r[0] = okl ? ldg2(p - C) : 0ull;
        r[1] = ldg2(p);
        r[2] = ldg2(p + C);
        r[3] = okr ? ldg2(p + 2 * C) : 0ull;
    };
    u64 r0[4], r1[4], r2[4], rn[4];
    load_row(y0 - 1, r0);
    load_row(y0, r1);
    load_row(y0 + 1, r2);
#pragma unroll
    for (int i = 0; i < RS; ++i) {
        const int y = y0 + i;
        if (i + 1 < RS) load_row(y + 2, rn);              // next iteration's bottom row: issued one iteration ahead
#pragma unroll
        for (int e = 0; e < 2; ++e) {                     // the two output columns
            u64 acc = bv;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                acc = ffma2(w[d], r0[e + d], acc);
                acc = ffma2(w[3 + d], r1[e + d], acc);
                acc = ffma2(w[6 + d], r2[e + d], acc);
            }
            const float2 v = unpk2(lrelu_agc2(acc));
            const size_t o = ((img * H + y) * (size_t)W + x0 + e) * C + c;
            if (out) *reinterpret_cast<float2*>(out + o) = v;
            if (out_hi) {   // pre-split A operand for the wgmma GEMM (layers whose Cout spans several CTA N tiles)
                __half h0, l0, h1, l1;
                split_f16(v.x, kActSplitScale, h0, l0);
                split_f16(v.y, kActSplitScale, h1, l1);
                *reinterpret_cast<__half2*>(out_hi + o) = __halves2half2(h0, h1);
                *reinterpret_cast<__half2*>(out_lo + o) = __halves2half2(l0, l1);
            }
        }
#pragma unroll
        for (int d = 0; d < 4; ++d) { r0[d] = r1[d]; r1[d] = r2[d]; r2[d] = rn[d]; }
    }
}

cudaError_t launch_dw3x3(const float* in, const float* w9, const float* bias, float* out, __half* out_hi, __half* out_lo,
                         int n, int H, int W, int C, cudaStream_t s) {
    const int rs = (H >= 8) ? 8 : 4, strips = H / rs;
    const size_t per_img = (size_t)strips * (W / 2) * (C / 2);
    return for_image_groups(n, per_img, [&](int i0, int cnt) {
        const uint32_t items = (uint32_t)(per_img * cnt);
        const size_t off = (size_t)i0 * H * W * C;
        auto kern = (rs == 8) ? dw3x3_act_kernel<8> : dw3x3_act_kernel<4>;
        launch_pdl(kern, dim3((items + 255) / 256), dim3(256), 0, s, in + off, w9, bias, out ? out + off : nullptr, out_hi ? out_hi + off : nullptr,
                   out_lo ? out_lo + off : nullptr, items, host_log2(W), host_log2(H), host_log2(C / 2), host_log2(strips));
    });
}

// --------------------------------------------------------------------------------------
// depthwise 3x3 + bias + act + FIR 4x4 / stride 2 / pad 1 (SeparableConv2d.conv1 + Downsample2d).
//
// Thread = (channel PAIR, low-res column ox, strip of RS low-res rows).  It walks down the hi-res
// input rows once, keeping a rolling 3-row x 6-column window in registers (L1-served 64-bit loads,
// a warp reads 256 contiguous bytes per pixel), evaluates each activated depthwise value of its 4
// columns exactly once per row and scatters it into the two FIR accumulators it contributes to
// (rows 2oy-1..2oy+2 feed output oy).  All MACs are FFMAs on channel pairs.
// Depthwise outputs outside the image are ZERO (the FIR zero-pads the ACTIVATED tensor,
// migan_inference.py:62-70), not act(bias).
// --------------------------------------------------------------------------------------
// RS = low-res rows per thread (template: the row walk is fully unrolled).  Thread = (channel pair, PAIR of adjacent
// low-res columns ox0 = 2*oxp, ox0 + 1, strip of RS rows).  Register plan per thread:
//   v[8]       the current input row (columns 2ox0-2 .. 2ox0+5), fetched one row ahead (software pipelining)
//   dw[3][6]   partial depthwise sums of the three depthwise rows the current input row touches; the two middle
//              depthwise columns feed both outputs, so every activated depthwise value is computed exactly once
//              horizontally (the one-column version evaluated each column in two threads)
//   w[9], bias per-channel-pair constants; FIR taps from a shared-memory table; 8 column pointers advanced per row
template <int RS>
__global__ void __launch_bounds__(256, 2)
dw3x3_down_kernel(const float* __restrict__ in, const float* __restrict__ w9, const float* __restrict__ bias,
                  const float* __restrict__ fir16, float* __restrict__ out_f32,
                  __half* __restrict__ out_hi, __half* __restrict__ out_lo, uint32_t items, int lw2, int lh2, int lcp, int lstrips) {
    const uint32_t idx = blockIdx.x * 256u + threadIdx.x;
    const int W2 = 1 << lw2, H2 = 1 << lh2, W = 2 * W2, H = 2 * H2, C = 2 << lcp;
    const int c = (int)(idx & ((1u << lcp) - 1)) * 2;
    uint32_t t = idx >> lcp;
    const int ox0 = (int)(t & ((W2 >> 1) - 1)) * 2;
    t >>= (lw2 - 1);
    const int strip = (int)(t & ((1u << lstrips) - 1));
    const size_t img = t >> lstrips;
    const int oy0 = strip * RS;

    // FIR taps live in shared memory ([16][C], conflict-free 64-bit reads along the channel pairs)
    extern __shared__ float s_fir[];
    for (int i = threadIdx.x; i < 16 * C; i += 256) s_fir[i] = __ldg(fir16 + i);
    __syncthreads();
    if (idx >= items) return;
    const u64* firp = reinterpret_cast<const u64*>(s_fir + c);
    const int fstride = C >> 1;                           // u64 elements between taps
    u64 wv[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wv[k] = ldg2(w9 + k * C + c);
    const u64 bv = ldg2(bias + c);

    const int iy_first = 2 * oy0 - 2;
    const float* colp[8];
    bool colok[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int ix = 2 * ox0 - 2 + j;
        colok[j] = (ix >= 0 && ix < W);
        colp[j] = in + ((img * H + iy_first) * (size_t)W + (colok[j] ? ix : 0)) * C + c;   // only dereferenced when valid
    }
    const size_t row_stride = (size_t)W * C;
    bool dwok[6];
#pragma unroll
    for (int tx = 0; tx < 6; ++tx) dwok[tx] = (2 * ox0 - 1 + tx >= 0) && (2 * ox0 - 1 + tx < W);

    u64 dw[3][6];
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2)
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[s2][tx] = bv;
    u64 accA[2] = {0ull, 0ull}, accB[2] = {0ull, 0ull};   // FIR accumulators of output rows k-1 / k, columns ox0 / ox0+1

    // input rows r = 0 .. 2RS+3 (iy = iy_first + r); input row r completes depthwise row gy = iy - 1 (q = r - 2)
    u64 vn[8];
    auto fetch_row = [&](int r) {
        const int iy = iy_first + r;
        const bool rowok = (iy >= 0 && iy < H);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            vn[j] = (rowok && colok[j]) ? ldg2(colp[j]) : 0ull;
            colp[j] += row_stride;
        }
    };
    fetch_row(0);
#pragma unroll
    for (int r = 0; r < 2 * RS + 4; ++r) {
        const int iy = iy_first + r;
        u64 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = vn[j];
        if (r + 1 < 2 * RS + 4) fetch_row(r + 1);
        // ky = 2 -> depthwise row iy-1 (slot (r+1)%3, completes), ky = 1 -> row iy (slot (r+2)%3), ky = 0 -> row iy+1 (slot r%3)
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                dw[(r + 1) % 3][tx] = ffma2(wv[6 + kx], v[tx + kx], dw[(r + 1) % 3][tx]);
                dw[(r + 2) % 3][tx] = ffma2(wv[3 + kx], v[tx + kx], dw[(r + 2) % 3][tx]);
                dw[r % 3][tx] = ffma2(wv[kx], v[tx + kx], dw[r % 3][tx]);
            }
        }
        if (r >= 2) {                                     // depthwise row gy = iy - 1 is complete
            const int q = r - 2;                          // gy = 2*oy0 - 1 + q
            const int gy = iy - 1;
            const int tyB = (q & 1) ? 1 : 0, tyA = tyB + 2;
            if (gy >= 0 && gy < H) {
#pragma unroll
                for (int tx = 0; tx < 6; ++tx) {
                    if (!dwok[tx]) continue;
                    const u64 d = lrelu_agc2(dw[(r + 1) % 3][tx]);
                    if (tx < 4) {                         // tap column tx of output ox0
                        accB[0] = ffma2(firp[(tyB * 4 + tx) * fstride], d, accB[0]);
                        accA[0] = ffma2(firp[(tyA * 4 + tx) * fstride], d, accA[0]);
                    }
                    if (tx >= 2) {                        // tap column tx-2 of output ox0+1
                        accB[1] = ffma2(firp[(tyB * 4 + tx - 2) * fstride], d, accB[1]);
                        accA[1] = ffma2(firp[(tyA * 4 + tx - 2) * fstride], d, accA[1]);
                    }
                }
            }
            if ((q & 1) && q >= 3) {                      // gy = 2k even: last tap of output row k-1 = oy0 + (q-3)/2
                const int orow = oy0 + ((q - 3) >> 1);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const size_t o = ((img * H2 + orow) * W2 + ox0 + e) * (size_t)C + c;
                    const float2 ov = unpk2(accA[e]);
                    if (out_f32) *reinterpret_cast<float2*>(out_f32 + o) = ov;
                    if (out_hi) {
                        __half h0, l0, h1, l1;
                        split_f16(ov.x, kActSplitScale, h0, l0);
                        split_f16(ov.y, kActSplitScale, h1, l1);
                        *reinterpret_cast<__half2*>(out_hi + o) = __halves2half2(h0, h1);
                        *reinterpret_cast<__half2*>(out_lo + o) = __halves2half2(l0, l1);
                    }
                }
            }
            if (q & 1) { accA[0] = accB[0]; accA[1] = accB[1]; accB[0] = 0ull; accB[1] = 0ull; }
        }
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[(r + 1) % 3][tx] = bv;   // slot is reused by depthwise row iy + 2
    }
}

cudaError_t configure_elementwise() { return cudaSuccess; }

cudaError_t launch_dw3x3_down(const float* in, const float* w9, const float* bias, const float* fir16,
                              float* out_f32, __half* out_hi, __half* out_lo,
                              int n, int H, int W, int C, cudaStream_t s) {
    const int H2 = H / 2, W2 = W / 2;
    const int rs = (H2 >= 8) ? 8 : 4, strips = H2 / rs;
    const size_t per_img = (size_t)strips * (W2 / 2) * (C / 2);
    return for_image_groups(n, per_img, [&](int i0, int cnt) {
        const uint32_t items = (uint32_t)(per_img * cnt);
        const size_t oi = (size_t)i0 * H * W * C, oo = (size_t)i0 * H2 * W2 * C;
        auto kern = (rs == 8) ? dw3x3_down_kernel<8> : dw3x3_down_kernel<4>;
        kern<<<(items + 255) / 256, 256, 16 * C * sizeof(float), s>>>(in + oi, w9, bias, fir16, out_f32 ? out_f32 + oo : nullptr,
                                                out_hi ? out_hi + oo : nullptr, out_lo ? out_lo + oo : nullptr,
                                                items, host_log2(W2), host_log2(H2), host_log2(C / 2), host_log2(strips));
    });
}

// --------------------------------------------------------------------------------------
// Tensor-core feed variant of the kernel above: same thread mapping and row walk, specialised for the pre-split fp16
// hi/lo output.  The generic kernel spends a large share of its instructions on address arithmetic (eight 64-bit column
// pointers, runtime C) and scalar min/max.  Here
//   * C is a template parameter: one row pointer, every column / tap offset is an immediate;
//   * the taps and bias arrive pre-multiplied by kActSplitScale * sqrt(2) (the table the wgmma prologue uses), so the
//     activation is clamp(max(v, 0.2 v), +-256 * 64) -- one multiply, two max and one min per value -- and
//     the FIR output is already scaled for the fp16 hi/lo split (the FIR is linear);
//   * two channels per thread, kept as float2 pairs.
// --------------------------------------------------------------------------------------
__device__ __forceinline__ float fmax3f(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float2 ffma2f(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2f(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

template <int RS, int C>
__global__ void __launch_bounds__(256, 2)
dw3x3_down_split_kernel(const float* __restrict__ in, const float* __restrict__ w9s, const float* __restrict__ biass,
                        const float* __restrict__ fir16, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                        uint32_t items, int lw2, int lh2, int lstrips) {
    constexpr int CP = C / 2;                              // channel pairs
    constexpr float kLim = kActClamp * kActSplitScale;
    const uint32_t idx = blockIdx.x * 256u + threadIdx.x;
    const int W2 = 1 << lw2, H2 = 1 << lh2, W = 2 * W2, H = 2 * H2;
    const int c = (int)(idx % CP) * 2;
    uint32_t t = idx / CP;
    const int ox0 = (int)(t & ((W2 >> 1) - 1)) * 2;
    t >>= (lw2 - 1);
    const int strip = (int)(t & ((1u << lstrips) - 1));
    const size_t img = t >> lstrips;
    const int oy0 = strip * RS;

    extern __shared__ float s_fir[];                       // [16][C]
    pdl_trigger();
    for (int i = threadIdx.x; i < 16 * C; i += 256) s_fir[i] = __ldg(fir16 + i);
    pdl_wait();                                            // the taps are weights; the input is the predecessor's output
    __syncthreads();
    if (idx >= items) return;
    const float2* firp = reinterpret_cast<const float2*>(s_fir + c);
    float2 wv[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wv[k] = __ldg(reinterpret_cast<const float2*>(w9s + k * C + c));
    const float2 bv = __ldg(reinterpret_cast<const float2*>(biass + c));

    const int iy_first = 2 * oy0 - 2;
    const bool left_ok = (ox0 > 0), right_ok = (ox0 + 2 < W2);            // columns 2ox0-2, 2ox0-1 / 2ox0+4, 2ox0+5 exist
    // one row pointer: column j of the 8-column window is at j * C floats (immediate offsets)
    const float* rowp = in + ((img * H + iy_first) * (size_t)W + (2 * ox0 - 2)) * C + c;
    const size_t row_stride = (size_t)W * C;

    float2 dw[3][6];
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2)
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[s2][tx] = bv;
    const float2 zero2 = make_float2(0.f, 0.f), alpha2 = make_float2(kLreluAlpha, kLreluAlpha);
    float2 accA[2] = {zero2, zero2}, accB[2] = {zero2, zero2};   // FIR accumulators of output rows k-1 / k, columns ox0 / ox0+1

    float2 vn[8];
    auto fetch_row = [&](int r) {
        const int iy = iy_first + r;
        const bool rowok = (iy >= 0 && iy < H);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const bool ok = rowok && (j >= 2 || left_ok) && (j < 6 || right_ok);
            vn[j] = ok ? __ldg(reinterpret_cast<const float2*>(rowp + j * C)) : zero2;
        }
        rowp += row_stride;
    };
    fetch_row(0);
#pragma unroll
    for (int r = 0; r < 2 * RS + 4; ++r) {
        const int iy = iy_first + r;
        float2 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = vn[j];
        if (r + 1 < 2 * RS + 4) fetch_row(r + 1);
        // ky = 2 -> depthwise row iy-1 (slot (r+1)%3, completes), ky = 1 -> row iy (slot (r+2)%3), ky = 0 -> row iy+1 (slot r%3)
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                dw[(r + 1) % 3][tx] = ffma2f(wv[6 + kx], v[tx + kx], dw[(r + 1) % 3][tx]);
                dw[(r + 2) % 3][tx] = ffma2f(wv[3 + kx], v[tx + kx], dw[(r + 2) % 3][tx]);
                dw[r % 3][tx] = ffma2f(wv[kx], v[tx + kx], dw[r % 3][tx]);
            }
        }
        if (r >= 2) {                                     // depthwise row gy = iy - 1 is complete
            const int q = r - 2;                          // gy = 2*oy0 - 1 + q
            const int gy = iy - 1;
            const int tyB = (q & 1) ? 1 : 0, tyA = tyB + 2;
            if (gy >= 0 && gy < H) {
#pragma unroll
                for (int tx = 0; tx < 6; ++tx) {
                    if ((tx == 0 && !left_ok) || (tx == 5 && !right_ok)) continue;   // depthwise column outside the image: zero
                    const float2 a = dw[(r + 1) % 3][tx], b = fmul2f(a, alpha2);
                    const float2 d = make_float2(fminf(fmax3f(a.x, b.x, -kLim), kLim), fminf(fmax3f(a.y, b.y, -kLim), kLim));
                    if (tx < 4) {                         // tap column tx of output ox0
                        accB[0] = ffma2f(firp[(tyB * 4 + tx) * CP], d, accB[0]);
                        accA[0] = ffma2f(firp[(tyA * 4 + tx) * CP], d, accA[0]);
                    }
                    if (tx >= 2) {                        // tap column tx-2 of output ox0+1
                        accB[1] = ffma2f(firp[(tyB * 4 + tx - 2) * CP], d, accB[1]);
                        accA[1] = ffma2f(firp[(tyA * 4 + tx - 2) * CP], d, accA[1]);
                    }
                }
            }
            if ((q & 1) && q >= 3) {                      // gy = 2k even: last tap of output row k-1 = oy0 + (q-3)/2
                const int orow = oy0 + ((q - 3) >> 1);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const size_t o = ((img * H2 + orow) * W2 + ox0 + e) * (size_t)C + c;
                    const float2 ov = accA[e];            // already * kActSplitScale
                    const __half2 h = __floats2half2_rn(ov.x, ov.y);
                    const float2 hf = __half22float2(h);
                    *reinterpret_cast<__half2*>(out_hi + o) = h;
                    *reinterpret_cast<__half2*>(out_lo + o) = __floats2half2_rn(ov.x - hf.x, ov.y - hf.y);
                }
            }
            if (q & 1) { accA[0] = accB[0]; accA[1] = accB[1]; accB[0] = zero2; accB[1] = zero2; }
        }
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[(r + 1) % 3][tx] = bv;   // slot is reused by depthwise row iy + 2
    }
}

template <int RS, int C>
static void launch_down_split_inst(const float* in, const float* w9s, const float* biass, const float* fir16, __half* hi, __half* lo,
                                   uint32_t items, int W2, int H2, int strips, cudaStream_t s) {
    launch_pdl(dw3x3_down_split_kernel<RS, C>, dim3((items + 255) / 256), dim3(256), 16 * C * sizeof(float), s, in, w9s, biass, fir16, hi, lo, items,
               host_log2(W2), host_log2(H2), host_log2(strips));
}

// w9s / biass: depthwise taps and bias * kActSplitScale * sqrt(2).  C in {64, 128, 256, 512}.
cudaError_t launch_dw3x3_down_split(const float* in, const float* w9s, const float* biass, const float* fir16,
                                    __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s) {
    const int H2 = H / 2, W2 = W / 2;
    if (W2 < 2 || (C != 64 && C != 128 && C != 256 && C != 512)) return cudaErrorInvalidValue;
    const int rs = (H2 >= 8) ? 8 : 4, strips = H2 / rs;
    if (strips < 1) return cudaErrorInvalidValue;
    const size_t per_img = (size_t)strips * (W2 / 2) * (C / 2);
    return for_image_groups(n, per_img, [&](int i0, int cnt) {
        const uint32_t items = (uint32_t)(per_img * cnt);
        const float* ip = in + (size_t)i0 * H * W * C;
        __half* hp = out_hi + (size_t)i0 * H2 * W2 * C;
        __half* lp = out_lo + (size_t)i0 * H2 * W2 * C;
#define MIGAN_DOWN_CASE(RS_, C_) launch_down_split_inst<RS_, C_>(ip, w9s, biass, fir16, hp, lp, items, W2, H2, strips, s)
        if (rs == 8) {
            if (C == 64) MIGAN_DOWN_CASE(8, 64); else if (C == 128) MIGAN_DOWN_CASE(8, 128);
            else if (C == 256) MIGAN_DOWN_CASE(8, 256); else MIGAN_DOWN_CASE(8, 512);
        } else {
            if (C == 64) MIGAN_DOWN_CASE(4, 64); else if (C == 128) MIGAN_DOWN_CASE(4, 128);
            else if (C == 256) MIGAN_DOWN_CASE(4, 256); else MIGAN_DOWN_CASE(4, 512);
        }
#undef MIGAN_DOWN_CASE
    });
}


// --------------------------------------------------------------------------------------
// TMA-staged variant of dw3x3_down_split: same arithmetic per thread, but the input rows come from a shared-memory ring
// that a producer warp fills with cp.async.bulk.tensor -- six rows (55 KB) in flight per block instead of one register row
// per thread, which keeps more loads in flight than the register-streaming kernel's low occupancy allows.  Block = (image, strip of RS low-res rows, 16 low-res columns, 64-channel slab): 256 compute threads
// (channel pair x column pair) + 1 producer warp.  Rows / columns outside the image arrive as zeros (TMA out-of-bounds
// fill), which is exactly the depthwise conv's zero padding.
// --------------------------------------------------------------------------------------
constexpr int kDownRing = 6;
constexpr int kDownRowBytes = 36 * 64 * 4;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool down_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void down_wait(uint32_t bar, uint32_t parity) {
    while (!down_try_wait(bar, parity)) {}
}

template <int RS>
__global__ void __launch_bounds__(288, 2)
dw3x3_down_tma_kernel(const __grid_constant__ DownTensorMap desc, const float* __restrict__ w9s, const float* __restrict__ biass,
                      const float* __restrict__ fir16, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                      int C, int lw2, int lh2, int lstrips, int lslabs) {
    constexpr float kLim = kActClamp * kActSplitScale;
    constexpr int kRows = 2 * RS + 4;
    extern __shared__ __align__(128) unsigned char s_dyn[];
    __shared__ __align__(8) uint64_t s_bar[2 * kDownRing];
    float* s_fir = reinterpret_cast<float*>(s_dyn + kDownRing * kDownRowBytes);     // [16][64] taps of this slab
    const int W2 = 1 << lw2, H2 = 1 << lh2, H = 2 * H2;
    uint32_t b = blockIdx.x;
    const int slab = (int)(b & ((1u << lslabs) - 1)); b >>= lslabs;
    const int xtile = (int)(b & ((uint32_t)(W2 >> 4) - 1)); b >>= (lw2 - 4);
    const int strip = (int)(b & ((1u << lstrips) - 1));
    const int img = (int)(b >> lstrips);
    const int oy0 = strip * RS, iy_first = 2 * oy0 - 2;
    const int cs = slab * 64;
    const uint32_t bar0 = smem_addr(s_bar);
    if (threadIdx.x == 0) {
        for (int i = 0; i < kDownRing; ++i) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar0 + 8u * i), "r"(1));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar0 + 8u * (kDownRing + i)), "r"(8));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_trigger();
    for (int i = threadIdx.x; i < 16 * 64; i += 288) s_fir[i] = __ldg(fir16 + (i >> 6) * C + cs + (i & 63));
    pdl_wait();                                            // barriers and taps are set up under the predecessor's tail
    __syncthreads();

    if (threadIdx.x >= 256) {
        // ---- producer warp: one lane streams the rows of the slab window into the ring ----
        if (threadIdx.x == 256) {
            const uint64_t map = reinterpret_cast<uint64_t>(&desc);
            for (int r = 0; r < kRows; ++r) {
                const int st = r % kDownRing;
                if (r >= kDownRing) down_wait(bar0 + 8u * (kDownRing + st), ((r / kDownRing) - 1) & 1);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar0 + 8u * st), "r"(kDownRowBytes) : "memory");
                asm volatile(
                    "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                    ::"r"(smem_addr(s_dyn + st * kDownRowBytes)), "l"(map), "r"(bar0 + 8u * st),
                      "r"(cs), "r"(32 * xtile - 2), "r"(iy_first + r), "r"(img) : "memory");
            }
        }
        return;
    }

    // ---- compute threads: (channel pair, pair of low-res columns) ----
    const int c = (threadIdx.x & 31) * 2;                  // channel inside the slab
    const int oxp = threadIdx.x >> 5;                      // 0..7
    const int ox0 = xtile * 16 + 2 * oxp;
    const bool left_ok = (ox0 > 0), right_ok = (ox0 + 2 < W2);
    const float2* firp = reinterpret_cast<const float2*>(s_fir + c);
    float2 wv[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wv[k] = __ldg(reinterpret_cast<const float2*>(w9s + k * C + cs + c));
    const float2 bv = __ldg(reinterpret_cast<const float2*>(biass + cs + c));
    const unsigned char* win = s_dyn + (4 * oxp * 64 + c) * 4;      // window column j of ring slot st: win + st * kDownRowBytes + j * 256

    float2 dw[3][6];
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2)
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[s2][tx] = bv;
    const float2 zero2 = make_float2(0.f, 0.f), alpha2 = make_float2(kLreluAlpha, kLreluAlpha);
    float2 accA[2] = {zero2, zero2}, accB[2] = {zero2, zero2};

#pragma unroll
    for (int r = 0; r < kRows; ++r) {
        const int iy = iy_first + r;
        const int st = r % kDownRing;
        down_wait(bar0 + 8u * st, (r / kDownRing) & 1);
        float2 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const float2*>(win + st * kDownRowBytes + j * 256);
        if (r + kDownRing < kRows) {                         // slot is refilled later: release it once this warp has read it
            __syncwarp();
            if ((threadIdx.x & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar0 + 8u * (kDownRing + st)) : "memory");
        }
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                dw[(r + 1) % 3][tx] = ffma2f(wv[6 + kx], v[tx + kx], dw[(r + 1) % 3][tx]);
                dw[(r + 2) % 3][tx] = ffma2f(wv[3 + kx], v[tx + kx], dw[(r + 2) % 3][tx]);
                dw[r % 3][tx] = ffma2f(wv[kx], v[tx + kx], dw[r % 3][tx]);
            }
        }
        if (r >= 2) {                                     // depthwise row gy = iy - 1 is complete
            const int q = r - 2;
            const int gy = iy - 1;
            const int tyB = (q & 1) ? 1 : 0, tyA = tyB + 2;
            if (gy >= 0 && gy < H) {
#pragma unroll
                for (int tx = 0; tx < 6; ++tx) {
                    if ((tx == 0 && !left_ok) || (tx == 5 && !right_ok)) continue;   // depthwise column outside the image: zero
                    const float2 a = dw[(r + 1) % 3][tx], bb = fmul2f(a, alpha2);
                    const float2 d = make_float2(fminf(fmax3f(a.x, bb.x, -kLim), kLim), fminf(fmax3f(a.y, bb.y, -kLim), kLim));
                    if (tx < 4) {
                        accB[0] = ffma2f(firp[(tyB * 4 + tx) * 32], d, accB[0]);
                        accA[0] = ffma2f(firp[(tyA * 4 + tx) * 32], d, accA[0]);
                    }
                    if (tx >= 2) {
                        accB[1] = ffma2f(firp[(tyB * 4 + tx - 2) * 32], d, accB[1]);
                        accA[1] = ffma2f(firp[(tyA * 4 + tx - 2) * 32], d, accA[1]);
                    }
                }
            }
            if ((q & 1) && q >= 3) {
                const int orow = oy0 + ((q - 3) >> 1);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const size_t o = (((size_t)img * H2 + orow) * W2 + ox0 + e) * (size_t)C + cs + c;
                    const float2 ov = accA[e];
                    const __half2 h = __floats2half2_rn(ov.x, ov.y);
                    const float2 hf = __half22float2(h);
                    *reinterpret_cast<__half2*>(out_hi + o) = h;
                    *reinterpret_cast<__half2*>(out_lo + o) = __floats2half2_rn(ov.x - hf.x, ov.y - hf.y);
                }
            }
            if (q & 1) { accA[0] = accB[0]; accA[1] = accB[1]; accB[0] = zero2; accB[1] = zero2; }
        }
#pragma unroll
        for (int tx = 0; tx < 6; ++tx) dw[(r + 1) % 3][tx] = bv;
    }
}

cudaError_t launch_dw3x3_down_tma(const DownTensorMap& desc, const float* w9s, const float* biass, const float* fir16,
                                  __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s) {
    const int H2 = H / 2, W2 = W / 2;
    if (W2 < 16 || (W2 & (W2 - 1)) || C % 64 != 0) return cudaErrorInvalidValue;
    const int rs = (H2 >= 8) ? 8 : 4, strips = H2 / rs, slabs = C / 64;
    if (strips < 1 || (slabs & (slabs - 1))) return cudaErrorInvalidValue;
    const size_t blocks = (size_t)n * strips * (W2 / 16) * slabs;
    if (blocks == 0 || blocks > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    const size_t smem = (size_t)kDownRing * kDownRowBytes + 16 * 64 * sizeof(float);
    static bool attr_set[2] = {false, false};
    auto kern = (rs == 8) ? dw3x3_down_tma_kernel<8> : dw3x3_down_tma_kernel<4>;
    if (!attr_set[rs == 8]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr_set[rs == 8] = true;
    }
    return launch_pdl(kern, dim3((unsigned)blocks), dim3(288), smem, s, desc, w9s, biass, fir16, out_hi, out_lo, C, host_log2(W2), host_log2(H2),
                      host_log2(strips), host_log2(slabs));
}

// --------------------------------------------------------------------------------------
// 2x FIR up-sampling (polyphase: only the taps that meet a non-zero of the zero-inserted
// signal) + noise + act + skip.  out[o] = sum_t f[t] * z[o + t - 2], z[2i] = x[i], z[odd] = 0.
// --------------------------------------------------------------------------------------
// Thread = (low-res pixel, 4 channels) -> its 2x2 output pixels: 9 neighbour loads feed 4 outputs (instead of
// 4 loads per output) and the 16 per-channel taps come from a shared-memory table (instead of 4 global loads per output).
__global__ void __launch_bounds__(256)
up2_noise_act_skip_kernel(const float* __restrict__ t, const float* __restrict__ fir16,
                          const float* __restrict__ noise, const float* __restrict__ skip,
                          float* __restrict__ out, uint32_t items, int lw, int lh, int lcv) {
    extern __shared__ float4 s_taps[];                    // [16][C/4]
    const int w = 1 << lw, h = 1 << lh, W2 = 2 * w, C = 4 << lcv, CV = 1 << lcv;
    pdl_trigger();
    for (int i = threadIdx.x; i < 16 * CV; i += 256) s_taps[i] = ldg4(fir16 + i * 4);
    pdl_wait();
    __syncthreads();
    const uint32_t idx = blockIdx.x * 256u + threadIdx.x;
    if (idx >= items) return;
    const int cv = (int)(idx & (CV - 1));
    const uint32_t p = idx >> lcv;                        // low-res pixel index over the image group
    const int ix = (int)(p & (w - 1));
    const int iy = (int)((p >> lw) & (h - 1));
    const size_t img = p >> (lw + lh);
    const float* src = t + img * (size_t)h * w * C + cv * 4;
    float4 nb[3][3];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
            const int yy = iy + dy - 1, xx = ix + dx - 1;
            nb[dy][dx] = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? ldg4(src + ((size_t)yy * w + xx) * C)
                                                                   : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            // output (2iy+a, 2ix+b): taps ty = a, a+2 meet rows iy-1+a, iy+a ; tx = b, b+2 meet cols ix-1+b, ix+b
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int u = 0; u < 2; ++u)
#pragma unroll
                for (int v = 0; v < 2; ++v)
                    fma4(acc, s_taps[((a + 2 * u) * 4 + (b + 2 * v)) * CV + cv], nb[a + u][b + v]);
            const int oy = 2 * iy + a, ox = 2 * ix + b;
            if (noise) {
                const float nz = __ldg(noise + oy * W2 + ox);
                acc.x += nz; acc.y += nz; acc.z += nz; acc.w += nz;
            }
            acc = lrelu_agc4(acc);
            const size_t o = ((img * (size_t)(2 * h) + oy) * W2 + ox) * C + cv * 4;
            if (skip) {
                const float4 sk = ldg4(skip + o);
                acc.x += sk.x; acc.y += sk.y; acc.z += sk.z; acc.w += sk.w;
            }
            stg4(out + o, acc);
        }
}

cudaError_t launch_up2(const float* t, const float* fir16, const float* noise, const float* skip,
                       float* out, int n, int h, int w, int C, cudaStream_t s) {
    const size_t per_img = (size_t)h * w * (C / 4);
    return for_image_groups(n, per_img, [&](int i0, int cnt) {
        const uint32_t items = (uint32_t)(per_img * cnt);
        const size_t oi = (size_t)i0 * h * w * C, oo = (size_t)i0 * 4 * h * w * C;
        launch_pdl(up2_noise_act_skip_kernel, dim3((items + 255) / 256), dim3(256), 16 * C * sizeof(float), s,
                   t + oi, fir16, noise, skip ? skip + oo : nullptr, out + oo, items, host_log2(w), host_log2(h), host_log2(C / 4));
    });
}

// --------------------------------------------------------------------------------------
// torgb (C -> 3, with bias) + up-sampled previous image.  G lanes cooperate on one pixel
// (128-bit loads along C, warp-shuffle reduction), lane 0 of the group writes 3 planes.
// --------------------------------------------------------------------------------------
template <int G>
__global__ void __launch_bounds__(256)
torgb_img_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                 const float* __restrict__ img_lo, const float* __restrict__ fir, float* __restrict__ img_out,
                 int64_t npix, int r, int C) {
    pdl_trigger();
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int sub = lane % G;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t p = warp_global * (32 / G) + lane / G;
    const bool valid = p < npix;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (valid) {
        for (int c4 = sub; c4 < (C >> 2); c4 += G) {
            const float4 v = ldg4(x + p * C + c4 * 4);
            const float4 w0 = ldg4(w + c4 * 4), w1 = ldg4(w + C + c4 * 4), w2 = ldg4(w + 2 * C + c4 * 4);
            a0 = fmaf(v.x, w0.x, a0); a0 = fmaf(v.y, w0.y, a0); a0 = fmaf(v.z, w0.z, a0); a0 = fmaf(v.w, w0.w, a0);
            a1 = fmaf(v.x, w1.x, a1); a1 = fmaf(v.y, w1.y, a1); a1 = fmaf(v.z, w1.z, a1); a1 = fmaf(v.w, w1.w, a1);
            a2 = fmaf(v.x, w2.x, a2); a2 = fmaf(v.y, w2.y, a2); a2 = fmaf(v.z, w2.z, a2); a2 = fmaf(v.w, w2.w, a2);
        }
    }
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, off);
        a1 += __shfl_xor_sync(0xffffffffu, a1, off);
        a2 += __shfl_xor_sync(0xffffffffu, a2, off);
    }
    if (!valid || sub != 0) return;
    const int ox = (int)(p % r);
    const int oy = (int)((p / r) % r);
    const int64_t img = p / ((int64_t)r * r);
    float acc[3] = {a0 + __ldg(b), a1 + __ldg(b + 1), a2 + __ldg(b + 2)};
    if (img_lo) {
        const int h = r >> 1;
        float up[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            const int ty = (oy & 1) + 2 * a;
            const int iy = (oy + ty - 2) >> 1;
            if (iy < 0 || iy >= h) continue;
#pragma unroll
            for (int bb = 0; bb < 2; ++bb) {
                const int tx = (ox & 1) + 2 * bb;
                const int ix = (ox + tx - 2) >> 1;
                if (ix < 0 || ix >= h) continue;
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    up[k] = fmaf(__ldg(fir + (ty * 4 + tx) * 3 + k),
                                 __ldg(img_lo + ((img * 3 + k) * h + iy) * h + ix), up[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] = up[k] + acc[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) img_out[((img * 3 + k) * r + oy) * r + ox] = acc[k];
}

cudaError_t launch_torgb(const float* x, const float* w, const float* b, const float* img_lo,
                         const float* fir16x3, float* img_out, int n, int r, int C, cudaStream_t s) {
    const int64_t npix = (int64_t)n * r * r;
    if (C / 4 >= 32) {
        const int64_t threads = npix * 32;
        launch_pdl(torgb_img_kernel<32>, dim3(blocks_for(threads, 256)), dim3(256), 0, s, x, w, b, img_lo, fir16x3, img_out, npix, r, C);
    } else {
        const int64_t threads = npix * 16;
        launch_pdl(torgb_img_kernel<16>, dim3(blocks_for(threads, 256)), dim3(256), 0, s, x, w, b, img_lo, fir16x3, img_out, npix, r, C);
    }
    return cudaGetLastError();
}

// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
add_inplace_kernel(float* __restrict__ x, const float* __restrict__ y, int64_t n4) {
    pdl_trigger();
    pdl_wait();
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 a = reinterpret_cast<float4*>(x)[i];
    const float4 b = __ldg(reinterpret_cast<const float4*>(y) + i);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    reinterpret_cast<float4*>(x)[i] = a;
}

cudaError_t launch_add(float* x, const float* y, int64_t numel, cudaStream_t s) {
    launch_pdl(add_inplace_kernel, dim3(blocks_for(numel / 4, 256)), dim3(256), 0, s, x, y, numel / 4);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t total, int HW, int C) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // index into NCHW output
    if (i >= total) return;
    const int64_t q = i % HW;
    const int64_t c = (i / HW) % C;
    const int64_t img = i / ((int64_t)HW * C);
    out[i] = __ldg(in + (img * HW + q) * C + c);
}

cudaError_t launch_nhwc_to_nchw(const float* in, float* out, int n, int H, int W, int C, cudaStream_t s) {
    const int64_t total = (int64_t)n * H * W * C;
    nhwc_to_nchw_kernel<<<blocks_for(total, 256), 256, 0, s>>>(in, out, total, H * W, C);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
split_f16_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo, float scale, int64_t n4) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = __ldg(reinterpret_cast<const float4*>(in) + i);
    __half h[4], l[4];
    split_f16(v.x, scale, h[0], l[0]);
    split_f16(v.y, scale, h[1], l[1]);
    split_f16(v.z, scale, h[2], l[2]);
    split_f16(v.w, scale, h[3], l[3]);
    reinterpret_cast<uint2*>(hi)[i] = *reinterpret_cast<uint2*>(h);
    reinterpret_cast<uint2*>(lo)[i] = *reinterpret_cast<uint2*>(l);
}

cudaError_t launch_split_f16(const float* in, __half* hi, __half* lo, float scale, int64_t numel, cudaStream_t s) {
    split_f16_kernel<<<blocks_for(numel / 4, 256), 256, 0, s>>>(in, hi, lo, scale, numel / 4);
    return cudaGetLastError();
}

}  // namespace migan

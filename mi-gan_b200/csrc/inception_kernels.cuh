// Item kernels of the FID InceptionV3 forward and of the feature statistics (inception_abi.cu), in the style of
// comod_kernels.cuh: each functor produces output item i from global memory only and launches through ck_launch(), so
// the same code runs as a host loop in the emulation build (-DMIGAN_EMULATE).  The convolutions are not here: they are
// the tensor-core implicit GEMM of inception.cu.
//
// Layout: activations NHWC fp32 [n][H][W][C]; a functor that writes a channel slice takes the output's channel pitch
// ct and offset c0 (the concatenation of an Inception block's branches costs nothing).
#pragma once
#include <string.h>

#include "../../include/inception_b200.h"
#include "comod_kernels.cuh"

namespace incep {

using comod::f4;
using comod::ld4;
using comod::st4;

// ---- TF32 split of the convolution operands ---------------------------------------------------------------------
// hi = v with its low 13 mantissa bits cleared (a TF32 value, same exponent range as fp32), lo = v - hi (exact in
// fp32) rounded to the nearest TF32 value, ties away (cvt.rna.tf32.f32): hi + lo = v to about 2^-21 relative, and each
// product hi*hi, hi*lo, lo*hi of two TF32 values is exact in fp32.
CK_HD uint32_t f2u(float v) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(v);
#else
    uint32_t u; memcpy(&u, &v, 4); return u;
#endif
}
CK_HD float u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float v; memcpy(&v, &u, 4); return v;
#endif
}
CK_HD float tf32_trunc(float v) { return u2f(f2u(v) & 0xffffe000u); }
CK_HD float tf32_rna(float v) { return u2f((f2u(v) + 0x1000u) & 0xffffe000u); }
CK_HD void tf32_split(float v, float& hi, float& lo) {
    hi = tf32_trunc(v);
    lo = tf32_rna(v - hi);
}

// Packed weight operand of one convolution: K-major rows hi[o][k], lo[o][k] (NP x KP), k = (ky*kw + kx)*cinp + ci from
// w[cout][cin][kh][kw]; zero for ci >= cin (the first layer's 3 channels padded to 4), o >= cout and k >= kh*kw*cinp.
struct PackTf32K {     // items = NP*KP
    const float* w; float* hi; float* lo;
    int cin, cinp, cout, kh, kw, KP;
    CK_HD void operator()(int64_t i) const {
        const int k = (int)(i % KP), o = (int)(i / KP);
        float v = 0.f;
        const int tap = k / cinp, ci = k - tap * cinp;
        if (o < cout && tap < kh * kw && ci < cin) v = w[(((int64_t)o * cin + ci) * kh + tap / kw) * kw + tap % kw];
        float h, l;
        tf32_split(v, h, l);
        hi[i] = h;
        lo[i] = l;
    }
};

// ---- input stage: F.interpolate(x, (299, 299), mode="bilinear", align_corners=False), then 2x - 1 ---------------
// One output pixel (oy, ox) of an H x W image whose channel c at (y, x) is px(c, y, x), as NHWC {v0, v1, v2, 0}: channel
// 3 is zero (the first convolution reads 4-channel pixels).  Source index as ATen computes it in fp32:
// max(scale * (o + 0.5) - 0.5, 0), scale = in / out.  Both input layouts below evaluate this one expression, so an image
// gives the same bits through either when their loaders return the same floats.
//
// Every rounding is explicit (portable.cuh): these are the operations nvcc emits for the plain expression, FMAs where
// it contracts, and the ones ATen's CPU kernel performs, so the emulation build gives torch's CPU result bit for bit.
template <class Px>
CK_HD f4 bilinear_pixel(const Px& px, int H, int W, int OS, int oy, int ox) {
    const float sy = fmaxf(fma_rn(fdiv_rn((float)H, (float)OS), fadd_rn((float)oy, 0.5f), -0.5f), 0.f);
    const float sx = fmaxf(fma_rn(fdiv_rn((float)W, (float)OS), fadd_rn((float)ox, 0.5f), -0.5f), 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fminf(fmaxf(fsub_rn(sy, (float)y0), 0.f), 1.f), lx = fminf(fmaxf(fsub_rn(sx, (float)x0), 0.f), 1.f);
    const float hy = fsub_rn(1.f, ly), hx = fsub_rn(1.f, lx);
    float v[3];
    for (int c = 0; c < 3; ++c) {
        const float a = fma_rn(hx, px(c, y0, x0), fmul_rn(lx, px(c, y0, x1)));
        const float b = fma_rn(hx, px(c, y1, x0), fmul_rn(lx, px(c, y1, x1)));
        v[c] = fma_rn(fma_rn(hy, a, fmul_rn(ly, b)), 2.f, -1.f);
    }
    return f4{v[0], v[1], v[2], 0.f};
}

// fp32 NCHW [n][3][H][W] -> NHWC [n][299][299][4].
struct ResizeK {       // items = n*OS*OS
    const float* in; float* out; int H, W, OS;
    struct Px {
        const float* p; int64_t plane; int W;
        CK_HD float operator()(int c, int y, int x) const { return p[c * plane + (int64_t)y * W + x]; }
    };
    CK_HD void operator()(int64_t i) const {
        const int ox = (int)(i % OS); int64_t t = i / OS;
        const int oy = (int)(t % OS); const int64_t n = t / OS;
        const int64_t plane = (int64_t)H * W;
        st4(out + i * 4, bilinear_pixel(Px{in + n * 3 * plane, plane, W}, H, W, OS, oy, ox));
    }
};

// Decoded photos of any sizes, uint8 HWC RGB, packed one after the other in one buffer -> NHWC [n][299][299][4].  The
// loader is torchvision's ToTensor, v / 255 rounded once, so each photo's pixels equal ResizeK's on ToTensor(photo).
// Up to INCEPTION_U8_TABLE photos per launch; the table travels by value in the kernel parameter (batch_launch) with
// each photo's byte offset, its size and the launch's output item prefix: photo k owns items [start[k], start[k + 1]).
struct ResizeU8Batch {
    int64_t start[INCEPTION_U8_TABLE + 1];
    int64_t off[INCEPTION_U8_TABLE];
    int h[INCEPTION_U8_TABLE], w[INCEPTION_U8_TABLE];
    const uint8_t* photos; float* out;   // out: the first photo's output
    int n, OS;
};
static_assert(sizeof(ResizeU8Batch) <= 4000, "the photo table must fit the classic 4 KB kernel parameter space");

struct ResizeU8K {     // items = n*OS*OS
    const ResizeU8Batch& b;
    struct Px {
        const uint8_t* p; int W;
        CK_HD float operator()(int c, int y, int x) const {
            return fdiv_rn((float)p[((int64_t)y * W + x) * 3 + c], 255.f);
        }
    };
    CK_HD void operator()(int64_t i) const {
        const int k = comod::find_request(b.start, b.n, i);
        const int64_t j = i - b.start[k];
        const int ox = (int)(j % b.OS), oy = (int)(j / b.OS);
        st4(b.out + i * 4, bilinear_pixel(Px{b.photos + b.off[k], b.w[k]}, b.h[k], b.w[k], b.OS, oy, ox));
    }
};

// The table of photos [first, first + n) of a batch (n <= INCEPTION_U8_TABLE), writing y at the first one's output.
inline ResizeU8Batch u8_table(const uint8_t* photos, const int64_t* off, const int* h, const int* w, int first, int n,
                              float* y, int OS) {
    ResizeU8Batch b;
    b.photos = photos;
    b.out = y + (int64_t)first * OS * OS * 4;
    b.n = n;
    b.OS = OS;
    b.start[0] = 0;
    for (int k = 0; k < n; ++k) {
        b.off[k] = off[first + k];
        b.h[k] = h[first + k];
        b.w[k] = w[first + k];
        b.start[k + 1] = b.start[k] + (int64_t)OS * OS;
    }
    return b;
}

// ---- pools (3 x 3 windows) ------------------------------------------------------------------------------------------
// kind 0: max, stride 2, no padding (max_pool2d(3, 2)); 1: average, stride 1, padding 1, count_include_pad=False (the
// FID blocks' branch_pool); 2: max, stride 1, padding 1 (Mixed_7c's branch_pool; padding never wins a max).
// out[n][oy][ox][c0 + c] of a ct-channel tensor; C a multiple of 4.
struct PoolK {         // items = n*OH*OW*C/4
    const float* in; float* out; int kind, H, W, C, OH, OW, ct, c0;
    CK_HD void operator()(int64_t i) const {
        const int cq = C >> 2;
        const int c = (int)(i % cq) * 4; int64_t t = i / cq;
        const int ox = (int)(t % OW); t /= OW;
        const int oy = (int)(t % OH); const int64_t n = t / OH;
        const int s = kind == 0 ? 2 : 1, p = kind == 0 ? 0 : 1;
        const bool avg = kind == 1;
        f4 acc = avg ? f4{0.f, 0.f, 0.f, 0.f} : f4{-INFINITY, -INFINITY, -INFINITY, -INFINITY};
        int count = 0;
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * s - p + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * s - p + kx;
                if (ix < 0 || ix >= W) continue;
                const f4 v = ld4(in + ((n * H + iy) * (int64_t)W + ix) * C + c);
                if (avg) {
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                } else {
                    acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w);
                }
                ++count;
            }
        }
        if (avg) {
            const float d = (float)count;
            acc.x /= d; acc.y /= d; acc.z /= d; acc.w /= d;
        }
        st4(out + ((n * OH + oy) * (int64_t)OW + ox) * ct + c0 + c, acc);
    }
};

// adaptive_avg_pool2d(x, 1): out[n][c] = mean over the H*W pixels, summed in pixel order.
struct GlobalAvgK {    // items = n*C
    const float* in; float* out; int HW, C;
    CK_HD void operator()(int64_t i) const {
        const int c = (int)(i % C); const int64_t n = i / C;
        float s = 0.f;
        for (int p = 0; p < HW; ++p) s += in[(n * HW + p) * C + c];
        out[i] = s / (float)HW;
    }
};

// ---- feature statistics (float64) -------------------------------------------------------------------------------
struct StatsShiftK {   // items = dim: shift[d] = mean over the batch of x[:, d]
    const float* x; double* shift; int n, dim;
    CK_HD void operator()(int64_t d) const {
        double s = 0.0;
        for (int r = 0; r < n; ++r) s += (double)x[(int64_t)r * dim + d];
        shift[d] = s / n;
    }
};
// One entry of the rank-n update: sumsq[a][b] += sum_r (x[r][a] - shift[a]) (x[r][b] - shift[b]); the diagonal items
// also add sum[a].  Entries (a, b) and (b, a) see the same products in the same order: the result is exactly symmetric.
struct StatsUpdateK {  // items = dim*dim
    const float* x; const double* shift; double* sum; double* sumsq; int n, dim;
    CK_HD void operator()(int64_t i) const {
        const int a = (int)(i / dim), b = (int)(i % dim);
        const double sa = shift[a], sb = shift[b];
        double acc = 0.0, s1 = 0.0;
        for (int r = 0; r < n; ++r) {
            const double va = (double)x[(int64_t)r * dim + a] - sa, vb = (double)x[(int64_t)r * dim + b] - sb;
            acc += va * vb;
            s1 += va;
        }
        sumsq[i] += acc;
        if (a == b) sum[a] += s1;
    }
};


// The same two sums for each bin b of [nbins] over the rows r with bin[r] == b, in row order (a row whose bin is outside
// [0, nbins) is in none): the very operations StatsShiftK / StatsUpdateK perform on x[bin == b], and nothing for a bin
// with no row.  A bin's shift is set by the first call that gives it rows (count[b] == 0 before the call).
struct StatsShiftBinnedK {   // items = nbins*dim
    const float* x; const int* bin; const int64_t* count; double* shift; int n, dim;
    CK_HD void operator()(int64_t i) const {
        const int b = (int)(i / dim), d = (int)(i % dim);
        if (count[b] != 0) return;
        double s = 0.0;
        int c = 0;
        for (int r = 0; r < n; ++r) {
            if (bin[r] != b) continue;
            s += (double)x[(int64_t)r * dim + d];
            ++c;
        }
        if (c) shift[(int64_t)b * dim + d] = s / c;
    }
};
struct StatsUpdateBinnedK {  // items = nbins*dim*dim; item (b, 0, 0) also adds the bin's rows to count[b]
    const float* x; const int* bin; const double* shift; double* sum; double* sumsq; int64_t* count; int n, dim;
    CK_HD void operator()(int64_t i) const {
        const int64_t dd = (int64_t)dim * dim, e = i % dd;
        const int bn = (int)(i / dd), a = (int)(e / dim), b = (int)(e % dim);
        const double sa = shift[(int64_t)bn * dim + a], sb = shift[(int64_t)bn * dim + b];
        double acc = 0.0, s1 = 0.0;
        int c = 0;
        for (int r = 0; r < n; ++r) {
            if (bin[r] != bn) continue;
            const double va = (double)x[(int64_t)r * dim + a] - sa, vb = (double)x[(int64_t)r * dim + b] - sb;
            acc += va * vb;
            s1 += va;
            ++c;
        }
        if (!c) return;
        sumsq[i] += acc;
        if (a == b) sum[(int64_t)bn * dim + a] += s1;
        if (e == 0) count[bn] += c;
    }
};

}  // namespace incep

#ifndef MIGAN_EMULATE
namespace migan {
// One convolution on the tensor-core kernel (inception.cu): y[p][c0 + o] = relu(sum_k A[p][k] * B[o][k] + bias[o]) for
// o < cout, A gathered from x[n][H][W][cinp] (k = (ky*kw + kx)*cinp + ci, zero outside the image), B = bhi + blo.
struct IncepConvArgs {
    const float* x; const float* bhi; const float* blo; const float* bias; float* y;
    int n, H, W, cinp, OH, OW, kh, kw, stride, ph, pw, cout, KP, NP, ct, c0;
};
cudaError_t launch_incep_conv(const IncepConvArgs& a, cudaStream_t s);
}  // namespace migan
#endif

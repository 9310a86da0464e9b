// CUDA-core stages of the fused SeparableConv2d kernel (sepconv_tc.cu) that work on shared-memory tiles.
//
// Every function here is written against plain pointers into one pipeline stage of shared memory and takes the
// worker index `tg` (0..127: the thread's index inside its 128-thread prologue group) as an argument, with no
// barrier, shuffle or special register inside.  That is deliberate: the same source compiles as plain C++
// (-DMIGAN_EMULATE, tests/emul/build_stages.py) where a test loops tg = 0..127 over a host buffer filled the way
// the TMA unit fills the stage (box layout, out-of-bounds zero fill), so the halo / polyphase / swizzle index math is
// checked against the oracle on a machine without a GPU (tests/test_stages_emul.py).  The emulation build is TEST
// INFRASTRUCTURE; the product library is compiled without the macro.
//
// Stage layouts (one 32-channel chunk of one 8 x 16 output tile at origin (y0, x0), TMA boxes, no swizzle):
//   IN   [10 rows][18 cols][32 ch] fp32   rows y0-1 .. y0+8, cols x0-1 .. x0+16: the depthwise conv's input + halo
//   T    [ 6 rows][10 cols][32 ch] fp32   UP: raw 1x1 output of the up-sampling layer, rows y0/2-1 .. y0/2+4
//   NZ   [10 rows][24 cols]        fp32   UP: noise map rows y0-1 .. y0+8, cols x0-4 .. x0+19
//   XA   [4 planes][10 rows][24 cols] fp32 STEM: the generator input x (NCHW planes), same window as NZ
//        (W is the innermost tensor-map dimension of these two: the box starts 4 elements = 16 bytes left of the tile.
//         The box start is kept 16-byte aligned -- one starting at x0-2, 8 bytes off a 16-byte boundary, faulted the TMA
//         unit (illegal instruction) -- so the window is 24 wide and the 18 columns used sit at indices 3 .. 20.)
//   DIN  [20 rows][36 cols][16 ch] fp32   DOWN: input rows 2*y0-2 .. 2*y0+17, cols 2*x0-2 .. 2*x0+33 (16-ch chunk)
// A operand (one K block of 64 channels, M = 128 pixel rows): fp16 hi and lo planes, wgmma K-major SWIZZLE_128B:
//   byte(m, k) = (m >> 3) * 1024 + (m & 7) * 128 + (((k >> 3) ^ (m & 7)) << 4) + (k & 7) * 2
#pragma once
#include <stdint.h>

#ifdef MIGAN_EMULATE
#include <math.h>
#include <string.h>
#define SC_DEV static inline
#else
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#define SC_DEV __device__ __forceinline__
#endif

namespace migan {
namespace stages {

constexpr float kAlpha = 0.2f;                 // lrelu_agc (migan_inference.py:20-28): alpha, gain sqrt 2, clamp 256
constexpr float kGain = 1.41421356237309515f;
constexpr float kClamp = 256.0f;
constexpr float kSplit = 64.0f;                // power-of-two scale of the fp16 hi/lo split (common.cuh kActSplitScale)
constexpr int kAuxW = 24;                      // row length of the NZ / XA windows
constexpr int kAuxLeft = 4;                    // the windows start at column x0 - kAuxLeft; IN column c <-> window column c + 3

// A pair of fp32 values (two channels) handled together.  On the device P2 is float2 and every operation is two scalar
// FFMA / FMUL / FADD with round-to-nearest (Hopper has no packed fp32 instructions), so the emulation build below
// computes bit-identical results.
#ifdef MIGAN_EMULATE
struct P2 { float x, y; };
typedef P2 f2;
struct alignas(16) f4 { float x, y, z, w; };
SC_DEV P2 pk(float lo, float hi) { P2 r; r.x = lo; r.y = hi; return r; }
SC_DEV P2 ffma2(P2 a, P2 b, P2 c) { return pk(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
SC_DEV P2 fmul2(P2 a, P2 b) { return pk(a.x * b.x, a.y * b.y); }
SC_DEV P2 fadd2(P2 a, P2 b) { return pk(a.x + b.x, a.y + b.y); }
SC_DEV uint32_t f2_to_h2(float lo, float hi) {
    _Float16 a = (_Float16)lo, b = (_Float16)hi;
    uint16_t ua, ub; memcpy(&ua, &a, 2); memcpy(&ub, &b, 2);
    return (uint32_t)ua | ((uint32_t)ub << 16);
}
SC_DEV uint32_t fbits(float v) { uint32_t u; memcpy(&u, &v, 4); return u; }
SC_DEV float bitsf(uint32_t u) { float v; memcpy(&v, &u, 4); return v; }
SC_DEV float ldg1(const float* p) { return *p; }
SC_DEV void st_u2(uint8_t* p, uint32_t a, uint32_t b) { memcpy(p, &a, 4); memcpy(p + 4, &b, 4); }
SC_DEV float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
#else
typedef float2 P2;
typedef float2 f2;
typedef float4 f4;
SC_DEV P2 pk(float lo, float hi) { return make_float2(lo, hi); }
SC_DEV P2 ffma2(P2 a, P2 b, P2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
SC_DEV P2 fmul2(P2 a, P2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
SC_DEV P2 fadd2(P2 a, P2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
SC_DEV uint32_t f2_to_h2(float lo, float hi) { __half2 h = __floats2half2_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&h); }
SC_DEV uint32_t fbits(float v) { return __float_as_uint(v); }
SC_DEV float bitsf(uint32_t u) { return __uint_as_float(u); }
SC_DEV float ldg1(const float* p) { return __ldg(p); }
SC_DEV void st_u2(uint8_t* p, uint32_t a, uint32_t b) { *reinterpret_cast<uint2*>(p) = make_uint2(a, b); }
SC_DEV float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
#endif
SC_DEV P2 unpk(P2 v) { return v; }
SC_DEV P2 fsub2(P2 a, P2 b) { return ffma2(b, pk(-1.0f, -1.0f), a); }     // a - b, exact
SC_DEV P2 p2zero() { return pk(0.0f, 0.0f); }
typedef P2 u64;   // historical name of the packed pair in this file

SC_DEV int imin(int a, int b) { return a < b ? a : b; }
SC_DEV int imax(int a, int b) { return a > b ? a : b; }
SC_DEV int iclamp(int v, int lo, int hi) { return imin(imax(v, lo), hi); }

struct F4 { u64 lo, hi; };   // four floats as two packed pairs (the registers of a float4)
SC_DEV F4 as_f4(const f4 v) { F4 r; r.lo = pk(v.x, v.y); r.hi = pk(v.z, v.w); return r; }
SC_DEV f4 to_f4(const F4 v) { f4 r; r.x = v.lo.x; r.y = v.lo.y; r.z = v.hi.x; r.w = v.hi.y; return r; }
SC_DEV void fma4p(F4& acc, const F4 w, const F4 v) { acc.lo = ffma2(w.lo, v.lo, acc.lo); acc.hi = ffma2(w.hi, v.hi, acc.hi); }
SC_DEV void fma4s(F4& acc, const u64 w2, const F4 v) { acc.lo = ffma2(w2, v.lo, acc.lo); acc.hi = ffma2(w2, v.hi, acc.hi); }

// clamp(max(v, 0.2 v), +-lim) on a pair: lrelu_agc with the gain already folded into v (v = gain * pre-activation)
SC_DEV P2 act_pair(P2 v, float lim) {
    const P2 b = fmul2(v, pk(kAlpha, kAlpha));
    return pk(fminf(fmax3(v.x, b.x, -lim), lim), fminf(fmax3(v.y, b.y, -lim), lim));
}
// fp32 pair s (|s| <= 16384) -> fp16x2 hi and lo with hi + lo ~= s to 22 bits.  hi = s with the low 13 mantissa bits
// cleared (exactly representable in fp16), lo = fp16(s - hi).
SC_DEV void split_pack2(const P2 s, uint32_t& hi, uint32_t& lo) {
    const float hx = bitsf(fbits(s.x) & 0xFFFFE000u), hy = bitsf(fbits(s.y) & 0xFFFFE000u);
    const P2 d = fsub2(s, pk(hx, hy));
    hi = f2_to_h2(hx, hy);
    lo = f2_to_h2(d.x, d.y);
}
// byte offset of (row m, 16-byte chunk j of the 128-byte K row) in a SWIZZLE_128B K-major operand plane
SC_DEV uint32_t a_off(int m, uint32_t j) { return (uint32_t)(m >> 3) * 1024u + (uint32_t)(m & 7) * 128u + ((j ^ (uint32_t)(m & 7)) << 4); }

// ---------------------------------------------------------------------------------------------------------------
// Depthwise 3x3 + bias + lrelu_agc on one 32-channel chunk -> its half of the A operand K block (fp16 hi/lo).
// The taps / bias carry S = kSplit * sqrt(2):  S * clamp(lrelu(v) * sqrt2, +-256) == clamp(max(v', .2 v'), +-256 kSplit).
// Worker = (column, 4-channel vector); it slides a 3x3 window down the TH rows: 3 LDS.128 per output row, all
// offsets compile-time.  SeparableConv2d.conv1 + activation, migan_inference.py:155-157.
//   sin   IN stage (float4 units)      w9/bias  [9][cin] / [cin] tap tables (shared memory or global)
//   g     which 32-channel half of the 64-channel K block this chunk is (0/1);  cg0 = first channel of the chunk
// ---------------------------------------------------------------------------------------------------------------
template <int TN, int TH, int TW>
SC_DEV void prologue_chunk(const f4* __restrict__ sin, uint8_t* __restrict__ a_hi, uint8_t* __restrict__ a_lo,
                           const float* __restrict__ w9, const float* __restrict__ bias, int cin, int cg0, int g, int tg) {
    constexpr int NCOLS = TN * TW;
    constexpr int ROW_F4 = (TW + 2) * 8;                   // float4 per halo'd input row (8 float4 / pixel)
#pragma unroll
    for (int rep = 0; rep < (NCOLS * 8 + 127) / 128; ++rep) {
        const int item = tg + rep * 128;
        const int cvec = item & 7, colidx = item >> 3;
        const int col = (colidx & 3) * (NCOLS >> 2) + (colidx >> 2);   // spreads a warp over 4 distinct swizzle rows
        const int img_l = col / TW, x = col % TW;
        const int cg = cg0 + cvec * 4;
        F4 w[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) w[t] = as_f4(*reinterpret_cast<const f4*>(w9 + t * cin + cg));
        const F4 bv = as_f4(*reinterpret_cast<const f4*>(bias + cg));
        const f4* base = sin + (img_l * (TH + 2) * (TW + 2) + x) * 8 + cvec;
        const uint32_t jchunk = (uint32_t)(g * 4 + (cvec >> 1));
        const uint32_t sub = (uint32_t)(cvec & 1) * 8;
        // Two output rows per step: four independent accumulation chains, loads of both rows issued up front.
        F4 r0[3], r1[3], r2[3], r3[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) { r0[d] = as_f4(base[d * 8]); r1[d] = as_f4(base[ROW_F4 + d * 8]); }
#pragma unroll
        for (int y = 0; y < TH; y += 2) {
#pragma unroll
            for (int d = 0; d < 3; ++d) { r2[d] = as_f4(base[(y + 2) * ROW_F4 + d * 8]); r3[d] = as_f4(base[(y + 3) * ROW_F4 + d * 8]); }
            F4 a = bv, b = bv;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                fma4p(a, w[d], r0[d]);     fma4p(b, w[d], r1[d]);
                fma4p(a, w[3 + d], r1[d]); fma4p(b, w[3 + d], r2[d]);
                fma4p(a, w[6 + d], r2[d]); fma4p(b, w[6 + d], r3[d]);
            }
            constexpr float kLim = kClamp * kSplit;
            uint32_t hi0x, hi0y, lo0x, lo0y, hi1x, hi1y, lo1x, lo1y;
            split_pack2(unpk(act_pair(a.lo, kLim)), hi0x, lo0x);
            split_pack2(unpk(act_pair(b.lo, kLim)), hi1x, lo1x);
            split_pack2(unpk(act_pair(a.hi, kLim)), hi0y, lo0y);
            split_pack2(unpk(act_pair(b.hi, kLim)), hi1y, lo1y);
            const int m0 = (img_l * TH + y) * TW + x, m1 = m0 + TW;      // rows of the M tile
            const uint32_t off0 = a_off(m0, jchunk) + sub, off1 = a_off(m1, jchunk) + sub;
            st_u2(a_hi + off0, hi0x, hi0y);
            st_u2(a_lo + off0, lo0x, lo0y);
            st_u2(a_hi + off1, hi1x, hi1y);
            st_u2(a_lo + off1, lo1x, lo1y);
#pragma unroll
            for (int d = 0; d < 3; ++d) { r0[d] = r2[d]; r1[d] = r3[d]; }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// UP pre-stage: builds the depthwise conv's input IN[r][c] in place from the PREVIOUS layer's raw 1x1 output:
//   x = lrelu_agc( Upsample2d(t) + noise ) + skip          migan_inference.py:98-103, :165-169, :304-305
// Upsample2d = zero insertion + pad(2,1,2,1) + 4x4 FIR, i.e. the polyphase form
//   out[2i + a][2j + b] = sum_{u,v in {0,1}} f[a + 2u][b + 2v] * t[i - 1 + a + u][j - 1 + b + v]      (t = 0 outside)
// IN arrives holding the skip tensor (encoder feature, zero outside the image); pixels outside the image must stay
// ZERO (they are the depthwise conv's zero padding), not act(noise).
// `f` = the 16 taps * sqrt(2) (channel-uniform: checked on the host), NZ = noise * sqrt(2).
//
// Decomposition: the tile origin is even, so IN row 2i is the ODD image row 2m-1 and IN row 2i+1 the even row 2m
// (m = y0/2 + i), and both read the same two low-resolution rows m-1, m (phase a = 1 of cell m-1, phase a = 0 of cell m);
// likewise for columns.  A worker item is therefore one 2 x 2 block of IN pixels (rows 2i, 2i+1; cols 2j, 2j+1;
// i < 5, j < 9) computed from the 2 x 2 window T[i..i+1][j..j+1]: the 45 blocks tile the 10 x 18 window exactly -- no
// clamped indices, no discarded outputs, 4 loads of t per 4 outputs.  360 items (block, 4-channel vector) per chunk.
// ---------------------------------------------------------------------------------------------------------------
struct UpTaps { float f[16]; };

SC_DEV void prestage_up(f4* __restrict__ in, const f4* __restrict__ ta, const float* __restrict__ nz, const UpTaps& taps,
                        int y0, int x0, int R, int has_noise, int tg) {
    const int cvec = tg & 7;
#pragma unroll 1
    for (int item = tg; item < 360; item += 128) {
        const int cell = item >> 3;
        const int i = cell / 9, j = cell - i * 9;
        const f4* tp = ta + (i * 10 + j) * 8 + cvec;
        const F4 t00 = as_f4(tp[0]), t01 = as_f4(tp[8]), t10 = as_f4(tp[80]), t11 = as_f4(tp[88]);
        // rows / columns of the block that lie outside the image (only on border tiles)
        const bool row_out[2] = {(y0 == 0) && (i == 0), (y0 + 8 == R) && (i == 4)};
        const bool col_out[2] = {(x0 == 0) && (j == 0), (x0 + 16 == R) && (j == 8)};
        f4* px0 = in + ((2 * i) * 18 + 2 * j) * 8 + cvec;
        const float* nzp = nz + (2 * i) * kAuxW + 2 * j + kAuxLeft - 1;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int a = 1 - rr;                          // IN row 2i is phase a = 1, row 2i+1 phase a = 0
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
                const int b = 1 - cc;
                const float nzv = has_noise ? nzp[rr * kAuxW + cc] : 0.f;
                F4 acc; acc.lo = acc.hi = pk(nzv, nzv);
                const float f00 = taps.f[a * 4 + b], f01 = taps.f[a * 4 + b + 2];
                const float f10 = taps.f[(a + 2) * 4 + b], f11 = taps.f[(a + 2) * 4 + b + 2];
                fma4s(acc, pk(f00, f00), t00);
                fma4s(acc, pk(f01, f01), t01);
                fma4s(acc, pk(f10, f10), t10);
                fma4s(acc, pk(f11, f11), t11);
                f4* px = px0 + (rr * 18 + cc) * 8;
                const F4 sk = as_f4(*px);
                F4 o;
                o.lo = fadd2(act_pair(acc.lo, kClamp), sk.lo);
                o.hi = fadd2(act_pair(acc.hi, kClamp), sk.hi);
                if (row_out[rr] || col_out[cc]) { o.lo = p2zero(); o.hi = p2zero(); }
                *px = to_f4(o);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// STEM pre-stage: IN[r][c][ch] = lrelu_agc( fromrgb(x)[ch] + b[ch] ) for the chunk's 32 channels (zero outside the
// image): EncoderBlock.fromrgb + activation, migan_inference.py:193-196, recomputed on the halo so the 64-channel
// stem tensor never exists in HBM.  ws = weights * sqrt2 pair-interleaved [C0/2][4 planes][2], bs = [C0] bias * sqrt2
// (shared-memory table).
// Worker item = (pixel of the 10 x 18 window, channel vector): 1440 items per chunk.
// ---------------------------------------------------------------------------------------------------------------
template <bool kBorder>
SC_DEV void prestage_stem_t(f4* __restrict__ in, const float* __restrict__ xa, const float* __restrict__ ws,
                            const float* __restrict__ bs, int cg0, int y0, int x0, int R, int tg) {
    const int cvec = tg & 7;
    const int ch = cg0 + cvec * 4;
    // ws is pair-interleaved: [channel pair][plane][2] = (w[ch][i], w[ch+1][i]) adjacent, so a 128-bit load is two ready pairs
    const F4 wa = as_f4(*reinterpret_cast<const f4*>(ws + ch * 4)), wb = as_f4(*reinterpret_cast<const f4*>(ws + ch * 4 + 4));
    const F4 wc = as_f4(*reinterpret_cast<const f4*>(ws + ch * 4 + 8)), wd = as_f4(*reinterpret_cast<const f4*>(ws + ch * 4 + 12));
    const F4 bv = as_f4(*reinterpret_cast<const f4*>(bs + ch));
    const P2 wl[4] = {wa.lo, wa.hi, wb.lo, wb.hi};         // (ch, ch+1) x input plane 0..3
    const P2 wh[4] = {wc.lo, wc.hi, wd.lo, wd.hi};         // (ch+2, ch+3)
    const P2 bl = bv.lo, bh = bv.hi;
    int r = 0, c = tg >> 3;                                // pixel (tg >> 3) + 16 k, advanced incrementally (no division)
#pragma unroll 4
    for (int k = 0; k < 12; ++k) {
        const int px = (tg >> 3) + 16 * k;
        if (px >= 180) break;
        if (k > 0) { c += 16; if (c >= 18) { c -= 18; r += 1; } }
        const int Y = y0 - 1 + r, X = x0 - 1 + c;
        u64 lo = bl, hi = bh;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float xv = xa[i * (10 * kAuxW) + r * kAuxW + c + kAuxLeft - 1];
            const u64 x2 = pk(xv, xv);
            lo = ffma2(x2, wl[i], lo);
            hi = ffma2(x2, wh[i], hi);
        }
        F4 o;
        o.lo = act_pair(lo, kClamp);
        o.hi = act_pair(hi, kClamp);
        if (kBorder && !((Y >= 0) && (Y < R) && (X >= 0) && (X < R))) { o.lo = p2zero(); o.hi = p2zero(); }
        in[px * 8 + cvec] = to_f4(o);
    }
}
// Tiles that touch the image border zero the halo pixels outside the image; interior tiles (most of them) skip the test.
SC_DEV void prestage_stem(f4* __restrict__ in, const float* __restrict__ xa, const float* __restrict__ ws,
                          const float* __restrict__ bs, int cg0, int y0, int x0, int R, int tg) {
    if (y0 == 0 || x0 == 0 || y0 + 8 == R || x0 + 16 == R) prestage_stem_t<true>(in, xa, ws, bs, cg0, y0, x0, R, tg);
    else prestage_stem_t<false>(in, xa, ws, bs, cg0, y0, x0, R, tg);
}

}  // namespace stages
}  // namespace migan

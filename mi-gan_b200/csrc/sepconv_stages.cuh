// CUDA-core stages of the fused SeparableConv2d kernel (sepconv_tc.cu) that work on shared-memory tiles.
//
// Every function here is written against plain pointers into one pipeline stage of shared memory and takes the
// worker index `tg` (0..127: the thread's index inside its 128-thread prologue group) as an argument, with no
// barrier, shuffle or special register inside.  That is deliberate: the same source compiles as plain C++
// (-DMIGAN_EMULATE, tests/emul/build_emul.py) where a test loops tg = 0..127 over a host buffer filled the way
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
#include "portable.cuh"

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
CK_D P2 pk(float lo, float hi) { P2 r; r.x = lo; r.y = hi; return r; }
CK_D P2 ffma2(P2 a, P2 b, P2 c) { return pk(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
CK_D P2 fmul2(P2 a, P2 b) { return pk(a.x * b.x, a.y * b.y); }
CK_D P2 fadd2(P2 a, P2 b) { return pk(a.x + b.x, a.y + b.y); }
CK_D uint32_t f2_to_h2(float lo, float hi) {
    _Float16 a = (_Float16)lo, b = (_Float16)hi;
    uint16_t ua, ub; memcpy(&ua, &a, 2); memcpy(&ub, &b, 2);
    return (uint32_t)ua | ((uint32_t)ub << 16);
}
CK_D uint32_t fbits(float v) { uint32_t u; memcpy(&u, &v, 4); return u; }
CK_D float bitsf(uint32_t u) { float v; memcpy(&v, &u, 4); return v; }
CK_D float ldg1(const float* p) { return *p; }
CK_D void st_u2(uint8_t* p, uint32_t a, uint32_t b) { memcpy(p, &a, 4); memcpy(p + 4, &b, 4); }
CK_D float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
#else
typedef float2 P2;
typedef float2 f2;
typedef float4 f4;
CK_D P2 pk(float lo, float hi) { return make_float2(lo, hi); }
CK_D P2 ffma2(P2 a, P2 b, P2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
CK_D P2 fmul2(P2 a, P2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
CK_D P2 fadd2(P2 a, P2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
CK_D uint32_t f2_to_h2(float lo, float hi) { __half2 h = __floats2half2_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&h); }
CK_D uint32_t fbits(float v) { return __float_as_uint(v); }
CK_D float bitsf(uint32_t u) { return __uint_as_float(u); }
CK_D float ldg1(const float* p) { return __ldg(p); }
CK_D void st_u2(uint8_t* p, uint32_t a, uint32_t b) { *reinterpret_cast<uint2*>(p) = make_uint2(a, b); }
CK_D float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
#endif
CK_D P2 unpk(P2 v) { return v; }
CK_D P2 fsub2(P2 a, P2 b) { return ffma2(b, pk(-1.0f, -1.0f), a); }     // a - b, exact
CK_D P2 p2zero() { return pk(0.0f, 0.0f); }
typedef P2 u64;   // historical name of the packed pair in this file

CK_D int imin(int a, int b) { return a < b ? a : b; }
CK_D int imax(int a, int b) { return a > b ? a : b; }
CK_D int iclamp(int v, int lo, int hi) { return imin(imax(v, lo), hi); }

struct F4 { u64 lo, hi; };   // four floats as two packed pairs (the registers of a float4)
CK_D F4 as_f4(const f4 v) { F4 r; r.lo = pk(v.x, v.y); r.hi = pk(v.z, v.w); return r; }
CK_D f4 to_f4(const F4 v) { f4 r; r.x = v.lo.x; r.y = v.lo.y; r.z = v.hi.x; r.w = v.hi.y; return r; }
CK_D void fma4p(F4& acc, const F4 w, const F4 v) { acc.lo = ffma2(w.lo, v.lo, acc.lo); acc.hi = ffma2(w.hi, v.hi, acc.hi); }
CK_D void fma4s(F4& acc, const u64 w2, const F4 v) { acc.lo = ffma2(w2, v.lo, acc.lo); acc.hi = ffma2(w2, v.hi, acc.hi); }

// clamp(max(v, 0.2 v), +-lim) on a pair: lrelu_agc with the gain already folded into v (v = gain * pre-activation)
CK_D P2 act_pair(P2 v, float lim) {
    const P2 b = fmul2(v, pk(kAlpha, kAlpha));
    return pk(fminf(fmax3(v.x, b.x, -lim), lim), fminf(fmax3(v.y, b.y, -lim), lim));
}
// fp32 pair s (|s| <= 16384) -> fp16x2 hi and lo with hi + lo ~= s to 22 bits.  hi = s with the low 13 mantissa bits
// cleared (exactly representable in fp16), lo = fp16(s - hi).
CK_D void split_pack2(const P2 s, uint32_t& hi, uint32_t& lo) {
    const float hx = bitsf(fbits(s.x) & 0xFFFFE000u), hy = bitsf(fbits(s.y) & 0xFFFFE000u);
    const P2 d = fsub2(s, pk(hx, hy));
    hi = f2_to_h2(hx, hy);
    lo = f2_to_h2(d.x, d.y);
}
// byte offset of (row m, 16-byte chunk j of the 128-byte K row) in a SWIZZLE_128B K-major operand plane
CK_D uint32_t a_off(int m, uint32_t j) { return (uint32_t)(m >> 3) * 1024u + (uint32_t)(m & 7) * 128u + ((j ^ (uint32_t)(m & 7)) << 4); }

// ---------------------------------------------------------------------------------------------------------------
// Depthwise 3x3 + bias + lrelu_agc on one 32-channel chunk -> its half of the A operand K block (fp16 hi/lo).
// The taps / bias carry S = kSplit * sqrt(2):  S * clamp(lrelu(v) * sqrt2, +-256) == clamp(max(v', .2 v'), +-256 kSplit).
// Worker = (2 adjacent columns, 4-channel vector, RH = 4 rows); it slides a 3 x 4 input window down its rows: 4 LDS.128
// per input row for 2 output columns, (RH + 2) * 4 = 24 per 8 outputs (one column per worker took 30), all offsets
// compile-time.  Every output is the 9-tap chain from the bias in the same order (tap column outer, tap row inner).
// SeparableConv2d.conv1 + activation, migan_inference.py:155-157.
//   sin   IN stage (float4 units)      w9/bias  [9][cin] / [cin] tap tables (shared memory or global)
//   g     which 32-channel half of the 64-channel K block this chunk is (0/1);  cg0 = first channel of the chunk
// ---------------------------------------------------------------------------------------------------------------
template <int TN, int TH, int TW>
CK_D void prologue_chunk(const f4* __restrict__ sin, uint8_t* __restrict__ a_hi, uint8_t* __restrict__ a_lo,
                           const float* __restrict__ w9, const float* __restrict__ bias, int cin, int cg0, int g, int tg) {
    constexpr int NPAIR = TN * TW / 2;                     // column pairs of the tile (8 at 16x8 / 8x8, 16 at 4x4)
    constexpr int RH = 4;                                  // output rows per worker
    constexpr int NSEG = TH / RH;                          // row segments per column pair (2, or 1 at 4x4)
    constexpr int ROW_F4 = (TW + 2) * 8;                   // float4 per halo'd input row (8 float4 / pixel)
    static_assert(NPAIR * NSEG * 8 == 128, "one work item per prologue thread");
    const int cvec = tg & 7, wk = tg >> 3;
    // Swapping bits 0 and 1 of the worker index puts pairs 2 apart (columns 4 apart) in each half-warp: at 16x8 and 8x8
    // tiles the two halves of a warp's STS.64 then land on distinct swizzle rows (bit 2 of m & 7 differs), 2 wavefronts.
    const int u = (wk & ~3) | ((wk & 1) << 1) | ((wk >> 1) & 1);
    const int pair = u % NPAIR, seg = u / NPAIR;
    const int img_l = (2 * pair) / TW, x = (2 * pair) % TW, y0 = seg * RH;
    const int cg = cg0 + cvec * 4;
    F4 w[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = as_f4(*reinterpret_cast<const f4*>(w9 + t * cin + cg));
    const F4 bv = as_f4(*reinterpret_cast<const f4*>(bias + cg));
    const f4* base = sin + ((img_l * (TH + 2) + y0) * (TW + 2) + x) * 8 + cvec;
    const uint32_t jchunk = (uint32_t)(g * 4 + (cvec >> 1));
    const uint32_t sub = (uint32_t)(cvec & 1) * 8;
    // One output row per step, both columns: two independent accumulation chains; the input rows rotate through r0..r2.
    F4 r0[4], r1[4], r2[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) { r0[d] = as_f4(base[d * 8]); r1[d] = as_f4(base[ROW_F4 + d * 8]); }
#pragma unroll
    for (int y = 0; y < RH; ++y) {
#pragma unroll
        for (int d = 0; d < 4; ++d) r2[d] = as_f4(base[(y + 2) * ROW_F4 + d * 8]);
        F4 a = bv, b = bv;                                 // columns x, x + 1
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            fma4p(a, w[d], r0[d]);     fma4p(b, w[d], r0[d + 1]);
            fma4p(a, w[3 + d], r1[d]); fma4p(b, w[3 + d], r1[d + 1]);
            fma4p(a, w[6 + d], r2[d]); fma4p(b, w[6 + d], r2[d + 1]);
        }
        constexpr float kLim = kClamp * kSplit;
        uint32_t hi0x, hi0y, lo0x, lo0y, hi1x, hi1y, lo1x, lo1y;
        split_pack2(unpk(act_pair(a.lo, kLim)), hi0x, lo0x);
        split_pack2(unpk(act_pair(b.lo, kLim)), hi1x, lo1x);
        split_pack2(unpk(act_pair(a.hi, kLim)), hi0y, lo0y);
        split_pack2(unpk(act_pair(b.hi, kLim)), hi1y, lo1y);
        const int m0 = (img_l * TH + y0 + y) * TW + x, m1 = m0 + 1;      // rows of the M tile
        const uint32_t off0 = a_off(m0, jchunk) + sub, off1 = a_off(m1, jchunk) + sub;
        st_u2(a_hi + off0, hi0x, hi0y);
        st_u2(a_lo + off0, lo0x, lo0y);
        st_u2(a_hi + off1, hi1x, hi1y);
        st_u2(a_lo + off1, lo1x, lo1y);
#pragma unroll
        for (int d = 0; d < 4; ++d) { r0[d] = r1[d]; r1[d] = r2[d]; }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// UP pre-stage: builds the depthwise conv's input IN[r][c] in place from the PREVIOUS layer's raw 1x1 output:
//   x = lrelu_agc( Upsample2d(t) + noise ) + skip          migan_inference.py:98-103, :165-169, :304-305
// Upsample2d = zero insertion + pad(2,1,2,1) + 4x4 FIR, i.e. the polyphase form
//   out[2i + a][2j + b] = sum_{u,v in {0,1}} f[a + 2u][b + 2v] * t[i - 1 + a + u][j - 1 + b + v]      (t = 0 outside)
// IN arrives holding the skip tensor (encoder feature, zero outside the image); pixels outside the H x W image must
// stay ZERO (they are the depthwise conv's zero padding), not act(noise).  That covers the halo of every tile and, for a
// tile that reaches past the right or bottom edge, every IN row / column beyond it.
// `f` = the 16 taps * sqrt(2) (channel-uniform: checked on the host), NZ = noise * sqrt(2).
//
// Decomposition: the tile origin is even, so IN row 2i is the ODD image row 2m-1 and IN row 2i+1 the even row 2m
// (m = y0/2 + i), and both read the same two low-resolution rows m-1, m (phase a = 1 of cell m-1, phase a = 0 of cell m);
// likewise for columns.  A worker item is therefore one 2 x 2 block of IN pixels (rows 2i, 2i+1; cols 2j, 2j+1;
// i < 5, j < 9) computed from the 2 x 2 window T[i..i+1][j..j+1]: the 45 blocks tile the 10 x 18 window exactly -- no
// clamped indices, no discarded outputs, 4 loads of t per 4 outputs.  360 items (block, 4-channel vector) per chunk.
// ---------------------------------------------------------------------------------------------------------------
struct UpTaps { float f[16]; };

CK_D void prestage_up(f4* __restrict__ in, const f4* __restrict__ ta, const float* __restrict__ nz, const UpTaps& taps,
                        int y0, int x0, int H, int W, int has_noise, int tg) {
    const int cvec = tg & 7;
#pragma unroll 1
    for (int item = tg; item < 360; item += 128) {
        const int cell = item >> 3;
        const int i = cell / 9, j = cell - i * 9;
        const f4* tp = ta + (i * 10 + j) * 8 + cvec;
        const F4 t00 = as_f4(tp[0]), t01 = as_f4(tp[8]), t10 = as_f4(tp[80]), t11 = as_f4(tp[88]);
        // rows / columns of the block that lie outside the image: IN rows 2i, 2i+1 are image rows y0-1+2i, y0+2i
        const int ya = y0 - 1 + 2 * i, xa = x0 - 1 + 2 * j;
        const bool row_out[2] = {ya < 0 || ya >= H, ya + 1 >= H};
        const bool col_out[2] = {xa < 0 || xa >= W, xa + 1 >= W};
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

// The same on a square R x R image.
CK_D void prestage_up(f4* __restrict__ in, const f4* __restrict__ ta, const float* __restrict__ nz, const UpTaps& taps,
                        int y0, int x0, int R, int has_noise, int tg) {
    prestage_up(in, ta, nz, taps, y0, x0, R, R, has_noise, tg);
}

// ---------------------------------------------------------------------------------------------------------------
// STEM pre-stage: IN[r][c][ch] = lrelu_agc( fromrgb(x)[ch] + b[ch] ) for the chunk's 32 channels (zero outside the
// image): EncoderBlock.fromrgb + activation, migan_inference.py:193-196, recomputed on the halo so the 64-channel
// stem tensor never exists in HBM.  ws = weights * sqrt2 pair-interleaved [C0/2][4 planes][2], bs = [C0] bias * sqrt2
// (shared-memory table).
// Worker item = (pixel of the 10 x 18 window, channel vector): 1440 items per chunk.
// ---------------------------------------------------------------------------------------------------------------
template <bool kBorder>
CK_D void prestage_stem_t(f4* __restrict__ in, const float* __restrict__ xa, const float* __restrict__ ws,
                            const float* __restrict__ bs, int cg0, int y0, int x0, int H, int W, int tg) {
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
        if (kBorder && !((Y >= 0) && (Y < H) && (X >= 0) && (X < W))) { o.lo = p2zero(); o.hi = p2zero(); }
        in[px * 8 + cvec] = to_f4(o);
    }
}
// Tiles that touch (or reach past) the image border zero the pixels outside the image; interior tiles (most of them)
// skip the test.
CK_D void prestage_stem(f4* __restrict__ in, const float* __restrict__ xa, const float* __restrict__ ws,
                          const float* __restrict__ bs, int cg0, int y0, int x0, int H, int W, int tg) {
    if (y0 == 0 || x0 == 0 || y0 + 8 >= H || x0 + 16 >= W) prestage_stem_t<true>(in, xa, ws, bs, cg0, y0, x0, H, W, tg);
    else prestage_stem_t<false>(in, xa, ws, bs, cg0, y0, x0, H, W, tg);
}
// The same on a square R x R image.
CK_D void prestage_stem(f4* __restrict__ in, const float* __restrict__ xa, const float* __restrict__ ws,
                          const float* __restrict__ bs, int cg0, int y0, int x0, int R, int tg) {
    prestage_stem(in, xa, ws, bs, cg0, y0, x0, R, R, tg);
}

}  // namespace stages
}  // namespace migan

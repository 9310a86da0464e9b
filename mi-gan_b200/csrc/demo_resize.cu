// The reference demo's request path at any photo size, scripts/demo.py:26-66 and :120-143 (SURVEY.md 8(f) rank 1):
//
//   photo u8 [H][W][3] --PIL BICUBIC, only when W > R or H > R--> img_resized [h'][w'][3]                   (resize, :48-53)
//   mask  u8 [Hm][Wm][C] --PIL NEAREST to <= 512--> channel / invert / threshold --PIL NEAREST to <= R--> mask_resized
//                                                                                                   (read_mask, :26-45)
//   img_resized --PIL BICUBIC--> R x R, mask_resized --PIL NEAREST--> R x R -> x = cat([m - 0.5, (v*2/255-1) * m])
//                                                                                                  (preprocess, :56-66)
//   [generator]
//   y -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 --cv2.resize INTER_CUBIC--> h' x w' -> img_resized where the mask is 255,
//   the result elsewhere                                                                                    (:135-140)
//
// Every resize reproduces its library's uint8 arithmetic bit for bit (oracle/demo_oracle.py is the numpy model):
//   PIL BICUBIC   a = -0.5, taps normalised in double and quantised to 2^-22 (rounded away from zero), each pass
//                 clamp((2^21 + sum v*k) >> 22); horizontal pass first, a uint8 intermediate.  A pass whose size does not
//                 change is skipped by PIL; its table here is {0, 1, 0, ...}, which gives the same bytes.
//   PIL NEAREST   the source coordinate accumulates the scale in double (xo = s/2, xo += s per output) and truncates.
//   OpenCV CUBIC  the scalar path: A = -0.75 float coefficients quantised to 1/2048 (round half to even), integer
//                 horizontal pass.  The vertical pass of a row of 3 * w' values runs OpenCV's vector body on the first
//                 8 * floor(3 * w' / 8) of them, in float: ((S3*b3 + S2*b2) + S1*b1) + S0*b0 rounded half to even, and
//                 its scalar tail on the rest, in fixed point: (sum S*k + 2^21) >> 22.
// The mask's per-pixel steps (channel, invert, v < 255 -> 0) commute with NEAREST, so they run on the original mask at
// the composed source index of the two or three NEAREST steps.
//
// A pass of up to MIGAN_PIPE_MAX_BATCH requests runs one launch per stage covering every request; the request table
// travels by value in the kernel parameter (DemoBatch, < 4 KB) with the stage's item prefix (batch_launch, comod_kernels.cuh):
//   tables (every resampler's coefficients / indices, computed on the device) -> down-scale width pass -> down-scale
//   height pass (both only when a photo is larger than R) -> R x R resize + mask + x  |  y -> uint8 + OpenCV width pass
//   -> OpenCV height pass + composite.
// Item kernels (comod_kernels.cuh style): the emulation build (tests/emul/build_emul.py) runs the very same functors on
// the CPU.  Every product and sum is rounded on its own (the *_rn functions of portable.cuh, no FMA contraction), in
// double where the libraries use double.
#include "prepost.cuh"
#include "abi_error.h"

namespace comod {

constexpr int DEMO_MASK_MAX = 512;      // read_mask's first resize (:28)
constexpr int DEMO_UP_TAPS = 5;         // PIL bicubic taps of an up-scale (support 2): img_resized -> R x R
constexpr int PIL_BITS = 22;            // Pillow's PRECISION_BITS for 8-bit images
constexpr int CV_LANES = 8;             // int16 lanes of OpenCV's 128-bit baseline SIMD (the vertical pass's vector body)

// Pillow's kernel size of a bicubic table in_size -> out_size: ceil(support) * 2 + 1, support = 2 * max(in / out, 1).
CK_HD int pil_ksize(int in_size, int out_size) {
    const double scale = (double)in_size / (double)out_size;
    return (int)ceil(2.0 * (scale < 1.0 ? 1.0 : scale)) * 2 + 1;
}

CK_D double pil_bicubic(double x) {     // bicubic_filter, a = -0.5
    if (x < 0.0) x = -x;
    if (x < 1.0) return dadd_rn(dmul_rn(dmul_rn(dadd_rn(dmul_rn(1.5, x), -2.5), x), x), 1.0);   // ((a+2)x - (a+3))x x + 1
    if (x < 2.0) return dmul_rn(dadd_rn(dmul_rn(dadd_rn(dmul_rn(dadd_rn(x, -5.0), x), 8.0), x), -4.0), -0.5);  // (((x-5)x+8)x-4)a
    return 0.0;
}

// Entry x of Pillow's bicubic table in_size -> out_size (precompute_coeffs + normalize_coeffs_8bpc): the first source
// index and `ksize` fixed-point taps, zero past the window.  The weights are recomputed for the division by their sum
// instead of being held in a local array (a 4K photo has 31 taps).
CK_D void pil_entry(int in_size, int out_size, int ksize, int x, int* xmin, int* k) {
    const double scale = ddiv_rn((double)in_size, (double)out_size);
    const double fs = scale < 1.0 ? 1.0 : scale;
    const double support = dmul_rn(2.0, fs);
    const double ss = ddiv_rn(1.0, fs);
    const double center = dmul_rn(dadd_rn((double)x, 0.5), scale);
    int lo = (int)dadd_rn(dadd_rn(center, -support), 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)dadd_rn(dadd_rn(center, support), 0.5);
    if (hi > in_size) hi = in_size;
    int n = hi - lo;
    n = n < 0 ? 0 : (n > ksize ? ksize : n);
    double ww = 0.0;
    for (int i = 0; i < n; ++i) ww = dadd_rn(ww, pil_bicubic(dmul_rn(dadd_rn(dadd_rn((double)(i + lo), -center), 0.5), ss)));
    for (int i = 0; i < n; ++i) {
        double w = pil_bicubic(dmul_rn(dadd_rn(dadd_rn((double)(i + lo), -center), 0.5), ss));
        if (ww != 0.0) w = ddiv_rn(w, ww);
        const double q = dmul_rn(w, (double)(1 << PIL_BITS));
        k[i] = w < 0.0 ? (int)dadd_rn(q, -0.5) : (int)dadd_rn(q, 0.5);
    }
    for (int i = n; i < ksize; ++i) k[i] = 0;
    *xmin = lo;
}

// Source index of output x of Pillow's NEAREST resize in_size -> out_size (ImagingScaleAffine): the coordinate starts at
// s / 2 and adds s = in / out per output, in double; the same accumulation is replayed here for every output.
CK_D int pil_nearest(int in_size, int out_size, int x) {
    if (in_size == out_size) return x;
    const double s = ddiv_rn((double)in_size, (double)out_size);
    double xo = dadd_rn(0.0, dmul_rn(s, 0.5));
    for (int i = 0; i < x; ++i) xo = dadd_rn(xo, s);
    const int v = xo < 0.0 ? -1 : (int)xo;
    return v < 0 ? 0 : (v >= in_size ? in_size - 1 : v);
}

// Entry d of OpenCV's INTER_CUBIC table in_size -> out_size (resizeGeneric, interpolateCubic, fixed point): the first tap's
// neighbour sx (taps at sx-1 .. sx+2, clamped to the image by the caller) and the four coefficients in units of 1/2048.
CK_D void cv_entry(int in_size, int out_size, int d, int* sx, int* c) {
    const double scale = ddiv_rn(1.0, ddiv_rn((double)out_size, (double)in_size));     // 1. / inv_scale
    const float f = (float)dadd_rn(dmul_rn(dadd_rn((double)d, 0.5), scale), -0.5);
    const int s = (int)floorf(f);
    const float x = fadd_rn(f, -(float)s);
    const float x1 = fadd_rn(x, 1.f), y = fadd_rn(1.f, -x);
    const float A = -0.75f;
    const float c0 = fadd_rn(fmul_rn(fadd_rn(fmul_rn(fadd_rn(fmul_rn(A, x1), 3.75f), x1), -6.f), x1), 3.f);   // ((A(x+1) - 5A)(x+1) + 8A)(x+1) - 4A
    const float c1 = fadd_rn(fmul_rn(fmul_rn(fadd_rn(fmul_rn(1.25f, x), -2.25f), x), x), 1.f);              // ((A+2)x - (A+3))x x + 1
    const float c2 = fadd_rn(fmul_rn(fmul_rn(fadd_rn(fmul_rn(1.25f, y), -2.25f), y), y), 1.f);
    const float c3 = fadd_rn(fadd_rn(fadd_rn(1.f, -c0), -c1), -c2);
    *sx = s;
    c[0] = (int)rintf(fmul_rn(c0, 2048.f)); c[1] = (int)rintf(fmul_rn(c1, 2048.f));
    c[2] = (int)rintf(fmul_rn(c2, 2048.f)); c[3] = (int)rintf(fmul_rn(c3, 2048.f));
}

CK_HD int dm_clamp(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
CK_HD uint8_t pil_clip8(int acc) { return (uint8_t)dm_clamp(acc >> PIL_BITS, 0, 255); }

// One request of a pass.  rs is img_resized: the photo itself when it fits R, else the down-scale's output in the
// scratch; kdw / kdh are the down-scale's tap counts (0: the photo fits).  tab, dtmp and ptmp are carved from the scratch.
struct DemoReq {
    const uint8_t* img; const uint8_t* mask; uint8_t* out;
    uint8_t* rs;        // img_resized [h1][w1][3]
    uint8_t* dtmp;      // width pass of the down-scale [H][w1][3]
    int* tab;           // every table, demo_tabs layout
    int* ptmp;          // OpenCV width pass [R][w1][3], int
    int H, W, Hm, Wm, C, invert, w1, h1, wa, ha, kdw, kdh;
};
struct DemoBatch {
    int64_t start[MIGAN_PIPE_MAX_BATCH + 1];   // item prefix of the launch
    DemoReq r[MIGAN_PIPE_MAX_BATCH];
    const float* y; float* x;                  // generator output [n][3][R][R] / model input [n][4][R][R]
    float* img;                                // evaluation batch only: the unmasked photo v * 2 / 255 - 1 [n][3][R][R]
    int n, res;
};
static_assert(sizeof(DemoBatch) <= 4000, "the batch descriptor must fit the classic 4 KB kernel parameter space");

// The tables of one request, one after the other in r.tab (ints):
//   dwx [w1] dwk [w1][kdw] dhx [h1] dhk [h1][kdh]      PIL down-scale W -> w1, H -> h1 (empty when the photo fits)
//   uwx [R]  uwk [R][5]    uhx [R]  uhk [R][5]         PIL w1 -> R, h1 -> R
//   mrx [R]  mry [R]       mox [w1] moy [h1]           mask source column / row of the R x R grid and of the output
//   cxs [w1] cxk [w1][4]   cys [h1] cyk [h1][4]        OpenCV R -> w1, R -> h1
struct DemoTabs { int *dwx, *dwk, *dhx, *dhk, *uwx, *uwk, *uhx, *uhk, *mrx, *mry, *mox, *moy, *cxs, *cxk, *cys, *cyk; };
CK_HD int64_t demo_tab_ints(const DemoReq& r, int R, DemoTabs* t) {
    int64_t o = 0;
    int* p = r.tab;
    int** dst[16] = {&t->dwx, &t->dwk, &t->dhx, &t->dhk, &t->uwx, &t->uwk, &t->uhx, &t->uhk,
                     &t->mrx, &t->mry, &t->mox, &t->moy, &t->cxs, &t->cxk, &t->cys, &t->cyk};
    const int64_t len[16] = {r.kdw ? r.w1 : 0, (int64_t)r.w1 * r.kdw, r.kdh ? r.h1 : 0, (int64_t)r.h1 * r.kdh,
                             R, (int64_t)R * DEMO_UP_TAPS, R, (int64_t)R * DEMO_UP_TAPS,
                             R, R, r.w1, r.h1, r.w1, (int64_t)r.w1 * 4, r.h1, (int64_t)r.h1 * 4};
    for (int i = 0; i < 16; ++i) { if (t) *dst[i] = p ? p + o : nullptr; o += len[i]; }
    return o;
}
CK_HD DemoTabs demo_tabs(const DemoReq& r, int R) { DemoTabs t; demo_tab_ints(r, R, &t); return t; }

// read_mask's per-pixel steps (prepost.cuh mask_known) at one source pixel of the original mask.
CK_HD bool demo_known(const DemoReq& r, int y, int x) { return mask_known(r.mask, r.Wm, r.C, r.invert, y, x); }

enum { DS_TABLES, DS_DOWN_W, DS_DOWN_H, DS_SQUARE, DS_POST_W, DS_OUT, DS_COUNT };
CK_HD int64_t demo_items(int stage, const DemoReq& r, int R) {
    switch (stage) {
        case DS_TABLES: return (r.kdw ? (int64_t)r.w1 + r.h1 : 0) + (int64_t)4 * R + (int64_t)2 * (r.w1 + r.h1);
        case DS_DOWN_W: return r.kdw ? (int64_t)r.H * r.w1 : 0;
        case DS_DOWN_H: return r.kdw ? (int64_t)r.h1 * r.w1 : 0;
        case DS_SQUARE: return (int64_t)R * R;
        case DS_POST_W: return (int64_t)R * r.w1;
        default: return (int64_t)r.h1 * r.w1;
    }
}

// Every table entry of every request.  items per request = demo_items(DS_TABLES)
struct DemoTablesK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int R = b.res;
        const DemoTabs t = demo_tabs(r, R);
        int j = (int)(i - b.start[k]);
        const int nw = r.kdw ? r.w1 : 0, nh = r.kdh ? r.h1 : 0;
        if (j < nw) { pil_entry(r.W, r.w1, r.kdw, j, t.dwx + j, t.dwk + (int64_t)j * r.kdw); return; }
        j -= nw;
        if (j < nh) { pil_entry(r.H, r.h1, r.kdh, j, t.dhx + j, t.dhk + (int64_t)j * r.kdh); return; }
        j -= nh;
        if (j < R) { pil_entry(r.w1, R, DEMO_UP_TAPS, j, t.uwx + j, t.uwk + j * DEMO_UP_TAPS); return; }
        j -= R;
        if (j < R) { pil_entry(r.h1, R, DEMO_UP_TAPS, j, t.uhx + j, t.uhk + j * DEMO_UP_TAPS); return; }
        j -= R;
        if (j < R) { t.mrx[j] = pil_nearest(r.Wm, r.wa, pil_nearest(r.wa, r.w1, pil_nearest(r.w1, R, j))); return; }
        j -= R;
        if (j < R) { t.mry[j] = pil_nearest(r.Hm, r.ha, pil_nearest(r.ha, r.h1, pil_nearest(r.h1, R, j))); return; }
        j -= R;
        if (j < r.w1) { t.mox[j] = pil_nearest(r.Wm, r.wa, pil_nearest(r.wa, r.w1, j)); return; }
        j -= r.w1;
        if (j < r.h1) { t.moy[j] = pil_nearest(r.Hm, r.ha, pil_nearest(r.ha, r.h1, j)); return; }
        j -= r.h1;
        if (j < r.w1) { cv_entry(R, r.w1, j, t.cxs + j, t.cxk + 4 * j); return; }
        j -= r.w1;
        cv_entry(R, r.h1, j, t.cys + j, t.cyk + 4 * j);
    }
};

// Width pass of the down-scale, W -> w1 on every photo row.  items per request = H * w1 (0 when the photo fits)
struct DemoDownWK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const DemoTabs t = demo_tabs(r, b.res);
        const int y = (int)(j / r.w1), x = (int)(j - (int64_t)y * r.w1);
        const int x0 = t.dwx[x];
        const int* kk = t.dwk + (int64_t)x * r.kdw;
        const uint8_t* row = r.img + (int64_t)y * r.W * 3;
        int acc[3] = {1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1)};
        for (int tp = 0; tp < r.kdw; ++tp) {
            const uint8_t* p = row + (int64_t)dm_clamp(x0 + tp, 0, r.W - 1) * 3;
            for (int c = 0; c < 3; ++c) acc[c] += (int)p[c] * kk[tp];
        }
        uint8_t* o = r.dtmp + j * 3;
        for (int c = 0; c < 3; ++c) o[c] = pil_clip8(acc[c]);
    }
};

// Height pass of the down-scale, H -> h1, into img_resized.  items per request = h1 * w1 (0 when the photo fits)
struct DemoDownHK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const DemoTabs t = demo_tabs(r, b.res);
        const int y = (int)(j / r.w1), x = (int)(j - (int64_t)y * r.w1);
        const int y0 = t.dhx[y];
        const int* kk = t.dhk + (int64_t)y * r.kdh;
        int acc[3] = {1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1)};
        for (int tp = 0; tp < r.kdh; ++tp) {
            const uint8_t* p = r.dtmp + ((int64_t)dm_clamp(y0 + tp, 0, r.H - 1) * r.w1 + x) * 3;
            for (int c = 0; c < 3; ++c) acc[c] += (int)p[c] * kk[tp];
        }
        uint8_t* o = r.rs + j * 3;
        for (int c = 0; c < 3; ++c) o[c] = pil_clip8(acc[c]);
    }
};

// img_resized -> R x R (PIL bicubic: both passes, 5 x 5 taps, the width pass's uint8 value recomputed per row tap),
// mask_resized -> R x R (NEAREST), then PreU8K's arithmetic (prepost.cu) into x[k].  items per request = R * R
struct DemoSquareK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int R = b.res;
        const DemoTabs t = demo_tabs(r, R);
        const int oy = (int)(j / R), ox = (int)(j - (int64_t)oy * R);
        const int x0 = t.uwx[ox], y0 = t.uhx[oy];
        const int* kx = t.uwk + ox * DEMO_UP_TAPS;
        const int* ky = t.uhk + oy * DEMO_UP_TAPS;
        int acc[3] = {1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1)};
        for (int ty = 0; ty < DEMO_UP_TAPS; ++ty) {
            if (ky[ty] == 0) continue;
            const uint8_t* row = r.rs + (int64_t)dm_clamp(y0 + ty, 0, r.h1 - 1) * r.w1 * 3;
            int h[3] = {1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1), 1 << (PIL_BITS - 1)};
            for (int tx = 0; tx < DEMO_UP_TAPS; ++tx) {
                const uint8_t* p = row + dm_clamp(x0 + tx, 0, r.w1 - 1) * 3;
                for (int c = 0; c < 3; ++c) h[c] += (int)p[c] * kx[tx];
            }
            for (int c = 0; c < 3; ++c) acc[c] += (int)pil_clip8(h[c]) * ky[ty];
        }
        const int64_t plane = (int64_t)R * R;
        float* x = b.x + (int64_t)k * 4 * plane + j;
        const float m = demo_known(r, t.mry[oy], t.mrx[ox]) ? 1.f : 0.f;                     // mask // 255   (:60)
        x[0] = pre_mask_value(m);
        for (int c = 0; c < 3; ++c) x[(c + 1) * plane] = pre_img_value(pil_clip8(acc[c]), m);
        if (b.img)
            for (int c = 0; c < 3; ++c) b.img[((int64_t)k * 3 + c) * plane + j] = pre_img_value(pil_clip8(acc[c]), 1.f);
    }
};

// The evaluation script's composite and normalisations (scripts/evaluate_fid_lpips.py:246-249), every product and sum
// rounded on its own: composed = m * img + (1 - m) * y, then (v * 0.5 + 0.5).clamp(0, 1) of img (in place: `real`) and of
// composed.  m = x channel 0 + 0.5.  items = n * R * R
struct EvalCompositeK {
    const float* x; const float* y; float* real; float* composed; int64_t plane;
    CK_D static float unit(float v) { return fminf(fmaxf(fadd_rn(fmul_rn(v, 0.5f), 0.5f), 0.f), 1.f); }
    CK_D void operator()(int64_t i) const {
        const int64_t k = i / plane, p = i - k * plane;
        const float m = fadd_rn(x[k * 4 * plane + p], 0.5f);
        for (int c = 0; c < 3; ++c) {
            const int64_t o = (k * 3 + c) * plane + p;
            const float v = real[o];
            composed[o] = unit(fadd_rn(fmul_rn(m, v), fmul_rn(fadd_rn(1.f, -m), y[o])));
            real[o] = unit(v);
        }
    }
};

// y -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 (PostU8K's arithmetic) fused with OpenCV's width pass R -> w1 (integer).
// items per request = R * w1
struct DemoPostWK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int R = b.res;
        const DemoTabs t = demo_tabs(r, R);
        const int row = (int)(j / r.w1), x = (int)(j - (int64_t)row * r.w1);
        const int s = t.cxs[x];
        const int* cx = t.cxk + 4 * x;
        const float* y = b.y + (int64_t)k * 3 * R * R + (int64_t)row * R;
        int* o = r.ptmp + j * 3;
        for (int c = 0; c < 3; ++c) {
            int acc = 0;
            for (int tp = 0; tp < 4; ++tp)
                acc += (int)post_u8(y[(int64_t)c * R * R + dm_clamp(s - 1 + tp, 0, R - 1)]) * cx[tp];
            o[c] = acc;
        }
    }
};

// OpenCV's height pass R -> h1 (float, rounded half to even) fused with the composite (:139-140): img_resized where the
// mask is 255, the resized result elsewhere.  items per request = h1 * w1
struct DemoOutK {
    const DemoBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const DemoReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int R = b.res;
        const DemoTabs t = demo_tabs(r, R);
        const int y = (int)(j / r.w1), x = (int)(j - (int64_t)y * r.w1);
        uint8_t* o = r.out + j * 3;
        if (demo_known(r, t.moy[y], t.mox[x])) {
            const uint8_t* p = r.rs + j * 3;
            for (int c = 0; c < 3; ++c) o[c] = p[c];
            return;
        }
        const int s = t.cys[y];
        const int* cy = t.cyk + 4 * y;
        float bk[4];
        const int* src[4];
        for (int tp = 0; tp < 4; ++tp) {
            bk[tp] = fmul_rn((float)cy[tp], 1.f / (2048.f * 2048.f));
            src[tp] = r.ptmp + ((int64_t)dm_clamp(s - 1 + tp, 0, R - 1) * r.w1 + x) * 3;
        }
        const int body = (3 * r.w1 / CV_LANES) * CV_LANES;     // the row's values in OpenCV's vector body
        for (int c = 0; c < 3; ++c) {
            if (3 * x + c < body) {
                float acc = fadd_rn(fmul_rn((float)src[3][c], bk[3]), fmul_rn((float)src[2][c], bk[2]));
                acc = fadd_rn(acc, fmul_rn((float)src[1][c], bk[1]));
                acc = fadd_rn(acc, fmul_rn((float)src[0][c], bk[0]));
                o[c] = (uint8_t)fminf(fmaxf(rintf(acc), 0.f), 255.f);
            } else {                                            // the scalar tail: fixed point, 2 x 11 fraction bits
                const int acc = src[0][c] * cy[0] + src[1][c] * cy[1] + src[2][c] * cy[2] + src[3][c] * cy[3];
                o[c] = (uint8_t)dm_clamp((acc + (1 << 21)) >> 22, 0, 255);
            }
        }
    }
};

}  // namespace comod

namespace migan {

int demo_resized_size(int w, int h, int max_size, int* ow, int* oh);

namespace {

// The descriptors of a pass, with every request's regions carved out of `scratch` (nullptr: sizes only); returns the bytes.
// eval: the evaluation batch's layout -- the photo goes straight to R x R (one PIL resize, w1 = h1 = R, when it is not
// that size already) and the mask by one NEAREST step (wa, ha = the mask's size); no post-processing regions.
size_t demo_layout(const migan_demo_request* q, int n, int res, void* scratch, comod::DemoBatch* b, bool eval = false) {
    b->n = n; b->res = res; b->y = nullptr; b->x = nullptr; b->img = nullptr;
    unsigned char* base = static_cast<unsigned char*>(scratch);
    size_t off = 0;
    auto carve = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    for (int k = 0; k < n; ++k) {
        comod::DemoReq& r = b->r[k];
        r = {};
        r.img = q[k].img; r.mask = q[k].mask; r.out = q[k].out;
        r.H = q[k].H; r.W = q[k].W; r.Hm = q[k].Hm; r.Wm = q[k].Wm; r.C = q[k].mask_channels; r.invert = q[k].invert != 0;
        r.w1 = eval ? res : q[k].out_w; r.h1 = eval ? res : q[k].out_h;
        if (eval) { r.wa = r.Wm; r.ha = r.Hm; }
        else demo_resized_size(r.Wm, r.Hm, comod::DEMO_MASK_MAX, &r.wa, &r.ha);
        const bool down = r.w1 != r.W || r.h1 != r.H;
        r.kdw = down ? comod::pil_ksize(r.W, r.w1) : 0;
        r.kdh = down ? comod::pil_ksize(r.H, r.h1) : 0;
        r.tab = nullptr;
        r.tab = reinterpret_cast<int*>(carve((size_t)comod::demo_tab_ints(r, res, nullptr) * sizeof(int)));
        r.ptmp = eval ? nullptr : reinterpret_cast<int*>(carve((size_t)res * r.w1 * 3 * sizeof(int)));
        if (down) {
            r.dtmp = carve((size_t)r.H * r.w1 * 3);
            r.rs = carve((size_t)r.h1 * r.w1 * 3);
        } else {
            r.rs = const_cast<uint8_t*>(r.img);
        }
    }
    return off;
}

}  // namespace

// demo.py `resize` (:48-53): (int(w * r), int(h * r)), r = max_size / w if w > h else max_size / h, when either side is
// larger than max_size; the size itself otherwise.  Python's float arithmetic is IEEE double, so this is the same number.
int demo_resized_size(int w, int h, int max_size, int* ow, int* oh) {
    if (w > max_size || h > max_size) {
        const double ratio = w > h ? (double)max_size / (double)w : (double)max_size / (double)h;
        *ow = (int)((double)w * ratio);
        *oh = (int)((double)h * ratio);
    } else {
        *ow = w; *oh = h;
    }
    return 0;
}

// The demo batch, or the evaluation batch (eval: no output, and the photo goes straight to R x R).
int check_demo_batch(const char* who, const migan_demo_request* q, int n, int res, bool eval) {
    if (int rc = check_batch_size(who, q, n)) return rc;
    if (res < 1 || res > 8192) return fail(MIGAN_ERR_INVALID, "%s: bad resolution %d", who, res);
    for (int k = 0; k < n; ++k) {
        const migan_demo_request& r = q[k];
        if (eval && (!r.img || !r.mask)) return fail(MIGAN_ERR_INVALID, "%s: request %d: null image or mask", who, k);
        if (!eval && (!r.img || !r.mask || !r.out)) return fail(MIGAN_ERR_INVALID, "%s: request %d: null image, mask or output", who, k);
        if (r.H < 1 || r.W < 1 || r.Hm < 1 || r.Wm < 1)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: photo of %d x %d, mask of %d x %d", who, k, r.H, r.W, r.Hm, r.Wm);
        if (int rc = check_mask_channels(who, k, r.mask_channels)) return rc;
        if (eval) continue;
        int w1, h1, wa, ha, wb, hb;
        demo_resized_size(r.W, r.H, res, &w1, &h1);
        demo_resized_size(r.Wm, r.Hm, comod::DEMO_MASK_MAX, &wa, &ha);
        demo_resized_size(wa, ha, res, &wb, &hb);
        if (w1 < 1 || h1 < 1 || wa < 1 || ha < 1 || wb < 1 || hb < 1)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: a side resizes to 0 (photo %d x %d, mask %d x %d, resolution %d)", who, k,
                        r.W, r.H, r.Wm, r.Hm, res);
        if (wb != w1 || hb != h1)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: the mask resizes to %d x %d and the photo to %d x %d (w x h)", who, k, wb, hb, w1, h1);
        if (r.out_w != w1 || r.out_h != h1)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: output of %d x %d, the resized photo is %d x %d (w x h)", who, k, r.out_w,
                        r.out_h, w1, h1);
    }
    return MIGAN_OK;
}

size_t demo_scratch_bytes(const migan_demo_request* q, int n, int res) {
    comod::DemoBatch b;
    return demo_layout(q, n, res, nullptr, &b);
}

// Tables, the down-scale's two passes (only when a photo of the pass is larger than R) and the R x R resize into x.
int launch_demo_preprocess(const migan_demo_request* q, int n, int res, float* x, void* scratch, ck_stream_t s) {
    comod::DemoBatch b;
    demo_layout(q, n, res, scratch, &b);
    b.x = x;
    int e;
    comod::set_items(b, comod::DS_TABLES, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoTablesK>(b, s))) return e;
    comod::set_items(b, comod::DS_DOWN_W, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoDownWK>(b, s))) return e;
    comod::set_items(b, comod::DS_DOWN_H, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoDownHK>(b, s))) return e;
    comod::set_items(b, comod::DS_SQUARE, comod::demo_items);
    return (int)comod::batch_launch<comod::DemoSquareK>(b, s);
}

size_t eval_scratch_bytes(const migan_demo_request* q, int n, int res) {
    comod::DemoBatch b;
    return demo_layout(q, n, res, nullptr, &b, true);
}

// The demo's preprocess stages on the evaluation layout, with the unmasked photo values written to img as well.
int launch_eval_preprocess(const migan_demo_request* q, int n, int res, float* x, float* img, void* scratch, ck_stream_t s) {
    comod::DemoBatch b;
    demo_layout(q, n, res, scratch, &b, true);
    b.x = x;
    b.img = img;
    int e;
    comod::set_items(b, comod::DS_TABLES, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoTablesK>(b, s))) return e;
    comod::set_items(b, comod::DS_DOWN_W, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoDownWK>(b, s))) return e;
    comod::set_items(b, comod::DS_DOWN_H, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoDownHK>(b, s))) return e;
    comod::set_items(b, comod::DS_SQUARE, comod::demo_items);
    return (int)comod::batch_launch<comod::DemoSquareK>(b, s);
}

int launch_eval_composite(const float* x, const float* y, int n, int res, float* real, float* composed, ck_stream_t s) {
    const int64_t plane = (int64_t)res * res;
    return (int)comod::ck_launch(comod::EvalCompositeK{x, y, real, composed, plane}, n * plane, s);
}

// y -> uint8 + OpenCV width pass, then the height pass fused with the composite into each request's output.
int launch_demo_postprocess(const float* y, const migan_demo_request* q, int n, int res, void* scratch, ck_stream_t s) {
    comod::DemoBatch b;
    demo_layout(q, n, res, scratch, &b);
    b.y = y;
    int e;
    comod::set_items(b, comod::DS_POST_W, comod::demo_items);
    if ((e = (int)comod::batch_launch<comod::DemoPostWK>(b, s))) return e;
    comod::set_items(b, comod::DS_OUT, comod::demo_items);
    return (int)comod::batch_launch<comod::DemoOutK>(b, s);
}

}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

int migan_demo_resized_size(int w, int h, int max_size, int* out_w, int* out_h) {
    if (!out_w || !out_h) return fail(MIGAN_ERR_INVALID, "demo_resized_size: null argument");
    if (w < 1 || h < 1 || max_size < 1) return fail(MIGAN_ERR_INVALID, "demo_resized_size: bad arguments (%d x %d, max size %d)", w, h, max_size);
    return migan::demo_resized_size(w, h, max_size, out_w, out_h);
}

size_t b200_demo_scratch_bytes(const migan_demo_request* reqs, int n, int res) {
    if (migan::check_demo_batch("demo_scratch_bytes", reqs, n, res, false)) return 0;
    return migan::demo_scratch_bytes(reqs, n, res);
}

int b200_demo_preprocess(const migan_demo_request* reqs, int n, int res, float* x, void* scratch, size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_demo_batch("demo_preprocess", reqs, n, res, false)) return rc;
    if (!x || !scratch) return fail(MIGAN_ERR_INVALID, "demo_preprocess: null argument");
    const size_t need = migan::demo_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "demo_preprocess: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_demo_preprocess(reqs, n, res, x, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_demo_postprocess(const float* y, const migan_demo_request* reqs, int n, int res, void* scratch, size_t scratch_bytes,
                          void* stream) {
    if (int rc = migan::check_demo_batch("demo_postprocess", reqs, n, res, false)) return rc;
    if (!y || !scratch) return fail(MIGAN_ERR_INVALID, "demo_postprocess: null argument");
    const size_t need = migan::demo_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "demo_postprocess: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_demo_postprocess(y, reqs, n, res, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

size_t b200_eval_scratch_bytes(const migan_demo_request* reqs, int n, int res) {
    if (migan::check_demo_batch("eval_scratch_bytes", reqs, n, res, true)) return 0;
    return migan::eval_scratch_bytes(reqs, n, res);
}

int b200_eval_preprocess(const migan_demo_request* reqs, int n, int res, float* x, float* img, void* scratch,
                         size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_demo_batch("eval_preprocess", reqs, n, res, true)) return rc;
    if (!x || !img || !scratch) return fail(MIGAN_ERR_INVALID, "eval_preprocess: null argument");
    const size_t need = migan::eval_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "eval_preprocess: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_eval_preprocess(reqs, n, res, x, img, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_eval_composite(const float* x, const float* y, int n, int res, float* img, float* composed, void* stream) {
    if (!x || !y || !img || !composed) return fail(MIGAN_ERR_INVALID, "eval_composite: null argument");
    if (n < 1 || res < 1 || res > 8192) return fail(MIGAN_ERR_INVALID, "eval_composite: %d images at resolution %d", n, res);
    CUDA_TRY(migan::launch_eval_composite(x, y, n, res, img, composed, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

}  // extern "C"

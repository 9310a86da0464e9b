// Free-form masks of the evaluation protocol: RandomMask(s) of scripts/generate_masks.py (which the evaluation script's
// InferenceDataset also calls) and RandomMask(s, hole_range), identical bytes at the same position of numpy's legacy
// global stream.
//
//   migan_np_seed -> migan_mask_plan (host: numpy's RandomState draws, one fixed-size record per attempt)
//   --H2D--> mask_raster_kernel (an attempt's row band per CTA: rectangles, brush quads and discs painted as bit rows in
//   shared memory, 16-byte stores of 255 / 0, one hole-count atomic per CTA) -> mask_compact_kernel (the first n
//   attempts with h_min <= holes <= h_max, in attempt order; (0, s^2) for hole_range [0, 1])
//
// The brush is Pillow's (12.x) ImageDraw: a polyline of width w is the union of its two-point wide lines; each is a quad
// filled by Pillow's polygon scanline rule, which is not translation-invariant, so the quad rows are computed at absolute
// coordinates with Pillow's float32 operations each rounded on its own (PP_MUL / PP_ADD / PP_DIV of prepost.cuh), and the
// vertex discs are one fixed stamp per radius (kDiscHalf).  The brush is painted at the un-flipped coordinates and each
// span mirrored into the output, so the flips cost nothing.  oracle/masks_oracle.py states the same rules in numpy.
// The emulation build (tests/emul/build_emul.py) runs the same block functions with the threads of a block in turn.
#include "prepost.cuh"
#include "abi_error.h"

#include <cmath>
#include <cstring>

namespace comod {

constexpr int MK_THREADS = 256;
constexpr int MK_BAND = 16;                                  // output rows per CTA
constexpr int MK_W32_MAX = MIGAN_MASK_MAX_SIZE / 32;         // 32-bit words of a bit row at the largest s

#ifdef MIGAN_EMULATE
#define MK_CONST static const
#else
#define MK_CONST __constant__
#endif

// Half-width of Pillow's ellipse((x - r, y - r, x + r, y + r)) on row y + dy: kDiscHalf[r - 6][|dy|], r = 6..23 (width // 2
// for the widths 12..47 RandomBrush draws).  Every row of the stamp is one span centred on x; at the canvas edge the stamp
// is cropped.
MK_CONST uint8_t kDiscHalf[18][24] = {
    {6, 6, 6, 5, 4, 3, 2},
    {7, 7, 7, 6, 6, 5, 4, 2},
    {8, 8, 8, 7, 7, 6, 5, 4, 2},
    {9, 9, 9, 8, 8, 7, 7, 6, 4, 2},
    {10, 10, 10, 10, 9, 9, 8, 7, 6, 5, 3},
    {11, 11, 11, 11, 10, 10, 9, 8, 8, 6, 5, 3},
    {12, 12, 12, 12, 11, 11, 10, 10, 9, 8, 7, 5, 3},
    {13, 13, 13, 13, 12, 12, 12, 11, 10, 9, 8, 7, 6, 3},
    {14, 14, 14, 14, 13, 13, 13, 12, 11, 11, 10, 9, 7, 6, 3},
    {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3},
    {16, 16, 16, 16, 15, 15, 15, 14, 14, 13, 12, 12, 11, 9, 8, 6, 3},
    {17, 17, 17, 17, 17, 16, 16, 15, 15, 14, 14, 13, 12, 11, 10, 8, 6, 4},
    {18, 18, 18, 18, 18, 17, 17, 17, 16, 16, 15, 14, 13, 12, 11, 10, 9, 7, 4},
    {19, 19, 19, 19, 19, 18, 18, 18, 17, 17, 16, 15, 15, 14, 13, 12, 10, 9, 7, 4},
    {20, 20, 20, 20, 20, 19, 19, 19, 18, 18, 17, 17, 16, 15, 14, 13, 12, 11, 9, 7, 4},
    {21, 21, 21, 21, 21, 20, 20, 20, 19, 19, 18, 18, 17, 16, 16, 15, 14, 12, 11, 9, 7, 4},
    {22, 22, 22, 22, 22, 21, 21, 21, 20, 20, 20, 19, 18, 18, 17, 16, 15, 14, 13, 11, 10, 7, 4},
    {23, 23, 23, 23, 23, 22, 22, 22, 22, 21, 21, 20, 20, 19, 18, 17, 17, 16, 14, 13, 12, 10, 8, 4},
};

// An attempt is kept when its hole count lies in [h_min, h_max] (migan_mask_hole_bounds; (0, s^2) for hole_range [0, 1]).
CK_HD bool mask_accepted(int holes, int h_min, int h_max) { return holes >= h_min && holes <= h_max; }

// Pillow's ROUND_UP / ROUND_DOWN of a float: f + 0.5f / f - 0.5f in float for f >= 0, |f| +- 0.5 in double below.
PP_D int mk_round_up(float f) { return f >= 0.f ? (int)floorf(PP_ADD(f, 0.5f)) : -(int)floor(fabs((double)f) + 0.5); }
PP_D int mk_round_down(float f) { return f >= 0.f ? (int)ceilf(PP_ADD(f, -0.5f)) : -(int)ceil(fabs((double)f) - 0.5); }

struct MkEdge { int x0, y0, ymin, ymax; float dx; };
PP_D float mk_edge_x(const MkEdge& e, int y) { return PP_ADD(PP_MUL((float)(y - e.y0), e.dx), (float)e.x0); }

// xx[i] = v for a run-time i, with every index constant after unrolling (the list stays in registers).
PP_D void mk_set(float (&xx)[8], int i, float v) {
#pragma unroll
    for (int q = 0; q < 8; ++q)
        if (q == i) xx[q] = v;
}

// The spans Pillow's polygon fill paints on row y for the quad q = (x, y) x 4 on an s x s canvas: span(a, b) for each
// inclusive span before clipping (horizontal edges first, then the scanline pairs).  Pillow's edge table holds the
// non-horizontal edges in order; `rank` is an edge's index there.
template <class F>
PP_D void mk_quad_row(const int16_t* q, int s, int y, F&& span) {
    MkEdge e[4];
    bool flat[4];
    int ymin = s - 1, ymax = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int xa = q[2 * i], ya = q[2 * i + 1], xb = q[(2 * i + 2) & 7], yb = q[(2 * i + 3) & 7];
        const int lo = ya < yb ? ya : yb, hi = ya < yb ? yb : ya;
        ymin = lo < ymin ? lo : ymin;
        ymax = hi > ymax ? hi : ymax;
        flat[i] = ya == yb;                                  // drawn as a line, left out of the edge table
        if (flat[i] && y == ya) span(xa < xb ? xa : xb, xa < xb ? xb : xa);
        e[i] = MkEdge{xa, ya, lo, hi, flat[i] ? 0.f : PP_DIV((float)(xb - xa), (float)(yb - ya))};
    }
    ymin = ymin < 0 ? 0 : ymin;
    ymax = ymax > s ? s : ymax;
    if (y < ymin || y > ymax) return;
    float xx[8];
    int j = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (flat[i] || y < e[i].ymin || y > e[i].ymax) continue;
        const float x = mk_edge_x(e[i], y);
        mk_set(xx, j++, x);
        if (y == e[i].ymax && y < ymax) {                    // an edge's last row lists its x twice
            mk_set(xx, j++, x);
        } else if (e[i].dx != 0.f && (j & 1) && floorf(x) == x) {
            bool done = false;                               // a corner with an earlier edge of the same slope sign
            int rank = 0;
#pragma unroll
            for (int k = 0; k < i; ++k) {
                if (flat[k]) continue;
                const MkEdge& o = e[k];
                const bool same = !((e[i].dx > 0.f && o.dx <= 0.f) || (e[i].dx < 0.f && o.dx >= 0.f));
                if (!done && same && x == mk_edge_x(o, y)) {
                    const int off = y == ymax ? -1 : 1;
                    const float a = mk_edge_x(e[i], y + off), b = mk_edge_x(o, y + off);
                    float v;
                    if (y == e[i].ymax) v = e[i].dx > 0.f ? PP_ADD(fmaxf(a, b), 1.f) : PP_ADD(fminf(a, b), -1.f);
                    else v = e[i].dx > 0.f ? fminf(a, b) : PP_ADD(fmaxf(a, b), 1.f);
                    mk_set(xx, rank, v);                     // Pillow overwrites the entry at the edge's table index
                    done = true;
                }
                ++rank;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q)
        if (q >= j) xx[q] = INFINITY;
#pragma unroll
    for (int p = 0; p < 8; ++p)                              // odd-even transposition sort
#pragma unroll
        for (int q = p & 1; q + 1 < 8; q += 2)
            if (xx[q + 1] < xx[q]) { const float v = xx[q]; xx[q] = xx[q + 1]; xx[q + 1] = v; }
#pragma unroll
    for (int i = 1; i < 8; i += 2)
        if (i < j) span(mk_round_up(xx[i - 1]), mk_round_down(xx[i]));
}

PP_D void mk_or(uint32_t* w, uint32_t m) {
#ifdef MIGAN_EMULATE
    *w |= m;
#else
    atomicOr(w, m);
#endif
}

// Sets columns [a, b] (clipped to the canvas; mirrored when flip) of one bit row.
PP_D void mk_fill(uint32_t* row, int s, int a, int b, bool flip) {
    a = a < 0 ? 0 : a;
    b = b > s - 1 ? s - 1 : b;
    if (a > b) return;
    if (flip) { const int t = s - 1 - b; b = s - 1 - a; a = t; }
    for (int w = a >> 5; w <= b >> 5; ++w) {
        const int lo = a > 32 * w ? a & 31 : 0, hi = b < 32 * w + 31 ? b & 31 : 31;
        mk_or(row + w, (0xFFFFFFFFu >> (31 - hi)) & (0xFFFFFFFFu << lo));
    }
}

// Thread tid of nthr: every (primitive, row) item of output rows [y0, y0 + rows) of attempt `r`; bits [rows][w32] = 1
// where a hole is.  Rectangles are at output coordinates; the brush is evaluated on the un-flipped row and mirrored.
PP_D void mask_band_paint(const migan_mask_record& r, int s, int y0, int rows, int w32, int tid, int nthr, uint32_t* bits) {
    const int nr = r.n_rects, nq = r.n_segments, items = (nr + nq + r.n_discs) * rows;
    const bool flip_cols = (r.flips & 2) != 0;
    for (int i = tid; i < items; i += nthr) {
        const int p = i / rows, ro = i - p * rows, y = y0 + ro;
        uint32_t* row = bits + ro * w32;
        if (p < nr) {
            const int16_t* q = r.rects[p];
            if (y >= q[0] && y < q[1]) mk_fill(row, s, q[2], q[3] - 1, false);
            continue;
        }
        const int yb = (r.flips & 1) ? s - 1 - y : y;
        if (p < nr + nq) {
            const int16_t* q = r.quads[p - nr];
            if ((yb < q[1] && yb < q[3] && yb < q[5] && yb < q[7]) || (yb > q[1] && yb > q[3] && yb > q[5] && yb > q[7]))
                continue;                                    // outside the quad's rows
            mk_quad_row(q, s, yb, [&](int a, int b) { mk_fill(row, s, a, b, flip_cols); });
        } else {
            const int16_t* d = r.discs[p - nr - nq];
            const int dy = yb - d[1] < 0 ? d[1] - yb : yb - d[1];
            if (dy > d[2]) continue;
            const int hw = kDiscHalf[d[2] - 6][dy];
            mk_fill(row, s, d[0] - hw, d[0] + hw, flip_cols);
        }
    }
}

// Thread tid of nthr: the band's bytes (255 known, 0 hole) in 16-column chunks, one 16-byte store each when s % 16 == 0;
// returns the thread's hole count.
PP_D int mask_band_store(int s, int y0, int rows, int w32, int tid, int nthr, const uint32_t* bits, uint8_t* out) {
    const int nck = (s + 15) >> 4;
    int holes = 0;
    for (int i = tid; i < rows * nck; i += nthr) {
        const int ro = i / nck, x0 = (i - ro * nck) * 16, n = s - x0 < 16 ? s - x0 : 16;
        uint32_t b = (bits[ro * w32 + (x0 >> 5)] >> (x0 & 16)) & 0xFFFFu;
        if (n < 16) b &= (1u << n) - 1u;
#ifdef MIGAN_EMULATE
        holes += __builtin_popcount(b);
#else
        holes += __popc(b);
#endif
        uint8_t* dst = out + (int64_t)(y0 + ro) * s + x0;
        if (n == 16 && (s & 15) == 0) {
            uint32_t w[4];
            for (int k = 0; k < 4; ++k) {
                uint32_t v = 0;
                for (int t = 0; t < 4; ++t)
                    if (!((b >> (4 * k + t)) & 1u)) v |= 0xFFu << (8 * t);
                w[k] = v;
            }
#ifdef MIGAN_EMULATE
            memcpy(dst, w, 16);
#else
            *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
#endif
        } else {
            for (int t = 0; t < n; ++t) dst[t] = ((b >> t) & 1u) ? 0 : 255;
        }
    }
    return holes;
}

#ifdef MIGAN_EMULATE
inline int mask_raster_launch(const migan_mask_record* recs, int n_att, int s, uint8_t* attempts, int* holes, ck_stream_t) {
    const int w32 = (s + 31) / 32, nband = (s + MK_BAND - 1) / MK_BAND;
#pragma omp parallel for schedule(static)
    for (int a = 0; a < n_att; ++a) {
        static thread_local uint32_t bits[MK_BAND * MK_W32_MAX];
        int h = 0;
        for (int band = 0; band < nband; ++band) {
            const int y0 = band * MK_BAND, rows = s - y0 < MK_BAND ? s - y0 : MK_BAND;
            memset(bits, 0, sizeof(uint32_t) * rows * w32);
            uint8_t* out = attempts + (int64_t)a * s * s;
            for (int tid = 0; tid < MK_THREADS; ++tid) mask_band_paint(recs[a], s, y0, rows, w32, tid, MK_THREADS, bits);
            for (int tid = 0; tid < MK_THREADS; ++tid) h += mask_band_store(s, y0, rows, w32, tid, MK_THREADS, bits, out);
        }
        holes[a] = h;
    }
    return 0;
}

inline int mask_compact_launch(const uint8_t* attempts, const int* holes, int n_att, int s, int h_min, int h_max, int n,
                               uint8_t* out, ck_stream_t) {
    for (int a = 0, j = 0; a < n_att && j < n; ++a)
        if (mask_accepted(holes[a], h_min, h_max)) memcpy(out + (int64_t)(j++) * s * s, attempts + (int64_t)a * s * s, (size_t)s * s);
    return 0;
}
#else
__global__ void __launch_bounds__(MK_THREADS) mask_raster_kernel(const migan_mask_record* __restrict__ recs, int s, int w32,
                                                                 uint8_t* __restrict__ attempts, int* __restrict__ holes) {
    __shared__ uint32_t bits[MK_BAND * MK_W32_MAX];
    __shared__ int block_holes;
    const int a = blockIdx.y, y0 = blockIdx.x * MK_BAND, rows = min(MK_BAND, s - y0);
    for (int i = threadIdx.x; i < rows * w32; i += MK_THREADS) bits[i] = 0;
    if (threadIdx.x == 0) block_holes = 0;
    __syncthreads();
    mask_band_paint(recs[a], s, y0, rows, w32, threadIdx.x, MK_THREADS, bits);
    __syncthreads();
    int h = mask_band_store(s, y0, rows, w32, threadIdx.x, MK_THREADS, bits, attempts + (int64_t)a * s * s);
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xFFFFFFFFu, h, o);
    if ((threadIdx.x & 31) == 0 && h) atomicAdd(&block_holes, h);
    __syncthreads();
    if (threadIdx.x == 0 && block_holes) atomicAdd(holes + a, block_holes);
}

// blockIdx.y = output mask j: warp 0 finds the j-th accepted attempt (ballots over the hole counts in attempt order), then
// the block copies its chunk blockIdx.x of s * s bytes (16-byte copies when both planes are 16-byte aligned).
constexpr int MK_COPY_BYTES = MK_THREADS * 16 * 4;
__global__ void __launch_bounds__(MK_THREADS) mask_compact_kernel(const uint8_t* __restrict__ attempts,
                                                                  const int* __restrict__ holes, int n_att, int s,
                                                                  int h_min, int h_max, uint8_t* __restrict__ out) {
    __shared__ int src;
    const int j = blockIdx.y;
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        int seen = 0, found = -1;
        for (int base = 0; base < n_att && found < 0; base += 32) {
            const int a = base + lane;
            const unsigned m = __ballot_sync(0xFFFFFFFFu, a < n_att && mask_accepted(holes[a], h_min, h_max));
            const int c = __popc(m);
            if (seen + c > j) {
                unsigned mm = m;
                for (int t = 0; t < j - seen; ++t) mm &= mm - 1u;
                found = base + __ffs(mm) - 1;
            }
            seen += c;
        }
        if (lane == 0) src = found;
    }
    __syncthreads();
    if (src < 0) return;
    const int64_t plane = (int64_t)s * s, beg = (int64_t)blockIdx.x * MK_COPY_BYTES;
    const int64_t end = plane - beg < MK_COPY_BYTES ? plane : beg + MK_COPY_BYTES;
    const uint8_t* from = attempts + (int64_t)src * plane;
    uint8_t* to = out + (int64_t)j * plane;
    if (((plane | reinterpret_cast<uintptr_t>(from) | reinterpret_cast<uintptr_t>(to)) & 15) == 0) {
        for (int64_t o = beg + 16 * threadIdx.x; o < end; o += 16 * MK_THREADS)
            *reinterpret_cast<uint4*>(to + o) = *reinterpret_cast<const uint4*>(from + o);
    } else {
        for (int64_t o = beg + threadIdx.x; o < end; o += MK_THREADS) to[o] = from[o];
    }
}

inline cudaError_t mask_raster_launch(const migan_mask_record* recs, int n_att, int s, uint8_t* attempts, int* holes,
                                      ck_stream_t st) {
    if (cudaError_t e = cudaMemsetAsync(holes, 0, sizeof(int) * n_att, st)) return e;
    mask_raster_kernel<<<dim3((s + MK_BAND - 1) / MK_BAND, n_att), MK_THREADS, 0, st>>>(recs, s, (s + 31) / 32, attempts, holes);
    return cudaGetLastError();
}

inline cudaError_t mask_compact_launch(const uint8_t* attempts, const int* holes, int n_att, int s, int h_min, int h_max,
                                       int n, uint8_t* out, ck_stream_t st) {
    const int64_t plane = (int64_t)s * s;
    mask_compact_kernel<<<dim3((unsigned)((plane + MK_COPY_BYTES - 1) / MK_COPY_BYTES), n), MK_THREADS, 0, st>>>(
        attempts, holes, n_att, s, h_min, h_max, out);
    return cudaGetLastError();
}
#endif

}  // namespace comod

namespace migan {

namespace {

// ---- numpy's legacy RandomState (MT19937 + the legacy distributions), keeping numpy's state ------------------------
constexpr int MT_N = 624, MT_M = 397;

void mt_twist(migan_np_random& st) {
    uint32_t* k = st.key;
    auto mix = [](uint32_t hi, uint32_t lo, uint32_t far) {
        const uint32_t y = (hi & 0x80000000u) | (lo & 0x7fffffffu);
        return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    };
    int i = 0;
    for (; i < MT_N - MT_M; ++i) k[i] = mix(k[i], k[i + 1], k[i + MT_M]);
    for (; i < MT_N - 1; ++i) k[i] = mix(k[i], k[i + 1], k[i + MT_M - MT_N]);
    k[MT_N - 1] = mix(k[MT_N - 1], k[0], k[MT_M - 1]);
    st.pos = 0;
}

uint32_t next_u32(migan_np_random& st) {
    if (st.pos >= MT_N) mt_twist(st);
    uint32_t y = st.key[st.pos++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

double next_double(migan_np_random& st) {                    // random(): 53 bits from two words
    const int32_t a = (int32_t)(next_u32(st) >> 5), b = (int32_t)(next_u32(st) >> 6);
    return (a * 67108864.0 + b) / 9007199254740992.0;
}

int64_t randint(migan_np_random& st, int64_t lo, int64_t hi) {   // [lo, hi): masked rejection on 32-bit words
    const uint64_t rng = (uint64_t)(hi - lo - 1);
    if (rng == 0) return lo;
    if (rng == 0xFFFFFFFFull) return lo + next_u32(st);
    uint64_t mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    uint64_t v;
    while ((v = (next_u32(st) & mask)) > rng) {}
    return lo + (int64_t)v;
}

double uniform(migan_np_random& st, double a, double b) {
    const double range = b - a;
    return a + range * next_double(st);
}

double gauss(migan_np_random& st) {                          // polar method; the second value is cached
    if (st.has_gauss) {
        st.has_gauss = 0;
        const double g = st.gauss;
        st.gauss = 0.0;
        return g;
    }
    double x1, x2, r2;
    do {
        x1 = 2.0 * next_double(st) - 1.0;
        x2 = 2.0 * next_double(st) - 1.0;
        const double p1 = x1 * x1, p2 = x2 * x2;             // separate roundings: numpy's build contracts nothing
        r2 = p1 + p2;
    } while (r2 >= 1.0 || r2 == 0.0);
    const double f = sqrt(-2.0 * log(r2) / r2);
    st.gauss = f * x1;
    st.has_gauss = 1;
    return f * x2;
}

double normal(migan_np_random& st, double loc, double scale) {
    const double g = scale * gauss(st);
    return loc + g;
}

double clip(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Pillow's ROUND_UP / ROUND_DOWN of a double (the wide line's offsets).
int round_up_d(double f) { return f >= 0 ? (int)floor(f + 0.5) : -(int)floor(fabs(f) + 0.5); }
int round_down_d(double f) { return f >= 0 ? (int)ceil(f - 0.5) : -(int)ceil(fabs(f) - 0.5); }

// Pillow's wide line from (x0, y0) to (x1, y1): the quad's vertices (x, y) x 4, or the point four times.
void wide_line_quad(int x0, int y0, int x1, int y1, int width, int16_t* q) {
    const int dx = x1 - x0, dy = y1 - y0;
    if (dx == 0 && dy == 0) {
        for (int i = 0; i < 4; ++i) { q[2 * i] = (int16_t)x0; q[2 * i + 1] = (int16_t)y0; }
        return;
    }
    const double big = hypot((double)dx, (double)dy), small = (width - 1) / 2.0;
    const double rmax = round_up_d(small) / big, rmin = round_down_d(small) / big;
    const int dxmin = round_down_d(rmin * dy), dxmax = round_down_d(rmax * dy);
    const int dymin = round_down_d(rmin * dx), dymax = round_down_d(rmax * dx);
    const int v[8] = {x0 - dxmin, y0 + dymax, x1 - dxmin, y1 + dymax, x1 + dxmax, y1 - dymin, x0 + dxmax, y0 - dymin};
    for (int i = 0; i < 8; ++i) q[i] = (int16_t)v[i];
}

// One attempt of RandomMask(s, hole_range): its draws in the reference's order (scripts/generate_masks.py RandomMask /
// RandomBrush).  tries = {int(10 * coef), int(5 * coef), int(20 * coef)}; {10, 5, 20} for hole_range [0, 1].
void plan_attempt(migan_np_random& st, int s, const int (&tries)[3], migan_mask_record& r) {
    r.n_rects = r.n_segments = r.n_discs = 0;
    const int sizes[2] = {s / 2, s};
    for (int f = 0; f < 2; ++f) {
        const int64_t n = randint(st, 0, tries[f]);
        for (int64_t t = 0; t < n; ++t) {
            const int64_t w = randint(st, 0, sizes[f]), h = randint(st, 0, sizes[f]);
            const int64_t x = randint(st, -(w / 2), s - w + w / 2), y = randint(st, -(h / 2), s - h + h / 2);
            int16_t* q = r.rects[r.n_rects++];
            q[0] = (int16_t)(y > 0 ? y : 0); q[1] = (int16_t)(y + h < s ? y + h : s);
            q[2] = (int16_t)(x > 0 ? x : 0); q[3] = (int16_t)(x + w < s ? x + w : s);
        }
    }
    const double mean = 2 * M_PI / 5, spread = 2 * M_PI / 15;
    const double radius = sqrt((double)(s * s + s * s)) / 8, scale = floor(radius / 2);
    const int64_t ntry = randint(st, 0, tries[2]);
    for (int64_t t = 0; t < ntry; ++t) {
        const int nv = (int)randint(st, 4, 18);
        const double lo = mean - uniform(st, 0, spread);
        const double hi = mean + uniform(st, 0, spread);
        double angle[17];
        for (int i = 0; i < nv; ++i) angle[i] = i % 2 == 0 ? 2 * M_PI - uniform(st, lo, hi) : uniform(st, lo, hi);
        int px[18], py[18];
        px[0] = (int)randint(st, 0, s);
        py[0] = (int)randint(st, 0, s);
        for (int i = 0; i < nv; ++i) {
            const double rr = clip(normal(st, radius, scale), 0, 2 * radius);
            const double cx = rr * cos(angle[i]), sy = rr * sin(angle[i]);
            px[i + 1] = (int)clip(px[i] + cx, 0, s);
            py[i + 1] = (int)clip(py[i] + sy, 0, s);
        }
        const int width = (int)uniform(st, 12, 48);
        for (int i = 0; i < nv; ++i) wide_line_quad(px[i], py[i], px[i + 1], py[i + 1], width, r.quads[r.n_segments++]);
        for (int i = 0; i <= nv; ++i) {
            int16_t* d = r.discs[r.n_discs++];
            d[0] = (int16_t)px[i]; d[1] = (int16_t)py[i]; d[2] = (int16_t)(width / 2); d[3] = 0;
        }
        next_double(st);                                     // the try's two transposes, whose results are discarded
        next_double(st);
    }
    r.flips = next_double(st) > 0.5 ? 1 : 0;
    r.flips |= next_double(st) > 0.5 ? 2 : 0;
}

}  // namespace

void np_seed(migan_np_random* st, uint32_t seed) {
    for (int i = 0; i < MT_N; ++i) {
        st->key[i] = seed;
        seed = 1812433253u * (seed ^ (seed >> 30)) + (uint32_t)i + 1u;
    }
    st->pos = MT_N;
    st->has_gauss = 0;
    st->gauss = 0.0;
}

int check_mask_size(const char* who, int s, int n_att) {
    if (s < MIGAN_MASK_MIN_SIZE || s > MIGAN_MASK_MAX_SIZE)
        return fail(MIGAN_ERR_INVALID, "%s: mask size %d (%d to %d)", who, s, MIGAN_MASK_MIN_SIZE, MIGAN_MASK_MAX_SIZE);
    if (n_att < 1 || n_att > MIGAN_MASK_MAX_ATTEMPTS)
        return fail(MIGAN_ERR_INVALID, "%s: %d attempts (1 to %d per call)", who, n_att, MIGAN_MASK_MAX_ATTEMPTS);
    return MIGAN_OK;
}

// RandomMask's coef = min(lo + hi, 1.0) and its tries int(10 * coef), int(5 * coef), int(20 * coef), as Python evaluates
// them in float64.  Refuses a range outside 0 <= lo < hi <= 1 and one with int(5 * coef) == 0 (lo + hi < 0.2), where
// numpy's randint(0) raises.
int hole_range_tries(const char* who, double lo, double hi, int (&tries)[3]) {
    if (!(std::isfinite(lo) && std::isfinite(hi) && 0.0 <= lo && lo < hi && hi <= 1.0))
        return fail(MIGAN_ERR_INVALID, "%s: hole_range [%.17g, %.17g] (0 <= lo < hi <= 1)", who, lo, hi);
    const double sum = lo + hi, coef = sum < 1.0 ? sum : 1.0;
    tries[0] = (int)(10.0 * coef);
    tries[1] = (int)(5.0 * coef);
    tries[2] = (int)(20.0 * coef);
    if (tries[1] == 0)
        return fail(MIGAN_ERR_INVALID, "%s: hole_range [%.17g, %.17g] draws randint(int(5 * %.17g)) = randint(0), which numpy "
                    "refuses (lo + hi >= 0.2)", who, lo, hi, coef);
    return MIGAN_OK;
}

// The hole counts RandomMask(s, [lo, hi]) keeps: hole_ratio = 1 - np.mean(mask) = 1 - fl(k / s^2) with k = s^2 - holes
// known pixels, rejected when hole_ratio <= lo or hole_ratio >= hi.  hole_ratio never decreases with the hole count, so
// the kept counts are one interval [*h_min, *h_max] (empty when *h_min > *h_max), found by bisection.
static double hole_ratio(int holes, int s) {
    const double n = (double)s * s;
    return 1.0 - (n - holes) / n;
}

int hole_bounds(int s, double lo, double hi, int* h_min, int* h_max) {
    int tries[3];
    if (int rc = hole_range_tries("mask_hole_bounds", lo, hi, tries)) return rc;
    const int n = s * s;
    int a = 0, b = n + 1;                                    // above lo: never at 0 holes; b = n + 1 stands for none
    while (b - a > 1) {
        const int m = a + (b - a) / 2;
        (hole_ratio(m, s) > lo ? b : a) = m;
    }
    *h_min = b;
    a = -1, b = n;                                           // below hi: never at n holes; a = -1 stands for none
    while (b - a > 1) {
        const int m = a + (b - a) / 2;
        (hole_ratio(m, s) < hi ? a : b) = m;
    }
    *h_max = a;
    return MIGAN_OK;
}

int mask_plan(migan_np_random* st, int s, const int (&tries)[3], int n_att, migan_mask_record* recs,
              migan_np_random* states) {
    if (int rc = check_mask_size("mask_plan", s, n_att)) return rc;
    if (st->pos < 0 || st->pos > MT_N) return fail(MIGAN_ERR_INVALID, "mask_plan: state position %d (0 to %d)", st->pos, MT_N);
    for (int k = 0; k < n_att; ++k) {
        plan_attempt(*st, s, tries, recs[k]);
        if (states) states[k] = *st;
    }
    return MIGAN_OK;
}

int launch_mask_raster(const migan_mask_record* recs, int n_att, int s, uint8_t* attempts, int* holes, ck_stream_t st) {
    return (int)comod::mask_raster_launch(recs, n_att, s, attempts, holes, st);
}

int launch_mask_compact(const uint8_t* attempts, const int* holes, int n_att, int s, int h_min, int h_max, int n,
                        uint8_t* out, ck_stream_t st) {
    if (n < 1) return 0;
    return (int)comod::mask_compact_launch(attempts, holes, n_att, s, h_min, h_max, n, out, st);
}

}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

int migan_np_seed(migan_np_random* state, uint32_t seed) {
    if (!state) return fail(MIGAN_ERR_INVALID, "np_seed: null state");
    migan::np_seed(state, seed);
    return MIGAN_OK;
}

int migan_mask_plan(migan_np_random* state, int s, int n_attempts, migan_mask_record* records, migan_np_random* states) {
    if (!state || !records) return fail(MIGAN_ERR_INVALID, "mask_plan: null argument");
    return migan::mask_plan(state, s, {10, 5, 20}, n_attempts, records, states);
}

int migan_mask_plan_range(migan_np_random* state, int s, double lo, double hi, int n_attempts, migan_mask_record* records,
                          migan_np_random* states) {
    if (!state || !records) return fail(MIGAN_ERR_INVALID, "mask_plan_range: null argument");
    int tries[3];
    if (int rc = migan::hole_range_tries("mask_plan_range", lo, hi, tries)) return rc;
    return migan::mask_plan(state, s, tries, n_attempts, records, states);
}

int migan_mask_hole_bounds(int s, double lo, double hi, int* h_min, int* h_max) {
    if (!h_min || !h_max) return fail(MIGAN_ERR_INVALID, "mask_hole_bounds: null argument");
    if (s < MIGAN_MASK_MIN_SIZE || s > MIGAN_MASK_MAX_SIZE)
        return fail(MIGAN_ERR_INVALID, "mask_hole_bounds: mask size %d (%d to %d)", s, MIGAN_MASK_MIN_SIZE, MIGAN_MASK_MAX_SIZE);
    return migan::hole_bounds(s, lo, hi, h_min, h_max);
}

int b200_mask_raster(const migan_mask_record* records, int n_attempts, int s, uint8_t* attempts, int* holes, void* stream) {
    if (int rc = migan::check_mask_size("mask_raster", s, n_attempts)) return rc;
    if (!records || !attempts || !holes) return fail(MIGAN_ERR_INVALID, "mask_raster: null argument");
    if (reinterpret_cast<uintptr_t>(attempts) & 15) return fail(MIGAN_ERR_INVALID, "mask_raster: attempts not 16-byte aligned");
    CUDA_TRY(migan::launch_mask_raster(records, n_attempts, s, attempts, holes, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_mask_compact_range(const uint8_t* attempts, const int* holes, int n_attempts, int s, int h_min, int h_max, int n,
                            uint8_t* out, void* stream) {
    if (int rc = migan::check_mask_size("mask_compact", s, n_attempts)) return rc;
    if (n < 0 || n > 65535) return fail(MIGAN_ERR_INVALID, "mask_compact: %d masks (0 to 65535 per call)", n);
    if (!attempts || !holes || (n && !out)) return fail(MIGAN_ERR_INVALID, "mask_compact: null argument");
    CUDA_TRY(migan::launch_mask_compact(attempts, holes, n_attempts, s, h_min, h_max, n, out, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_mask_compact(const uint8_t* attempts, const int* holes, int n_attempts, int s, int n, uint8_t* out, void* stream) {
    return b200_mask_compact_range(attempts, holes, n_attempts, s, 1, s * s - 1, n, out, stream);
}

}  // extern "C"

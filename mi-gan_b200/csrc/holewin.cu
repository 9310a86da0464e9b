// Hole-window request path: find the holes of a photo of any size and plan the windows around them that the
// full-resolution path (fullres.cu) inpaints; every pixel outside those windows keeps the photo's value.
//
//   mask u8 [H][W][C] --b200_hole_cells--> cells u8 [ceil(H/q)][ceil(W/q)] (1 = the q x q cell holds a hole pixel)
//   --D2H--> migan_hole_windows (host) -> windows {y0, x0, h, w} -> b200_window_preprocess -> forward_fc at the window's
//   padded extent -> b200_window_postprocess (fullres.cu's item functors on the window's crop)
//
// q = R / 4 is the granularity of forward_fc.  The cells kernel reads each mask byte once: a block covers one row of
// cells and up to HC_SEG_PX pixel columns, its threads walk the rows of the band in 16-byte aligned chunks (one 16-byte
// load when the chunk lies inside the row's bytes, byte loads at the ends), and a hole marks the cell's byte in shared
// memory; the block then writes one byte per cell, so every cell byte is written exactly once and needs no clearing.
// The hole test is prepost.cuh's (mask_channel + known_value), the same as the pre- and post-processing's.
// The kernel is one body over portable.cuh's block layer, which the emulation build (tests/emul/build_emul.py) runs on
// the host.
#include "prepost.cuh"
#include "abi_error.h"

#include <algorithm>
#include <cstring>
#include <vector>

namespace comod {

constexpr int HC_THREADS = 256;
constexpr int HC_SEG_PX = 512;                // pixel columns of a block (rounded down to whole cells, at least one)
constexpr int HC_MAX_S = HC_SEG_PX / 2;       // cells of a block at the smallest cell (q = 2, R = 8)

struct CellsReq { const uint8_t* mask; int H, W, C, invert, gh, gw, nseg; };
struct CellsBatch {
    int64_t block_start[MIGAN_PIPE_MAX_BATCH + 1];   // block prefix of the launch
    int64_t cell_start[MIGAN_PIPE_MAX_BATCH + 1];    // cell-byte prefix: request k's cells start at cell_start[k]
    CellsReq r[MIGAN_PIPE_MAX_BATCH];
    int n, qshift, S;                                // q = 1 << qshift; S cells per block
};
static_assert(sizeof(CellsBatch) <= 4000, "the batch descriptor must fit the classic 4 KB kernel parameter space");

// The cells of one block: request k, cell row cy, cell columns [cx0, cx0 + ncx); pixel rows [y0, y1), columns [px0, px1).
struct CellsBlock { int k, cy, cx0, ncx, y0, y1, px0, px1; };

CK_HD CellsBlock cells_block(const CellsBatch& b, int64_t blk) {
    CellsBlock g;
    g.k = find_request(b.block_start, b.n, blk);
    const CellsReq& r = b.r[g.k];
    const int64_t j = blk - b.block_start[g.k];
    g.cy = (int)(j / r.nseg);
    g.cx0 = (int)(j - (int64_t)g.cy * r.nseg) * b.S;
    g.ncx = r.gw - g.cx0 < b.S ? r.gw - g.cx0 : b.S;
    g.y0 = g.cy << b.qshift;
    g.y1 = r.H - g.y0 < (1 << b.qshift) ? r.H : g.y0 + (1 << b.qshift);
    g.px0 = g.cx0 << b.qshift;
    const int64_t px1 = (int64_t)(g.cx0 + g.ncx) << b.qshift;
    g.px1 = px1 < r.W ? (int)px1 : r.W;
    return g;
}

// Thread tid of nthr: the 16-byte chunks of the block's rows; flags[c] = 1 when cell cx0 + c holds a hole pixel.
CK_D void cells_block_scan(const CellsBatch& b, const CellsBlock& g, int tid, int nthr, uint8_t* flags) {
    const CellsReq& r = b.r[g.k];
    const int C = r.C, ch = mask_channel(C);
    const int64_t span = (int64_t)(g.px1 - g.px0) * C;            // bytes of the block's part of a row
    const int nck = (int)((span + 15) >> 4) + 1;                   // chunks a row part can touch
    const int items = (g.y1 - g.y0) * nck;                         // q x (max(HC_SEG_PX, q) x C / 16 + 2) at most
    const uintptr_t base = reinterpret_cast<uintptr_t>(r.mask);
    for (int i = tid; i < items; i += nthr) {
        const int y = g.y0 + i / nck, k = i % nck;
        const int64_t row = (int64_t)y * r.W * C;                  // byte offset of the row
        const int64_t rb0 = row + (int64_t)g.px0 * C, rb1 = rb0 + span;
        const int64_t co = (int64_t)(((base + rb0) & ~(uintptr_t)15) - base) + 16 * (int64_t)k;   // the chunk, from mask
        const int lo = rb0 > co ? (int)(rb0 - co) : 0;
        const int hi = rb1 - co < 16 ? (int)(rb1 - co) : 16;
        if (hi <= lo) continue;
        uint32_t w[4];
        if (lo == 0 && hi == 16) {
#ifdef MIGAN_EMULATE
            memcpy(w, r.mask + co, 16);
#else
            const uint4 u = *reinterpret_cast<const uint4*>(r.mask + co);
            w[0] = u.x; w[1] = u.y; w[2] = u.z; w[3] = u.w;
#endif
        } else {
#pragma unroll
            for (int t = 0; t < 4; ++t) w[t] = 0;
#pragma unroll
            for (int t = 0; t < 16; ++t)
                if (t >= lo && t < hi) w[t >> 2] |= (uint32_t)r.mask[co + t] << ((t & 3) * 8);
        }
        const int64_t rel = co + lo - row;                        // row-relative byte offset of chunk byte lo
        const int64_t x64 = C == 1 ? rel : (C == 2 ? rel >> 1 : (C == 4 ? rel >> 2 : rel / 3));
        int x = (int)x64, c = (int)(rel - x64 * C);
#pragma unroll
        for (int t = 0; t < 16; ++t) {
            if (t >= lo && t < hi) {
                if (c == ch && !known_value((int)((w[t >> 2] >> ((t & 3) * 8)) & 255u), r.invert))
                    flags[(x >> b.qshift) - g.cx0] = 1;
                if (++c == C) { c = 0; ++x; }
            }
        }
    }
}

CK_D void cells_block_store(const CellsBatch& b, const CellsBlock& g, int tid, int nthr, const uint8_t* flags,
                            uint8_t* cells) {
    const CellsReq& r = b.r[g.k];
    uint8_t* out = cells + b.cell_start[g.k] + (int64_t)g.cy * r.gw + g.cx0;
    for (int t = tid; t < g.ncx; t += nthr) out[t] = flags[t];
}

template <class B>
CK_D void hole_cells_block(const B& blk, const CellsBatch& b, int64_t blk_idx, uint8_t* flags, uint8_t* cells) {
    const CellsBlock g = cells_block(b, blk_idx);
    blk.each([&](int tid) {
        for (int t = tid; t < g.ncx; t += HC_THREADS) flags[t] = 0;
    });
    blk.sync();
    blk.each([&](int tid) { cells_block_scan(b, g, tid, HC_THREADS, flags); });
    blk.sync();
    blk.each([&](int tid) { cells_block_store(b, g, tid, HC_THREADS, flags, cells); });
}

#ifdef MIGAN_EMULATE
inline int cells_launch(const CellsBatch& b, uint8_t* cells, ck_stream_t) {
    return ck_blocks<HC_THREADS>(b.block_start[b.n], HC_MAX_S,
                                 [&](auto& blk, int64_t k, void* flags) { hole_cells_block(blk, b, k, (uint8_t*)flags, cells); });
}
#else
__global__ void __launch_bounds__(HC_THREADS) hole_cells_kernel(const __grid_constant__ CellsBatch b, uint8_t* cells) {
    __shared__ uint8_t flags[HC_MAX_S];
    hole_cells_block(DeviceBlock(), b, blockIdx.x, flags, cells);
}
inline cudaError_t cells_launch(const CellsBatch& b, uint8_t* cells, ck_stream_t s) {
    hole_cells_kernel<<<(unsigned)b.block_start[b.n], HC_THREADS, 0, s>>>(b, cells);
    return cudaGetLastError();
}
#endif

}  // namespace comod

namespace migan {

namespace {

int log2_resolution(int res) {               // log2(R) for a power of two >= 8, else -1
    if (res < 8 || (res & (res - 1))) return -1;
    int s = 0;
    while ((1 << s) < res) ++s;
    return s;
}

comod::CellsBatch cells_batch(const migan_cells_request* q, int n, int res) {
    comod::CellsBatch b;
    b.n = n;
    b.qshift = log2_resolution(res) - 2;
    b.S = std::max(1, comod::HC_SEG_PX >> b.qshift);
    b.block_start[0] = b.cell_start[0] = 0;
    for (int k = 0; k < n; ++k) {
        comod::CellsReq& r = b.r[k];
        r.mask = q[k].mask; r.H = q[k].H; r.W = q[k].W; r.C = q[k].mask_channels; r.invert = q[k].invert != 0;
        r.gh = (int)(((int64_t)r.H + (1 << b.qshift) - 1) >> b.qshift);
        r.gw = (int)(((int64_t)r.W + (1 << b.qshift) - 1) >> b.qshift);
        r.nseg = (r.gw + b.S - 1) / b.S;
        b.block_start[k + 1] = b.block_start[k] + (int64_t)r.gh * r.nseg;
        b.cell_start[k + 1] = b.cell_start[k] + (int64_t)r.gh * r.gw;
    }
    return b;
}

struct Span { int64_t s, L; };

// The window rule on one axis of side n for the cell span [c0, c1] with a margin of m cells.
Span window_axis(int64_t c0, int64_t c1, int64_t n, int64_t R, int64_t q, int64_t m) {
    const int64_t a = std::max<int64_t>(0, (c0 - m) * q);
    const int64_t b = std::min<int64_t>(n, (c1 + 1 + m) * q);
    const int64_t L = std::min<int64_t>(n, std::max<int64_t>(R, (b - a + q - 1) / q * q));
    const int64_t s = std::min<int64_t>(std::max<int64_t>(a - (L - (b - a)) / 2, 0), n - L);
    return {s, L};
}

struct Win {
    int64_t r0, r1, c0, c1;   // the cell span: rows [r0, r1], columns [c0, c1]
    Span y, x;
};

}  // namespace

int check_hole_cells(const char* who, const migan_cells_request* q, int n, int res) {
    if (int rc = check_batch_size(who, q, n)) return rc;
    if (log2_resolution(res) < 0) return fail(MIGAN_ERR_INVALID, "%s: resolution %d (a power of two >= 8)", who, res);
    for (int k = 0; k < n; ++k) {
        if (!q[k].mask) return fail(MIGAN_ERR_INVALID, "%s: request %d: null mask", who, k);
        if (q[k].H < 1 || q[k].W < 1) return fail(MIGAN_ERR_INVALID, "%s: request %d: mask of %d x %d (H x W)", who, k, q[k].H, q[k].W);
        if (int rc = check_mask_channels(who, k, q[k].mask_channels)) return rc;
    }
    if (cells_batch(q, n, res).block_start[n] > INT32_MAX) return fail(MIGAN_ERR_INVALID, "%s: masks too large", who);
    return MIGAN_OK;
}

size_t hole_cells_bytes(const migan_cells_request* q, int n, int res) { return (size_t)cells_batch(q, n, res).cell_start[n]; }

int launch_hole_cells(const migan_cells_request* q, int n, int res, uint8_t* cells, ck_stream_t s) {
    return (int)comod::cells_launch(cells_batch(q, n, res), cells, s);
}

int hole_windows_max(const char* who, int H, int W, int res, int* max_windows) {
    if (H < 1 || W < 1 || log2_resolution(res) < 0)
        return fail(MIGAN_ERR_INVALID, "%s: photo of %d x %d (H x W) at resolution %d (a power of two >= 8)", who, H, W, res);
    const int64_t m = (int64_t)(H / std::min(res, H)) * (W / std::min(res, W));
    if (m > INT32_MAX) return fail(MIGAN_ERR_INVALID, "%s: photo of %d x %d (H x W): too many windows", who, H, W);
    *max_windows = (int)m;
    return MIGAN_OK;
}

int hole_windows(const uint8_t* cells, int H, int W, int res, int margin, int* win4, int max_windows, int* count) {
    int bound = 0;
    if (int rc = hole_windows_max("hole_windows", H, W, res, &bound)) return rc;
    if (margin < 0) return fail(MIGAN_ERR_INVALID, "hole_windows: margin of %d cells", margin);
    const int64_t R = res, q = res / 4;
    const int64_t gh = (H + q - 1) / q, gw = (W + q - 1) / q;
    auto make = [&](int64_t r0, int64_t r1, int64_t c0, int64_t c1) {
        return Win{r0, r1, c0, c1, window_axis(r0, r1, H, R, q, margin), window_axis(c0, c1, W, R, q, margin)};
    };
    auto overlap = [](const Span& a, const Span& b) { return a.s < b.s + b.L && b.s < a.s + a.L; };
    std::vector<Win> list;
    for (int64_t cy = 0; cy < gh; ++cy)
        for (int64_t cx = 0; cx < gw; ++cx) {
            if (!cells[cy * gw + cx]) continue;
            Win cur = make(cy, cy, cx, cx);
            for (;;) {
                auto it = std::find_if(list.begin(), list.end(),
                                       [&](const Win& w) { return overlap(cur.y, w.y) && overlap(cur.x, w.x); });
                if (it == list.end()) break;
                cur = make(std::min(cur.r0, it->r0), std::max(cur.r1, it->r1), std::min(cur.c0, it->c0), std::max(cur.c1, it->c1));
                list.erase(it);
            }
            list.push_back(cur);
        }
    std::sort(list.begin(), list.end(), [](const Win& a, const Win& b) { return a.y.s != b.y.s ? a.y.s < b.y.s : a.x.s < b.x.s; });
    if ((int64_t)list.size() > max_windows) return fail(MIGAN_ERR_INVALID, "hole_windows: %zu windows, room for %d", list.size(), max_windows);
    for (size_t k = 0; k < list.size(); ++k) {
        win4[4 * k] = (int)list[k].y.s; win4[4 * k + 1] = (int)list[k].x.s;
        win4[4 * k + 2] = (int)list[k].y.L; win4[4 * k + 3] = (int)list[k].x.L;
    }
    *count = (int)list.size();
    return MIGAN_OK;
}

}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

size_t b200_hole_cells_bytes(const migan_cells_request* reqs, int n, int res) {
    if (migan::check_hole_cells("hole_cells_bytes", reqs, n, res)) return 0;
    return migan::hole_cells_bytes(reqs, n, res);
}

int b200_hole_cells(const migan_cells_request* reqs, int n, int res, uint8_t* cells, void* stream) {
    if (int rc = migan::check_hole_cells("hole_cells", reqs, n, res)) return rc;
    if (!cells) return fail(MIGAN_ERR_INVALID, "hole_cells: null cells");
    CUDA_TRY(migan::launch_hole_cells(reqs, n, res, cells, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int migan_hole_windows_max(int H, int W, int res, int* max_windows) {
    if (!max_windows) return fail(MIGAN_ERR_INVALID, "hole_windows_max: null argument");
    return migan::hole_windows_max("hole_windows_max", H, W, res, max_windows);
}

int migan_hole_windows(const uint8_t* cells, int H, int W, int res, int margin, int* win4, int max_windows, int* count) {
    if (!cells || !win4 || !count) return fail(MIGAN_ERR_INVALID, "hole_windows: null argument");
    return migan::hole_windows(cells, H, W, res, margin, win4, max_windows, count);
}

}  // extern "C"

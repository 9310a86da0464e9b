// Fused SeparableConv2d on Hopper tensor cores (sm_90a): the hot kernel of the generator.
//
//   out = epi( PW( act( DW3x3( src ) + b ) ) )          lib/model_zoo/migan_inference.py:154-170
//
//   src                        where the depthwise conv's input comes from (SepconvSource):
//                                NHWC   a TMA-staged tile + 1-pixel halo of an NHWC fp32 tensor
//                                UP     rebuilt in shared memory from the PREVIOUS layer's raw low-resolution 1x1 output:
//                                       lrelu_agc(Upsample2d(t) + noise) + skip (:98-103, :165-169, :304-305) -- the
//                                       up-sampled tensor never exists in HBM
//                                STEM   fromrgb 1x1 (4 -> C0) + activation (:193-196) recomputed on the halo from the
//                                       generator input x -- the stem tensor never exists in HBM
//                                SPLIT  no depthwise stage: a pre-split fp16 hi/lo A operand is loaded by TMA
//   DW3x3 + bias + lrelu_agc   CUDA cores, fp32 (sepconv_stages.cuh)
//   PW (1x1 conv, Cin -> Cout) wgmma.mma_async m64nNk16 kind f16 with fp32 accumulators in registers: M = 128 pixels (two
//                              m64 instructions) x n_tile channels per CTA tile.  fp32-faithful mode (n_tile = 64): both
//                              operands are split into fp16 (hi, lo) pairs; main = Ah * Bh, corr = Ah * Bl + Al * Bh in
//                              separate accumulators, summed in the epilogue.  Fast mode (n_tile <= 128): Ah * Bh only.
//   epi                        registers: * 2^-k, + noise, lrelu_agc [-> torgb + image] -> NHWC fp32 (each quad of lanes
//                              writes 32 contiguous bytes per pixel row and column block)
//
// One persistent CTA per SM, 16 warps = 4 warpgroups, warp-specialised:
//   warpgroups 0-1  prologue       two groups of 4 warps: pre-stage (UP / STEM) + depthwise conv -> fp16 hi/lo A operand
//   warpgroup 2     MMA + epilogue issues the wgmma of an M tile, then drains its accumulators
//   warpgroup 3     TMA producer   one lane: input chunks, weight K blocks, L2 prefetch
// The accumulators of an M = 128 tile (main + corr of 64 channels, or 128 channels in fast mode) are 128 registers per thread of one warpgroup, so setmaxnreg moves
// registers from the producer warpgroup (which needs few) to the MMA warpgroup; the prologue keeps 128.
// All hand-offs are mbarrier pipelines (input ring, A ring, B ring).
//
// Stationary A (n_group > 1): a CTA tile is one pixel tile x n_group consecutive N tiles.  The A ring then has one slot
// per K block (a_stages = num_kb): the prologue runs once per pixel tile and the whole K extent of A stays resident
// while the MMA warpgroup walks the group's N tiles; a slot is released only after the group's last N tile has retired
// it.  n_group = 1 is the plain schedule (one N tile per CTA tile, A streamed through a shallow ring).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "sepconv_stages.cuh"
#include "sepconv_tc.h"

namespace migan {

namespace {

using namespace stages;

constexpr int kThreads = 512;      // 4 warpgroups
constexpr int kNumProWarps = 8;    // warps 0-7
constexpr int kMmaWarp0 = 8;       // warps 8-11: one warpgroup (wgmma is issued by all four warps together)
constexpr int kProducerWarp = 12;  // warps 12-15: lane 0 of warp 12 is the producer, the rest only release registers
constexpr int kProRegs = 144;      // setmaxnreg per thread: 2 x 144 (prologue) + 184 (MMA) + 40 (producer) = 4 x 128,
constexpr int kMmaRegs = 184;      // the whole register file
constexpr int kProducerRegs = 40;
constexpr int kTileM = 128;
constexpr int kMaxTileN = 128;     // accumulator registers of the MMA warpgroup: kMaxTileN per thread
constexpr int kKBlock = 64;        // channels per A/B stage (128 bytes of fp16: one SW128 row)
constexpr int kChunkC = 32;        // channels per input chunk (128 bytes of fp32)
constexpr uint32_t kABytes = kTileM * kKBlock * 2;   // 16 KB per hi or lo
constexpr uint32_t kAStage = 2 * kABytes;            // hi + lo
constexpr uint32_t kSmemLimit = 232448;              // 227 KB
constexpr int kMaxRgbC = 256;      // fused torgb: the widest cout whose weights the static table s_rgb holds
constexpr int kRgbBias = 3 * kMaxRgbC, kRgbFir = 3 * kMaxRgbC + 4;   // offsets inside the torgb table s_rgb
constexpr uint32_t kStaticSmem = 4096;               // barriers + torgb table (static __shared__), rounded up

struct Params {
    CUtensorMap map_in, map_t, map_aux, map_a_hi, map_a_lo, map_w_hi, map_w_lo;
    CUtensorMap map_nz, map_img;              // epilogue windows: noise [H][W] (pitch noise_pitch), img_lo [n][3][H/2][W/2]
    const float* w9;                          // [9][cin] depthwise taps * (kActSplitScale * sqrt 2)
    const float* bias;                        // [cin]              * (kActSplitScale * sqrt 2)
    const float* noise;                       // [H][noise_pitch]
    float* out;                               // NHWC output
    float inv_scale;
    int n, H, W, cin, cout, noise_pitch;
    int act, passes;
    int source;                               // SepconvSource
    int tile_n, tile_h, tile_w, n_tile;      // n_tile = output channels per N tile (64 or 128)
    int tiles_x, tiles_y, tiles_n, num_n_tiles, num_tiles;   // num_n_tiles = cout / n_tile; tiles_x = ceil(W / tile_w) ...
    int n_group;                              // N tiles per CTA tile (power of two; > 1: stationary A)
    int l_nt;                                 // log2 of num_n_tiles / n_group (a power of two)
    int l_tw, l_th;                           // log2 of tile_w / tile_h (powers of two): the epilogue's pixel decode
    FastDiv div_tx, div_ty;                   // by tiles_x / tiles_y (not powers of two at a rectangular extent)
    int num_kb;                               // cin / 64
    int in_stages, a_stages, b_stages, b_resident;
    uint32_t in_tx_bytes;                     // bytes the TMA unit delivers per input stage
    uint32_t in_stage_stride;                 // rounded to 1024
    uint32_t off_t, off_aux;                  // T / NZ|XA areas inside an input stage
    uint32_t off_in, off_a, off_b;            // smem offsets from the 1024-aligned base
    uint32_t off_dw;                          // [10][cin] depthwise taps + bias staged in smem (0xFFFFFFFF: read from global)
    uint32_t off_stem;                        // STEM: [cin][4] + [cin] fromrgb table
    int prefetch;                             // L2 prefetch distance of the producer, in chunks / K-blocks
    // UP pre-stage
    UpTaps up_taps;
    int up_has_noise;
    // STEM pre-stage
    const float* stem_w;
    const float* stem_b;
    // fused torgb + image path (SynthesisBlock.forward, migan_inference.py:308-313); needs all of cout in one CTA tile
    // (n_group == num_n_tiles)
    int torgb, store_out;
    const float* rgb_w;                       // [3][cout]
    const float* rgb_b;                       // [3]
    const float* rgb_fir;                     // [16][3] up-sampling taps of the image path
    const float* img_lo;                      // [n][3][H/2][W/2] planar, or null (first block)
    float* img_out;                           // [n][3][H][W] planar
    // Epilogue window ring: per CTA tile, the producer brings the tile's noise (NZ, tile_h x tile_w, at the stage's start)
    // and the low-resolution image window (IMG, [tile_n][3][img_bh][img_bw] at ep_off_img) into shared memory.  0 stages:
    // no ring (nothing to bring, or no room left by the layout); the epilogue then reads global memory.
    int ep_stages;
    uint32_t off_ep, ep_stage_stride, ep_off_img, ep_tx_bytes;
    int img_bw, img_bh;
    int* error_flag;
};

// ---------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint: the warp sleeps in hardware until the phase completes or the hint elapses,
// instead of burning issue slots.
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity), "r"(200000u) : "memory");
    return ok != 0;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// Bounded wait: a protocol bug must never hang the GPU -- record which wait gave up and trap instead.  The bound is
// wall-clock time (seconds), so a profiler replay or a co-tenant cannot turn a legitimately long wait into a false
// positive.  The record goes to a host-mapped word (it survives the trap).  The clock is only looked at every 1024
// failed probes: the common path is the probe loop alone.
__device__ __noinline__ void mbar_timeout(int code, uint32_t parity, int* error_flag) {
    if (error_flag) {
        *reinterpret_cast<volatile int*>(error_flag) = code | ((int)parity << 12) | ((int)(blockIdx.x & 0xFFF) << 16);
        __threadfence_system();
    }
    __trap();
}
// kRelaxed: a waiter with slack (the producer behind a ring) backs off between probes, so that it does not compete for
// issue slots with the warps doing the arithmetic.
template <bool kRelaxed = false>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int code, int* error_flag) {
    if (mbar_try_wait(bar, parity)) return;
    unsigned long long t0 = 0;
    for (;;) {
#pragma unroll 1
        for (int i = 0; i < 1024; ++i) {
            if (kRelaxed) asm volatile("nanosleep.u32 256;" ::: "memory");
            if (mbar_try_wait(bar, parity)) return;
        }
        const unsigned long long t = globaltimer_ns();
        if (t0 == 0) t0 = t;
        else if (t - t0 > 4000000000ull) mbar_timeout(code, parity, error_flag);
    }
}
__device__ __forceinline__ void bar_sync_named(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma: all 128 threads of the warpgroup issue together; the accumulators live in their registers.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Ties the accumulator registers to a point in the program: the compiler may not move their reads or writes across it
// (the asynchronous wgmma writes them until wg_wait).
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N> struct Wgmma;
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major fp16 in shared memory, fp32 accumulators.
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(accumulate));
    }
};
template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(accumulate));
    }
};

// wgmma shared-memory descriptor: K-major operand, 128-byte swizzle, rows of 64 fp16 (128 B), 8-row groups 1024 B apart
// (SBO).  Bit layout: cute/arch/mma_sm90_desc.hpp GmmaDescriptor.  Advancing the start address by 32 bytes steps 16
// elements along K inside the swizzled row; by 64 rows x 128 B it selects the second m64 half of the M tile.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // start address  [0,14)
    d |= (uint64_t)1 << 16;                              // LBO (unused for swizzled K-major) [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;                    // SBO = 1024 B   [32,46)
    d |= (uint64_t)1 << 62;                              // layout type: SWIZZLE_128B [62,64)
    return d;
}

struct TileCoord {
    int n0, y0, x0, nt;   // first image / row / column of the M tile, first N tile of the CTA tile's group
};
// Every source uses spatial tiles (tile_n images x tile_h rows x tile_w columns = 128 pixels).  The tile counts are not
// powers of two once the extents are not: two multiply-high divisions per tile (FastDiv), few registers -- the producer
// warpgroup decodes tiles under a 40-register budget.
__device__ __forceinline__ TileCoord decode_tile(const Params& p, int tile) {
    TileCoord c;
    c.nt = (tile & ((1 << p.l_nt) - 1)) * p.n_group;
    const uint32_t m = (uint32_t)tile >> p.l_nt;
    const uint32_t q = p.div_tx.div(m), q2 = p.div_ty.div(q);
    c.x0 = (int)(m - q * p.div_tx.d) * p.tile_w;
    c.y0 = (int)(q - q2 * p.div_ty.d) * p.tile_h;
    c.n0 = (int)q2 * p.tile_n;
    return c;
}

// Ring-buffer cursor: stage index + phase parity, advanced incrementally (no div/mod on the hot path).
struct Ring {
    int stage, phase, n, step;
    __device__ __forceinline__ Ring(int n_, int start = 0, int step_ = 1) : stage(start), phase(0), n(n_), step(step_) {}
    __device__ __forceinline__ void advance() {
        stage += step;
        if (stage >= n) { stage -= n; phase ^= 1; }
    }
};

// mbarriers: [0,8) full_in  [8,16) empty_in  [16,24) full_a  [24,32) empty_a  [32,40) full_b  [40,48) empty_b
//            [48,52) full_ep  [52,56) empty_ep
constexpr int kNumBars = 56;
constexpr int kMaxAStages = 8;
constexpr int kMaxEpStages = 4;
static_assert(kNumBars * 8 + (3 * kMaxRgbC + 4 + 48) * 4 <= (int)kStaticSmem, "static shared memory outgrew kStaticSmem");
__device__ __forceinline__ uint32_t bar_full_a(uint32_t bar0, int s) { return bar0 + 8u * (16 + s); }
__device__ __forceinline__ uint32_t bar_empty_a(uint32_t bar0, int s) { return bar0 + 8u * (24 + s); }
__device__ __forceinline__ uint32_t bar_full_b(uint32_t bar0, int s) { return bar0 + 8u * (32 + s); }
__device__ __forceinline__ uint32_t bar_empty_b(uint32_t bar0, int s) { return bar0 + 8u * (40 + s); }
__device__ __forceinline__ uint32_t bar_full_ep(uint32_t bar0, int s) { return bar0 + 8u * (48 + s); }
__device__ __forceinline__ uint32_t bar_empty_ep(uint32_t bar0, int s) { return bar0 + 8u * (52 + s); }
// Origin of a tile's low-resolution image window: one row above the tile's first tap row, and the first tap column
// rounded down to 4 floats, so that the TMA box starts on a 16-byte boundary.
__device__ __forceinline__ int img_win_y(int y0) { return (y0 >> 1) - 1; }
__device__ __forceinline__ int img_win_x(int x0) { return ((x0 >> 1) - 1) & ~3; }
__device__ __forceinline__ void mma_release(const Params& p, uint32_t bar0, int sa, int sb, bool release_a) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {             // one arrival per warp: each warp waited for its own wgmma groups
        if (release_a) mbar_arrive(bar_empty_a(bar0, sa));
        if (!p.b_resident) mbar_arrive(bar_empty_b(bar0, sb));
    }
}

// ---------------------------------------------------------------------------------------
// MMA + epilogue warpgroup.  NT = n_tile.  Accumulator register j * 4 + i * 2 + c of m64 half h holds
// pixel row 64 h + 16 (warp % 4) + lane / 4 + 8 i, output channel 8 j + 2 (lane % 4) + c of the tile.
// kSplit (fp32-faithful mode): main = Ah * Bh and corr = Ah * Bl + Al * Bh in two accumulator arrays, summed in the
// epilogue.  Every wgmma has the same shape (m64 nNT k16), so the hardware orders the accumulator accesses of
// consecutive instructions without a fence and they pipeline.  The 2^-11-sized corrections have their own accumulator
// because the tensor core truncates on every accumulate: added into the large main sum they cost ~0.5 ulp of the MAIN
// sum per MMA (one accumulator measured on the H100: mean-abs error 1.6e-4 on the migan-256 reference fixture, above
// the 1e-4 bound).
// kRing: the tile's noise and image taps come from the epilogue window ring in shared memory (Params::ep_stages); the
// compiler may then move those loads freely around the global stores.  Without it they are read from global memory.
// The ring is planned for activated 3-pass launches only, so kRing also fixes act = 1: the unactivated path's constants
// are not kept around the row loop.
// ---------------------------------------------------------------------------------------
template <int NT, bool kSplit, bool kRing>
__device__ __forceinline__ void mma_epilogue(const Params& p, uint32_t smem_base, const uint8_t* smem_gen, uint32_t bar0,
                                             const float* s_rgb, int my_tiles) {
    constexpr int NA = NT / 2;                       // accumulator registers per m64 half
    constexpr int NC = kSplit ? NA : 1;              // correction accumulator (unused in fast mode)
    const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int num_kb = p.num_kb;
    const uint32_t b_stage_bytes = (uint32_t)NT * kKBlock * 2 * 2;   // [Bh ; Bl]
    float acc[2][NA], cor[2][NC];
    float rgb_acc[4];                                // torgb sum of colour lane % 4 over the group's N tiles, per pixel row
    Ring ra(p.a_stages), rb(p.b_stages), re(kRing ? p.ep_stages : 1);
    for (int it = 0; it < my_tiles; ++it) {
      const TileCoord tc = decode_tile(p, blockIdx.x + it * gridDim.x);
      for (int j = 0; j < p.n_group; ++j) {
        // Stationary A (n_group > 1): slot kb holds K block kb for the whole group.  The first N tile waits for it, the
        // last one releases it.
        const bool first_n = (j == 0), last_n = (j == p.n_group - 1);
        int prev_sa = 0, prev_sb = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
            const int sa = (p.n_group > 1) ? kb : ra.stage;
            if (first_n) {
                mbar_wait(bar_full_a(bar0, sa), ra.phase, 210 + sa, p.error_flag);
                ra.advance();
            }
            const int sb = p.b_resident ? kb : rb.stage;
            mbar_wait(bar_full_b(bar0, sb), p.b_resident ? 0 : rb.phase, 220 + sb, p.error_flag);
            if (!p.b_resident) rb.advance();
            const uint32_t a_hi = smem_base + p.off_a + sa * kAStage;
            const uint32_t b_hi = smem_base + p.off_b + sb * b_stage_bytes;
            const uint64_t dah = wgmma_desc_sw128(a_hi), dal = wgmma_desc_sw128(a_hi + kABytes);
            const uint64_t dbh = wgmma_desc_sw128(b_hi), dbl = wgmma_desc_sw128(b_hi + b_stage_bytes / 2);
            wg_fence_acc(acc[0]);
            wg_fence_acc(acc[1]);
            if constexpr (kSplit) { wg_fence_acc(cor[0]); wg_fence_acc(cor[1]); }
            wg_fence();
#pragma unroll
            for (int k = 0; k < kKBlock / 16; ++k) {
                const uint64_t adv = (uint64_t)(k * 32 >> 4);   // 16 fp16 = 32 bytes along K inside the SW128 row
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t mh = (uint64_t)(h * 64 * 128 >> 4);
                    Wgmma<NT>::mma(acc[h], dah + mh + adv, dbh + adv, (kb | k) != 0);
                    if constexpr (kSplit) {
                        Wgmma<NT>::mma(cor[h], dah + mh + adv, dbl + adv, (kb | k) != 0);
                        Wgmma<NT>::mma(cor[h], dal + mh + adv, dbh + adv, 1u);
                    }
                }
            }
            wg_commit();
            if (kb > 0) {                        // the previous K block's MMAs have retired: its A / B slots are free
                wg_wait<1>();
                mma_release(p, bar0, prev_sa, prev_sb, last_n);
            }
            prev_sa = sa; prev_sb = sb;
        }
        wg_wait<0>();
        wg_fence_acc(acc[0]);
        wg_fence_acc(acc[1]);
        if constexpr (kSplit) { wg_fence_acc(cor[0]); wg_fence_acc(cor[1]); }
        mma_release(p, bar0, prev_sa, prev_sb, last_n);

        // ---- epilogue: the four pixel rows of this thread, straight from the accumulators ----
        const int chan0 = (tc.nt + j) * NT;
        const float scale_g = p.inv_scale * kActGain;
        // The stage holding this tile's windows: waited for before the group's first epilogue, released after its last.
        const float* ep_nz = nullptr;
        const float* ep_img = nullptr;
        if constexpr (kRing) {
            if (first_n) mbar_wait(bar_full_ep(bar0, re.stage), re.phase, 230 + re.stage, p.error_flag);
            ep_nz = reinterpret_cast<const float*>(smem_gen + p.off_ep + re.stage * p.ep_stage_stride);
            ep_img = ep_nz + p.ep_off_img / 4;
        }
        // pixel of the thread's row r (0..3): image / row / column inside the tile and in the tensor
        struct RowPx { int limg, ly, lx, pimg, poy, pox; bool valid; };
        auto row_px = [&](int r) {
            const int m = (r >> 1) * 64 + wq * 16 + (lane >> 2) + 8 * (r & 1);
            RowPx q;
            q.limg = m >> (p.l_tw + p.l_th); q.ly = (m >> p.l_tw) & (p.tile_h - 1); q.lx = m & (p.tile_w - 1);
            q.pimg = tc.n0 + q.limg; q.poy = tc.y0 + q.ly; q.pox = tc.x0 + q.lx;
            q.valid = q.pimg < p.n && q.poy < p.H && q.pox < p.W;   // partial tiles at the right / bottom edge
            return q;
        };
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int h = r >> 1, i = r & 1;
            const RowPx q = row_px(r);
            const int ly = q.ly, lx = q.lx, pimg = q.pimg, poy = q.poy, pox = q.pox;
            const bool valid = q.valid;
            // The NZ window is zero past the extents; rows of images past n read some noise but are never stored.
            float nz;
            if constexpr (kRing) nz = p.noise ? ep_nz[(ly << p.l_tw) + lx] : 0.f;
            else nz = (p.noise && valid) ? __ldg(p.noise + poy * p.noise_pitch + pox) : 0.f;
            const float nz_g = nz * kActGain;
            float* out_px = p.out + (((size_t)pimg * p.H + poy) * p.W + pox) * p.cout + chan0 + 2 * (lane & 3);
#pragma unroll
            for (int jj = 0; jj < NT / 8; ++jj) {
                float o[2];
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float v = kSplit ? acc[h][jj * 4 + i * 2 + c] + cor[h][(jj * 4 + i * 2 + c) % NC] : acc[h][jj * 4 + i * 2 + c];
                    if (kRing || p.act) {            // clamp(lrelu(f) * sqrt2) with the gain folded into the scale
                        const float a = fmaf(v, scale_g, nz_g);
                        o[c] = fminf(fmax3(a, a * kLreluAlpha, -kActClamp), kActClamp);
                    } else {
                        o[c] = fmaf(v, p.inv_scale, nz);
                    }
                    acc[h][jj * 4 + i * 2 + c] = o[c];   // the activated row, for torgb below
                }
                if (p.store_out && valid) *reinterpret_cast<float2*>(out_px + 8 * jj) = make_float2(o[0], o[1]);
            }
        }
        if (p.torgb) {
            // 1x1 conv Cout -> 3 on the activated rows (the CTA tile holds all of cout).  One pass per colour, channel pairs
            // outside and the four rows inside, so each weight pair is read from shared memory once per tile, not once per
            // row; every row still adds the pairs in jj order.  (All three colours in one pass would hold 12 partial sums
            // and spill under the 184-register ceiling.)  The quad holds the pixel's channels of this N tile: it sums its
            // partials, and lane k keeps colour k (lane 3 a copy of colour 2).
            const int k = lane & 3;
            float sk[4];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float s[4] = {0.f, 0.f, 0.f, 0.f};     // colour c over this thread's channels, per pixel row
#pragma unroll
                for (int jj = 0; jj < NT / 8; ++jj) {
                    const int ch = chan0 + 8 * jj + 2 * k;   // even, and cout is even: an 8-byte aligned pair
                    const float2 w = *reinterpret_cast<const float2*>(s_rgb + c * p.cout + ch);
#pragma unroll
                    for (int r = 0; r < 4; ++r)
                        s[r] = fmaf(acc[r >> 1][jj * 4 + (r & 1) * 2 + 1], w.y, fmaf(acc[r >> 1][jj * 4 + (r & 1) * 2], w.x, s[r]));
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) {
#pragma unroll
                    for (int x = 1; x < 4; x <<= 1) s[r] += __shfl_xor_sync(0xffffffffu, s[r], x);
                    if (c == 0 || k >= c) sk[r] = s[r];
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const RowPx q = row_px(r);
                const int limg = q.limg, pimg = q.pimg, poy = q.poy, pox = q.pox;
                const bool valid = q.valid;
                // img = upsample(img_lo) + (torgb(x) + b)   (migan_inference.py:308-313); planar NCHW.  Lane k adds colour k
                // of the row up over the group's N tiles in registers; after the last N tile it writes the pixel.
                rgb_acc[r] = first_n ? sk[r] : rgb_acc[r] + sk[r];
                if (last_n && k < 3 && valid) {
                    float rv = rgb_acc[r] + s_rgb[kRgbBias + k];
                    if (p.img_lo) {
                        const int hl = p.H >> 1, wl = p.W >> 1;
                        // IMG window: plane (limg, k), rows from img_win_y(y0), columns from img_win_x(x0), zero outside
                        // the low-resolution image (TMA out-of-bounds fill, the taps' zero padding)
                        const float* win = nullptr;
                        int wy0 = 0, wx0 = 0;
                        if constexpr (kRing) {
                            win = ep_img + (limg * 3 + k) * p.img_bh * p.img_bw;
                            wy0 = img_win_y(tc.y0); wx0 = img_win_x(tc.x0);
                        }
                        float up = 0.f;
#pragma unroll
                        for (int a = 0; a < 2; ++a)
#pragma unroll
                            for (int bb = 0; bb < 2; ++bb) {
                                const int iy = (poy + (poy & 1) + 2 * a - 2) >> 1, ix = (pox + (pox & 1) + 2 * bb - 2) >> 1;
                                const int ty = (poy & 1) + 2 * a, tx = (pox & 1) + 2 * bb;
                                float lo;
                                if constexpr (kRing) {
                                    lo = win[(iy - wy0) * p.img_bw + (ix - wx0)];
                                } else {
                                    const bool ok = iy >= 0 && iy < hl && ix >= 0 && ix < wl;
                                    lo = ok ? __ldg(p.img_lo + (((size_t)pimg * 3 + k) * hl + iy) * wl + ix) : 0.f;
                                }
                                up = fmaf(s_rgb[kRgbFir + (ty * 4 + tx) * 3 + k], lo, up);
                            }
                        rv = up + rv;
                    }
                    p.img_out[(((size_t)pimg * 3 + k) * p.H + poy) * p.W + pox] = rv;
                }
            }
        }
        if constexpr (kRing) {
            if (last_n) {                              // the group's last epilogue has read the stage
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty_ep(bar0, re.stage));
                re.advance();
            }
        }
      }
    }
}

// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
sepconv_tc_kernel(const __grid_constant__ Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bars[kNumBars];
    __shared__ __align__(16) float s_rgb[3 * kMaxRgbC + 4 + 48];    // torgb weights [3][cout<=256], bias[3(+1)], fir[16][3]

    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    const uint32_t bar0 = smem_u32(bars);
    auto full_in = [&](int s) { return bar0 + 8u * (0 + s); };
    auto empty_in = [&](int s) { return bar0 + 8u * (8 + s); };
    auto full_a = [&](int s) { return bar_full_a(bar0, s); };
    auto empty_a = [&](int s) { return bar_empty_a(bar0, s); };
    auto full_b = [&](int s) { return bar_full_b(bar0, s); };
    auto empty_b = [&](int s) { return bar_empty_b(bar0, s); };

    const int a_dw = (p.source != SEPCONV_SRC_SPLIT);
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.in_stages; ++s) { mbar_init(full_in(s), 1); mbar_init(empty_in(s), kNumProWarps / 2); }
        for (int s = 0; s < p.a_stages; ++s) { mbar_init(full_a(s), a_dw ? kNumProWarps : 1); mbar_init(empty_a(s), 4); }
        for (int s = 0; s < p.b_stages; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), 4); }
        for (int s = 0; s < p.ep_stages; ++s) { mbar_init(bar_full_ep(bar0, s), 1); mbar_init(bar_empty_ep(bar0, s), 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == kProducerWarp && lane == 0) {
        if (p.source == SEPCONV_SRC_SPLIT) { prefetch_tensormap(&p.map_a_hi); prefetch_tensormap(&p.map_a_lo); }
        else if (p.source == SEPCONV_SRC_STEM) prefetch_tensormap(&p.map_aux);
        else prefetch_tensormap(&p.map_in);
        if (p.source == SEPCONV_SRC_UP) { prefetch_tensormap(&p.map_t); if (p.up_has_noise) prefetch_tensormap(&p.map_aux); }
        prefetch_tensormap(&p.map_w_hi); prefetch_tensormap(&p.map_w_lo);
        if (p.ep_stages) {
            if (p.noise) prefetch_tensormap(&p.map_nz);
            if (p.torgb && p.img_lo) prefetch_tensormap(&p.map_img);
        }
    }
    if (p.torgb) {
        for (int i = threadIdx.x; i < 3 * p.cout; i += kThreads) s_rgb[i] = __ldg(p.rgb_w + i);
        if (threadIdx.x < 3) s_rgb[kRgbBias + threadIdx.x] = __ldg(p.rgb_b + threadIdx.x);
        if (threadIdx.x < 48 && p.img_lo) s_rgb[kRgbFir + threadIdx.x] = __ldg(p.rgb_fir + threadIdx.x);
    }
    if (a_dw && p.off_dw != 0xFFFFFFFFu) {   // depthwise taps + bias for all channels: read per chunk by every prologue thread
        float* sdw = reinterpret_cast<float*>(smem_gen + p.off_dw);
        for (int i = threadIdx.x; i < 9 * p.cin; i += kThreads) sdw[i] = __ldg(p.w9 + i);
        for (int i = threadIdx.x; i < p.cin; i += kThreads) sdw[9 * p.cin + i] = __ldg(p.bias + i);
    }
    if (p.source == SEPCONV_SRC_STEM) {
        float* st = reinterpret_cast<float*>(smem_gen + p.off_stem);
        // pair-interleaved: [channel pair][plane][2] so that the pre-stage reads (w[ch][i], w[ch+1][i]) as one register pair
        for (int i = threadIdx.x; i < 4 * p.cin; i += kThreads) st[(i >> 3) * 8 + (i & 3) * 2 + ((i >> 2) & 1)] = __ldg(p.stem_w + i);
        for (int i = threadIdx.x; i < p.cin; i += kThreads) st[4 * p.cin + i] = __ldg(p.stem_b + i);
    }
    pdl_trigger();           // the successor's blocks may start their own setup as soon as SMs free up
    pdl_wait();              // barriers and the weight tables above are set up under the predecessor's tail; its output is read below
    __syncthreads();

    const int num_kb = p.num_kb;
    const int my_tiles = (p.num_tiles > (int)blockIdx.x) ? (p.num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const uint32_t b_stage_bytes = (uint32_t)p.n_tile * kKBlock * 2 * 2;   // [Bh ; Bl] of one N tile

    if (warp >= kProducerWarp) {
        // ================================ TMA producer ================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        if (warp == kProducerWarp && lane == 0) {
            // L2 prefetch cursor: the smem rings are too shallow to cover HBM latency at full bandwidth, so the
            // producer also asks the L2 for the data `prefetch` loads ahead (possibly in the next tile).
            int pf_it = 0, pf_kb = 0, pf_g = 0;
            auto prefetch_next = [&]() {
                if (pf_it >= my_tiles) return;
                if (a_dw) {
                    const TileCoord t2 = decode_tile(p, blockIdx.x + pf_it * gridDim.x);
                    if (p.source != SEPCONV_SRC_STEM)
                        tma_prefetch_4d(&p.map_in, pf_kb * kKBlock + pf_g * kChunkC, t2.x0 - 1, t2.y0 - 1, t2.n0);
                    if (++pf_g < 2) return;
                    pf_g = 0;
                } else {
                    const TileCoord t2 = decode_tile(p, blockIdx.x + pf_it * gridDim.x);
                    tma_prefetch_4d(&p.map_a_hi, pf_kb * kKBlock, t2.x0, t2.y0, t2.n0);
                    tma_prefetch_4d(&p.map_a_lo, pf_kb * kKBlock, t2.x0, t2.y0, t2.n0);
                }
                if (++pf_kb == num_kb) { pf_kb = 0; ++pf_it; }
            };
            for (int c = 0; c < p.prefetch; ++c) prefetch_next();
            Ring rin(p.in_stages), ra(p.a_stages), rb(p.b_stages), rep(p.ep_stages ? p.ep_stages : 1);
            for (int it = 0; it < my_tiles; ++it) {
              const TileCoord tc = decode_tile(p, blockIdx.x + it * gridDim.x);
              for (int j = 0; j < p.n_group; ++j) {
                for (int kb = 0; kb < num_kb; ++kb) {
                    // A (or the prologue's input) once per pixel tile; the group's later N tiles only need their weights
                    if (j == 0 && a_dw) {
                        for (int g = 0; g < 2; ++g) {
                            const int s = rin.stage;
                            if (p.prefetch) prefetch_next();
                            mbar_wait<true>(empty_in(s), rin.phase ^ 1, 100 + s, p.error_flag);
                            rin.advance();
                            mbar_expect_tx(full_in(s), p.in_tx_bytes);
                            const uint32_t dst = smem_base + p.off_in + s * p.in_stage_stride;
                            const int c0 = kb * kKBlock + g * kChunkC;
                            if (p.source == SEPCONV_SRC_STEM) {
                                tma_load_4d(dst + p.off_aux, &p.map_aux, full_in(s), tc.x0 - kAuxLeft, tc.y0 - 1, 0, tc.n0);
                            } else {
                                tma_load_4d(dst, &p.map_in, full_in(s), c0, tc.x0 - 1, tc.y0 - 1, tc.n0);
                                if (p.source == SEPCONV_SRC_UP) {
                                    tma_load_4d(dst + p.off_t, &p.map_t, full_in(s), c0, (tc.x0 >> 1) - 1, (tc.y0 >> 1) - 1, tc.n0);
                                    if (p.up_has_noise) tma_load_2d(dst + p.off_aux, &p.map_aux, full_in(s), tc.x0 - kAuxLeft, tc.y0 - 1);
                                }
                            }
                        }
                    } else if (j == 0) {
                        const int s = ra.stage;
                        if (p.prefetch) prefetch_next();
                        mbar_wait<true>(empty_a(s), ra.phase ^ 1, 110 + s, p.error_flag);
                        ra.advance();
                        mbar_expect_tx(full_a(s), kAStage);
                        tma_load_4d(smem_base + p.off_a + s * kAStage, &p.map_a_hi, full_a(s), kb * kKBlock, tc.x0, tc.y0, tc.n0);
                        tma_load_4d(smem_base + p.off_a + s * kAStage + kABytes, &p.map_a_lo, full_a(s), kb * kKBlock, tc.x0, tc.y0, tc.n0);
                    }
                    if (!p.b_resident || it == 0) {
                        const int s = p.b_resident ? kb : rb.stage;
                        if (!p.b_resident) { mbar_wait<true>(empty_b(s), rb.phase ^ 1, 120 + s, p.error_flag); rb.advance(); }
                        mbar_expect_tx(full_b(s), b_stage_bytes);
                        const uint32_t dst = smem_base + p.off_b + s * b_stage_bytes;
                        const int row = (tc.nt + j) * p.n_tile;
                        tma_load_2d(dst, &p.map_w_hi, full_b(s), kb * kKBlock, row);
                        tma_load_2d(dst + b_stage_bytes / 2, &p.map_w_lo, full_b(s), kb * kKBlock, row);
                    }
                    // The epilogue's windows, once per CTA tile, after the tile's operand loads (the epilogue runs last)
                    if (p.ep_stages && j == 0 && kb == num_kb - 1) {
                        const int s = rep.stage;
                        mbar_wait<true>(bar_empty_ep(bar0, s), rep.phase ^ 1, 130 + s, p.error_flag);
                        rep.advance();
                        mbar_expect_tx(bar_full_ep(bar0, s), p.ep_tx_bytes);
                        const uint32_t dst = smem_base + p.off_ep + s * p.ep_stage_stride;
                        if (p.noise) tma_load_2d(dst, &p.map_nz, bar_full_ep(bar0, s), tc.x0, tc.y0);
                        if (p.torgb && p.img_lo)
                            tma_load_4d(dst + p.ep_off_img, &p.map_img, bar_full_ep(bar0, s), img_win_x(tc.x0), img_win_y(tc.y0), 0, tc.n0);
                    }
                }
              }
            }
        }
    } else if (warp >= kMmaWarp0) {
        // ================================ MMA + epilogue ==============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMmaRegs));
        // the epilogue ring is planned for activated 3-pass launches only (plan_layout)
        if (p.ep_stages) mma_epilogue<64, true, true>(p, smem_base, smem_gen, bar0, s_rgb, my_tiles);
        else if (p.passes == 3) mma_epilogue<64, true, false>(p, smem_base, smem_gen, bar0, s_rgb, my_tiles);
        else if (p.n_tile == 128) mma_epilogue<128, false, false>(p, smem_base, smem_gen, bar0, s_rgb, my_tiles);
        else mma_epilogue<64, false, false>(p, smem_base, smem_gen, bar0, s_rgb, my_tiles);
    } else {
        // ================================ prologue (pre-stage + depthwise) ========================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kProRegs));
        if (!a_dw) return;
        const int g = warp >> 2;                          // channel half of the K-block this group produces
        const int tg = threadIdx.x - g * 128;
        Ring rin(p.in_stages, g, 2), ra(p.a_stages);     // this group owns input stages g, g+2, ...
        const float* w9p = (p.off_dw != 0xFFFFFFFFu) ? reinterpret_cast<const float*>(smem_gen + p.off_dw) : p.w9;
        const float* bp = (p.off_dw != 0xFFFFFFFFu) ? w9p + 9 * p.cin : p.bias;
        const float* stem_tab = reinterpret_cast<const float*>(smem_gen + p.off_stem);
        int tile = blockIdx.x;
        for (int it = 0; it < my_tiles; ++it, tile += gridDim.x) {
            for (int kb = 0; kb < num_kb; ++kb) {
                const int s = rin.stage;
                const int sa = ra.stage;
                mbar_wait(full_in(s), rin.phase, 400 + s, p.error_flag);
                rin.advance();
                uint8_t* stage = smem_gen + p.off_in + s * p.in_stage_stride;
                f4* sin = reinterpret_cast<f4*>(stage);
                const int cg0 = kb * kKBlock + g * kChunkC;
                // the tile origin is only needed by the pre-stages: decoded per chunk there, so that it is not held in
                // registers across the depthwise stage (which runs at the prologue's register limit)
                if (p.source == SEPCONV_SRC_UP) {
                    const TileCoord tc = decode_tile(p, tile);
                    prestage_up(sin, reinterpret_cast<const f4*>(stage + p.off_t), reinterpret_cast<const float*>(stage + p.off_aux),
                                p.up_taps, tc.y0, tc.x0, p.H, p.W, p.up_has_noise, tg);
                    bar_sync_named(1 + g, 128);
                } else if (p.source == SEPCONV_SRC_STEM) {
                    const TileCoord tc = decode_tile(p, tile);
                    prestage_stem(sin, reinterpret_cast<const float*>(stage + p.off_aux), stem_tab, stem_tab + 4 * p.cin,
                                  cg0, tc.y0, tc.x0, p.H, p.W, tg);
                    bar_sync_named(1 + g, 128);
                }
                mbar_wait(empty_a(sa), ra.phase ^ 1, 410 + sa, p.error_flag);
                ra.advance();
                uint8_t* a_hi = smem_gen + p.off_a + sa * kAStage;
                uint8_t* a_lo = a_hi + kABytes;
                if (p.tile_w == 16) prologue_chunk<1, 8, 16>(sin, a_hi, a_lo, w9p, bp, p.cin, cg0, g, tg);
                else if (p.tile_w == 8) prologue_chunk<2, 8, 8>(sin, a_hi, a_lo, w9p, bp, p.cin, cg0, g, tg);
                else prologue_chunk<8, 4, 4>(sin, a_hi, a_lo, w9p, bp, p.cin, cg0, g, tg);
                fence_proxy_async();        // generic-proxy smem writes -> visible to the tensor core / TMA (async proxy)
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(full_a(sa));
                    mbar_arrive(empty_in(s));
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

const char* encode_map(CUtensorMap* m, CUtensorMapDataType dt, int rank, const void* addr, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle sw) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return "cuTensorMapEncodeTiled entry point not available";
    cuuint64_t gdim[5], gstr[5];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(addr), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        static thread_local char msg[96];
        snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
        return msg;
    }
    return nullptr;
}

const char* encode_x_map(CUtensorMap* m, const void* x, int n, int H, int W) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, 4, (uint64_t)n};
    const uint64_t str[3] = {(uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)H * W * 16};
    const uint32_t box[4] = {(uint32_t)kAuxW, 10, 4, 1};
    return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

constexpr int kMaxDevices = 64;
int* g_error_flag[kMaxDevices] = {nullptr};        // device alias of the host-mapped timeout record, per device
int* g_error_flag_host[kMaxDevices] = {nullptr};

int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return e ? atoi(e) : dflt;
}

}  // namespace

// Params is kept opaque to the ABI layer: SepconvTcArgs carries it as bytes.
static_assert(sizeof(Params) <= sizeof(((SepconvTcArgs*)0)->params_blob), "params blob too small");

// Tensor map of an NHWC fp32 tensor for the TMA-staged down-sampling kernel (elementwise.cu): box = 64 channels x 36 columns x 1 row.
const char* make_down_tensor_map(DownTensorMap* desc, const float* in, int n, int H, int W, int C) {
    static_assert(sizeof(CUtensorMap) <= sizeof(DownTensorMap), "tensor map size");
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)n};
    const uint64_t str[3] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
    const uint32_t box[4] = {64u, 36u, 1u, 1u};
    return encode_map(reinterpret_cast<CUtensorMap*>(desc), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, in, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

cudaError_t configure_sepconv_tc() {
    cudaError_t e = cudaFuncSetAttribute(sepconv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSmemLimit - kStaticSmem));
    if (e != cudaSuccess) return e;
    int dev = 0;
    e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < kMaxDevices && !g_error_flag[dev]) {
        // host-mapped so that the record of a timed-out wait survives the trap that follows it
        e = cudaHostAlloc(reinterpret_cast<void**>(&g_error_flag_host[dev]), sizeof(int), cudaHostAllocMapped);
        if (e != cudaSuccess) return e;
        *g_error_flag_host[dev] = 0;
        e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&g_error_flag[dev]), g_error_flag_host[dev], 0);
    }
    return e;
}

int sepconv_tc_timeout_record(int device) {
    return (device >= 0 && device < kMaxDevices && g_error_flag_host[device]) ? *g_error_flag_host[device] : 0;
}

namespace {

// SMs the persistent grid may use.  MIGAN_TC_RESERVE_SMS leaves SMs free for a concurrently running collective.
int grid_sms() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms - std::max(0, std::min(env_int("MIGAN_TC_RESERVE_SMS", 0), sms / 2));
}

// Tiling, N grouping, ring depths and shared-memory layout of a launch.  They depend on the shapes, the source and
// whether torgb is fused, never on a pointer, so the generator's planner can ask before it commits to fusing torgb.
// candidate < 0 takes the first candidate layout that fits (production); candidate = i takes the i-th or fails (tests).
const char* plan_layout(Params& p, const SepconvTcDesc& d, int sms, uint32_t& smem_bytes, int candidate = -1,
                        int* num_candidates = nullptr, bool* dw_global = nullptr) {
    const int n = d.n, h = d.h, w = d.w, cin = d.cin, cout = d.cout;
    if (cin % kKBlock != 0 || cout % 64 != 0) return "cin must be a multiple of 64 and cout of 64";
    if (h < 4 || w < 4) return "extents must be >= 4";
    if ((d.noise || d.up_noise) && (d.noise_pitch < w || d.noise_pitch % 4 != 0)) return "noise pitch must be >= w and a multiple of 4";
    p.source = d.source;
    const bool dw = (d.source != SEPCONV_SRC_SPLIT);
    if ((d.source == SEPCONV_SRC_UP || d.source == SEPCONV_SRC_STEM) && std::min(h, w) < 16) return "fused prologues need 8 x 16 tiles (extents >= 16)";
    if (d.source == SEPCONV_SRC_STEM && w % 4 != 0) return "the stem prologue needs a width that is a multiple of 4 (16-byte x rows)";
    p.n = n; p.H = h; p.W = w; p.cin = cin; p.cout = cout; p.act = d.act; p.passes = d.passes;
    p.noise_pitch = d.noise_pitch;
    p.n_tile = (cout == 64 || d.passes == 3) ? 64 : kMaxTileN;   // main + corr of 64 channels fill the accumulators
    p.num_kb = cin / kKBlock;
    // Tile shapes are picked from the largest powers of two that fit the extents (at a square power-of-two level: the
    // level's side), so a level keeps its R x R tiling whatever its rectangular extent; the last tile of a row / column may
    // be partial.
    auto p2floor = [](int v) { int q = 1; while (2 * q <= v) q *= 2; return q; };
    if (dw) {   // spatial tiles with halo
        const int m = p2floor(std::min(h, w));
        p.tile_w = std::min(m, 16);
        p.tile_h = std::min(m, 8);
    } else {    // the pre-split operand: whole 128-pixel rows where the width allows (contiguous TMA boxes)
        p.tile_w = std::min(p2floor(w), 128);
        p.tile_h = std::min(p2floor(h), kTileM / p.tile_w);
    }
    p.tile_n = kTileM / (p.tile_w * p.tile_h);
    p.tiles_x = (w + p.tile_w - 1) / p.tile_w; p.tiles_y = (h + p.tile_h - 1) / p.tile_h; p.tiles_n = (n + p.tile_n - 1) / p.tile_n;
    p.div_tx = FastDiv((uint32_t)p.tiles_x); p.div_ty = FastDiv((uint32_t)p.tiles_y);
    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
    // Few pixel tiles (the 4 x 4 ... 16 x 16 levels at small batches): most SMs would idle while a few CTAs stream the
    // weight matrix.  Narrow N tiles spread the layer over 2 x the CTAs.
    if (!d.rgb && p.n_tile > 64 && cout >= 256 && m_tiles * (cout / p.n_tile) * 2 < sms)
        p.n_tile = 64;
    p.num_n_tiles = cout / p.n_tile;
    auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };

    // ---- input stage: IN area (+ T, NZ | XA) ----
    const uint32_t in_chunk_bytes = (uint32_t)(p.tile_n * (p.tile_h + 2) * (p.tile_w + 2) * kChunkC * 4);
    uint32_t stage_bytes = in_chunk_bytes;
    p.in_tx_bytes = in_chunk_bytes;
    p.up_has_noise = (d.source == SEPCONV_SRC_UP && d.up_noise) ? 1 : 0;
    if (d.source == SEPCONV_SRC_UP) {
        p.off_t = in_chunk_bytes;                 // 23040: 128-byte aligned
        p.off_aux = p.off_t + 6 * 10 * kChunkC * 4;
        stage_bytes = p.off_aux + 10 * kAuxW * 4;
        p.in_tx_bytes = in_chunk_bytes + 6 * 10 * kChunkC * 4 + (p.up_has_noise ? 10 * kAuxW * 4 : 0);
    } else if (d.source == SEPCONV_SRC_STEM) {
        p.off_aux = in_chunk_bytes;
        stage_bytes = p.off_aux + 4 * 10 * kAuxW * 4;
        p.in_tx_bytes = 4 * 10 * kAuxW * 4;
    }
    p.in_stage_stride = (stage_bytes + 1023u) & ~1023u;

    // ---- shared-memory budget -> N group and stage counts ----
    const uint32_t b_stage = (uint32_t)p.n_tile * kKBlock * 2 * 2;
    const uint32_t budget = kSmemLimit - kStaticSmem - 1024;   // static smem + alignment slack
    // The input ring is shared by the two prologue groups (even chunks -> group 0, odd -> group 1):
    // the stage count must be EVEN so that each stage always belongs to one group and every waiter
    // observes every phase of its barriers (parity waits alias otherwise).
    p.b_resident = (p.num_n_tiles == 1 && (uint32_t)p.num_kb * b_stage <= 65536) ? 1 : 0;
    const uint32_t tables = dw ? 40u * cin + (d.source == SEPCONV_SRC_STEM ? 20u * cin : 0u) : 0u;
    // candidate configurations in order of preference
    struct Cand { int n_group, in_stages, b_stages, a_stages; bool dw_global; };
    std::vector<Cand> cands;
    // Stationary A, for the sources with a prologue: it then runs once per pixel tile instead of once per N tile.  The
    // group is the widest that still gives every SM a CTA tile (all N tiles when torgb is fused).  The depthwise taps
    // move from shared memory to global (L1-cached) loads only where that is what makes the resident A fit.
    if (dw && p.num_n_tiles > 1 && p.num_kb <= kMaxAStages) {
        int g = p.num_n_tiles;
        if (!d.rgb)
            while (g > 1 && m_tiles * (p.num_n_tiles / g) < sms) g >>= 1;
        if (g > 1)
            for (bool dw_global : {false, true}) {
                if (dw_global && d.source == SEPCONV_SRC_STEM) continue;   // the fromrgb table lives next to the taps
                for (int bs : {3, 2})
                    for (int in_st : {6, 4, 2}) cands.push_back({g, in_st, bs, p.num_kb, dw_global});
            }
    }
    {
        // plain schedule: deeper input ring first, then a deeper A ring (the prologue runs ahead while the MMA warpgroup
        // drains its accumulators)
        const int b_res = p.b_resident ? p.num_kb : 0;
        // input ring depths to try, deepest first (even: each prologue group owns every other stage)
        const std::vector<int> ins = dw ? std::vector<int>{6, 4, 2} : std::vector<int>{0};
        const int bopts[2] = {b_res ? b_res : 3, b_res ? b_res : 2};
        for (int bi = 0; bi < 2; ++bi) {
            if (bi == 1 && bopts[1] == bopts[0]) break;
            const int bs = bopts[bi];
            for (int in_st : ins)
                for (int a_st : {4, dw ? 2 : 3}) cands.push_back({1, in_st, bs, a_st, false});
        }
    }
    if (num_candidates) *num_candidates = (int)cands.size();
    if (candidate >= (int)cands.size()) return "no such candidate layout";
    bool found = false;
    uint32_t used = 0;
    for (size_t i = candidate < 0 ? 0 : (size_t)candidate; i < cands.size(); ++i) {
        const Cand& c = cands[i];
        const uint32_t tab = c.dw_global ? 0u : tables;
        const uint32_t total = (uint32_t)c.in_stages * p.in_stage_stride + (uint32_t)c.a_stages * kAStage + (uint32_t)c.b_stages * b_stage + tab;
        if (total > budget) {
            if (candidate >= 0) return "candidate layout exceeds the shared-memory budget";
            continue;
        }
        if (dw_global) *dw_global = c.dw_global;
        p.n_group = c.n_group;
        p.in_stages = c.in_stages; p.a_stages = c.a_stages; p.b_stages = c.b_stages;
        p.off_in = 0;
        p.off_a = (uint32_t)c.in_stages * p.in_stage_stride;
        p.off_b = p.off_a + (uint32_t)c.a_stages * kAStage;
        p.off_dw = (dw && !c.dw_global) ? p.off_b + (uint32_t)c.b_stages * b_stage : 0xFFFFFFFFu;
        p.off_stem = p.off_b + (uint32_t)c.b_stages * b_stage + 40u * cin;
        smem_bytes = total + 1024;
        used = total;
        found = true;
        break;
    }
    if (!found) return "shared memory budget exceeded";
    if (d.rgb && (p.n_group != p.num_n_tiles || cout > kMaxRgbC))
        return "fused torgb needs all output channels of a pixel tile in one CTA tile (cout <= 256 with a resident A operand)";
    if (p.in_stages > 8 || p.a_stages > kMaxAStages || p.b_stages > 8) return "internal: ring too deep for the barrier table";

    // ---- epilogue window ring: placed after the chosen layout, in what it leaves of the budget, so that it never changes
    // the layout.  4 stages where they fit (the producer may run several CTA tiles ahead of the epilogue), else 2, else
    // none.  The IMG box needs 16-byte rows of the low-resolution image (W / 2 a multiple of 4).  Only the activated 3-pass
    // epilogue has a ring variant: more epilogue instances push the prologue's register allocation into spills. ----
    p.ep_stages = 0;
    const bool ep_img = d.rgb && d.rgb->img_lo;
    if (d.passes == 3 && d.act && (d.noise || ep_img) && (!ep_img || (w / 2) % 4 == 0)) {
        p.img_bh = (p.tile_h + 1) / 2 + 2;                 // tap rows of the tile, from one above (y0 may be odd at tile_h = 1)
        p.img_bw = (p.tile_w / 2 + 5 + 3) & ~3;            // tap columns + up to 3 of 16-byte alignment, in whole 16 bytes
        const uint32_t nz_bytes = d.noise ? (uint32_t)(p.tile_h * p.tile_w * 4) : 0u;
        const uint32_t img_bytes = ep_img ? (uint32_t)(p.tile_n * 3 * p.img_bh * p.img_bw * 4) : 0u;
        p.ep_off_img = (nz_bytes + 127u) & ~127u;          // TMA destinations: 128-byte aligned
        p.ep_tx_bytes = nz_bytes + img_bytes;
        p.ep_stage_stride = (p.ep_off_img + img_bytes + 127u) & ~127u;
        p.off_ep = (used + 127u) & ~127u;
        for (int st : {kMaxEpStages, 2})
            if (p.off_ep + (uint32_t)st * p.ep_stage_stride <= budget) { p.ep_stages = st; break; }
        if (p.ep_stages) smem_bytes = p.off_ep + (uint32_t)p.ep_stages * p.ep_stage_stride + 1024;
    }
    p.l_nt = ilog2(p.num_n_tiles / p.n_group);
    p.l_tw = ilog2(p.tile_w); p.l_th = ilog2(p.tile_h);
    p.num_tiles = m_tiles * (p.num_n_tiles / p.n_group);
    return nullptr;
}

}  // namespace

bool sepconv_tc_fuses_rgb(const SepconvTcDesc& d) {
    SepconvTcRgb rgb{};
    SepconvTcDesc q = d;
    q.rgb = &rgb;
    Params p;
    memset(&p, 0, sizeof(p));
    uint32_t smem_bytes = 0;
    return plan_layout(p, q, grid_sms(), smem_bytes) == nullptr;
}

namespace {

const char* plan_launch(SepconvTcArgs* args, const SepconvTcDesc& d, int sms, int candidate, SepconvTcPlanInfo* info) {
    Params p;
    memset(&p, 0, sizeof(p));
    const int n = d.n, h = d.h, w = d.w, cin = d.cin, cout = d.cout;
    const bool dw = (d.source != SEPCONV_SRC_SPLIT);
    if (args) {
        if (d.source == SEPCONV_SRC_SPLIT && !(d.a_hi && d.a_lo)) return "no A operand";
        if ((d.source == SEPCONV_SRC_NHWC || d.source == SEPCONV_SRC_UP) && !d.in_f32) return "no input tensor";
        if (d.source == SEPCONV_SRC_UP && !d.up_t) return "no low-resolution tensor for the up-sampling prologue";
        if (d.source == SEPCONV_SRC_STEM && !(d.stem_w && d.stem_b)) return "no fromrgb weights for the stem prologue";
    }
    uint32_t smem_bytes = 0;
    int num_candidates = 0;
    bool dw_global = false;
    if (const char* err = plan_layout(p, d, sms, smem_bytes, candidate, &num_candidates, &dw_global)) return err;
    if (args) {   // TMA reads global memory from 16-byte aligned bases only; else the epilogue reads the windows directly
        const uintptr_t nz_a = reinterpret_cast<uintptr_t>(d.noise), img_a = d.rgb ? reinterpret_cast<uintptr_t>(d.rgb->img_lo) : 0;
        if ((nz_a | img_a) & 15u) p.ep_stages = 0;
    }
    if (info) {
        *info = {p.n_group, p.in_stages, p.a_stages, p.b_stages, p.b_resident, dw_global ? 1 : 0,
                 p.tile_w, p.tile_h, p.tile_n, p.n_tile, std::min(p.num_tiles, sms), p.num_tiles, num_candidates,
                 p.ep_stages, p.ep_stages ? (int)p.off_ep : 0, p.ep_stages ? (int)p.ep_stage_stride : 0, (int)smem_bytes};
    }
    if (!args) return nullptr;
    p.w9 = d.w9; p.bias = d.bias; p.noise = d.noise; p.inv_scale = d.inv_scale; p.out = d.out;
    if (d.source == SEPCONV_SRC_UP) memcpy(p.up_taps.f, d.up_taps, sizeof(p.up_taps.f));
    if (d.source == SEPCONV_SRC_STEM) { p.stem_w = d.stem_w; p.stem_b = d.stem_b; }
    p.store_out = 1;
    if (d.rgb) {
        p.torgb = 1; p.store_out = d.rgb->store_out;
        p.rgb_w = d.rgb->w; p.rgb_b = d.rgb->b; p.rgb_fir = d.rgb->fir; p.img_lo = d.rgb->img_lo; p.img_out = d.rgb->img_out;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    p.error_flag = (dev >= 0 && dev < kMaxDevices) ? g_error_flag[dev] : nullptr;
    p.prefetch = dw ? 4 : 2;

    // ---- tensor maps ----
    const char* err = nullptr;
    if (d.source == SEPCONV_SRC_NHWC || d.source == SEPCONV_SRC_UP) {
        const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)w, (uint64_t)h, (uint64_t)n};
        const uint64_t str[3] = {(uint64_t)cin * 4, (uint64_t)w * cin * 4, (uint64_t)h * w * cin * 4};
        const uint32_t box[4] = {(uint32_t)kChunkC, (uint32_t)p.tile_w + 2, (uint32_t)p.tile_h + 2, (uint32_t)p.tile_n};
        if ((err = encode_map(&p.map_in, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.in_f32, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE))) return err;
    }
    if (d.source == SEPCONV_SRC_UP) {
        const int hl = h / 2, wl = w / 2;
        const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)wl, (uint64_t)hl, (uint64_t)n};
        const uint64_t str[3] = {(uint64_t)cin * 4, (uint64_t)wl * cin * 4, (uint64_t)hl * wl * cin * 4};
        const uint32_t box[4] = {(uint32_t)kChunkC, 10, 6, 1};
        if ((err = encode_map(&p.map_t, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.up_t, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE))) return err;
        if (p.up_has_noise) {
            const uint64_t nd[2] = {(uint64_t)w, (uint64_t)h};
            const uint64_t ns[1] = {(uint64_t)d.noise_pitch * 4};
            const uint32_t nb[2] = {(uint32_t)kAuxW, 10};
            if ((err = encode_map(&p.map_aux, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, d.up_noise, nd, ns, nb, CU_TENSOR_MAP_SWIZZLE_NONE))) return err;
        }
    }
    if (d.source == SEPCONV_SRC_SPLIT) {   // one 64-channel K block of a spatial tile: 128 rows of 128 bytes, in tile order
        const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)w, (uint64_t)h, (uint64_t)n};
        const uint64_t str[3] = {(uint64_t)cin * 2, (uint64_t)w * cin * 2, (uint64_t)h * w * cin * 2};
        const uint32_t box[4] = {(uint32_t)kKBlock, (uint32_t)p.tile_w, (uint32_t)p.tile_h, (uint32_t)p.tile_n};
        if ((err = encode_map(&p.map_a_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, d.a_hi, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B))) return err;
        if ((err = encode_map(&p.map_a_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, d.a_lo, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B))) return err;
    }
    {
        const uint64_t dims[2] = {(uint64_t)cin, (uint64_t)cout};
        const uint64_t str[1] = {(uint64_t)cin * 2};
        const uint32_t box[2] = {(uint32_t)kKBlock, (uint32_t)p.n_tile};
        if ((err = encode_map(&p.map_w_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, d.w_hi, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B))) return err;
        if ((err = encode_map(&p.map_w_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, d.w_lo, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B))) return err;
    }
    if (p.ep_stages && d.noise) {        // the noise plane's own extent: its padding columns and rows are never read
        const uint64_t nd[2] = {(uint64_t)w, (uint64_t)h};
        const uint64_t ns[1] = {(uint64_t)d.noise_pitch * 4};
        const uint32_t nb[2] = {(uint32_t)p.tile_w, (uint32_t)p.tile_h};
        if ((err = encode_map(&p.map_nz, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, d.noise, nd, ns, nb, CU_TENSOR_MAP_SWIZZLE_NONE))) return err;
    }
    if (p.ep_stages && p.torgb && p.img_lo) {
        const int hl = h / 2, wl = w / 2;
        const uint64_t dims[4] = {(uint64_t)wl, (uint64_t)hl, 3, (uint64_t)n};
        const uint64_t str[3] = {(uint64_t)wl * 4, (uint64_t)hl * wl * 4, (uint64_t)3 * hl * wl * 4};
        const uint32_t box[4] = {(uint32_t)p.img_bw, (uint32_t)p.img_bh, 3, (uint32_t)p.tile_n};
        if ((err = encode_map(&p.map_img, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, p.img_lo, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE))) return err;
    }
    if (!d.out && p.store_out) return "no output tensor";
    // Persistent grid = one CTA per usable SM.
    args->grid = (unsigned)std::min(p.num_tiles, sms);
    args->smem_bytes = smem_bytes;
    args->num_tiles = p.num_tiles;
    args->bound_x = nullptr;
    memcpy(args->params_blob, &p, sizeof(p));
    return nullptr;
}

}  // namespace

const char* sepconv_tc_plan_ex(SepconvTcArgs* args, const SepconvTcDesc& d) {
    return plan_launch(args, d, grid_sms(), -1, nullptr);
}

const char* sepconv_tc_plan_debug(SepconvTcArgs* args, const SepconvTcDesc& d, int sms, int candidate, SepconvTcPlanInfo* info) {
    if (sms == 0) sms = grid_sms();
    if (sms < 1) return "sms must be >= 1";
    return plan_launch(args, d, sms, candidate, info);
}

const char* sepconv_tc_plan(SepconvTcArgs* args, int passes, const float* in_f32, const __half* a_hi, const __half* a_lo,
                            const float* w9, const float* bias, const __half* w_hi, const __half* w_lo,
                            float inv_scale, const float* noise, float* out, int n, int res, int cin, int cout, int act,
                            const SepconvTcRgb* rgb) {
    SepconvTcDesc d;
    d.passes = passes;
    d.source = in_f32 ? SEPCONV_SRC_NHWC : SEPCONV_SRC_SPLIT;
    d.in_f32 = in_f32; d.a_hi = a_hi; d.a_lo = a_lo; d.w9 = w9; d.bias = bias; d.w_hi = w_hi; d.w_lo = w_lo;
    d.inv_scale = inv_scale; d.noise = noise; d.out = out; d.n = n; d.h = res; d.w = res; d.cin = cin; d.cout = cout; d.act = act; d.rgb = rgb;
    d.noise_pitch = res;
    return sepconv_tc_plan_ex(args, d);
}

cudaError_t launch_sepconv_tc(SepconvTcArgs& a, cudaStream_t s, float* img_out_override, const float* x_nchw) {
    Params* pp = reinterpret_cast<Params*>(a.params_blob);
    if (pp->source == SEPCONV_SRC_STEM) {
        if (!x_nchw) return cudaErrorInvalidValue;
        if (a.bound_x != x_nchw) {    // the caller's x changes between calls: re-point the input tensor map
            if (encode_x_map(&pp->map_aux, x_nchw, pp->n, pp->H, pp->W)) return cudaErrorInvalidValue;
            a.bound_x = x_nchw;
        }
    }
    Params p;
    memcpy(&p, a.params_blob, sizeof(p));
    if (img_out_override) p.img_out = img_out_override;
    return launch_pdl(sepconv_tc_kernel, dim3(a.grid), dim3(kThreads), a.smem_bytes, s, p);
}

}  // namespace migan

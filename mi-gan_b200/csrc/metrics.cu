// C ABI of the SSIM and PSNR evaluators (include/metrics_b200.h): argument checks, workspace layout and the two launches
// of each call.  The arithmetic is metrics_kernels.cuh's; the tile kernels are bodies over portable.cuh's block layer,
// run with a block's threads at once on the device and on the host in the emulation build (MIGAN_EMULATE).
//
// Workspace: the partials of the first launch, [n][parts] doubles (SSIM: parts = C * tiles; PSNR: parts = row chunks),
// then the n per-image sums.  No atomics: each block writes its own slot.
#include <math.h>

#include <algorithm>

#include "../../include/metrics_b200.h"
#include "abi_error.h"
#include "metrics_kernels.cuh"

namespace {
using metrics::kThreads;
using migan::fail;

// *out = the sum of the block's partials red[0 .. kThreads) in portable.cuh's fixed tree.
template <class B>
CK_D void tree_to(const B& blk, double* red, double* out) {
    block_tree<kThreads>(blk, red);
    blk.each([&](int t) {
        if (t == 0) *out = red[0];
    });
}

template <class B>
CK_D void ssim_block(const B& blk, const metrics::SsimArgs& a, int64_t b, double* g, double* red, void* smem) {
    double* hs = static_cast<double*>(smem);
    float* sx = reinterpret_cast<float*>(hs + (int64_t)5 * a.in_h() * metrics::kTileW);
    float* sy = sx + a.in_h() * a.in_w();
    blk.each([&](int t) {
        if (t < a.ws) g[t] = a.taps[t];
        a.stage(b, t, sx, sy);
    });
    blk.sync();
    blk.each([&](int t) { a.hpass(t, g, sx, sy, hs); });
    blk.sync();
    blk.each([&](int t) { red[t] = a.vpass(b, t, g, hs); });
    tree_to(blk, red, a.partial + b);
}

template <class B>
CK_D void psnr_block(const B& blk, const metrics::PsnrArgs& a, int64_t b, double* red) {
    blk.each([&](int t) { red[t] = a.thread_sum(b, t); });
    tree_to(blk, red, a.partial + b);
}

#ifdef MIGAN_EMULATE
int ssim_launch(const metrics::SsimArgs& a, int64_t blocks, ck_stream_t) {
    const size_t statics = (metrics::kMaxWindow + kThreads) * sizeof(double);
    return ck_blocks<kThreads>(blocks, statics + a.smem_bytes(), [&](auto& blk, int64_t b, void* smem) {
        double* g = static_cast<double*>(smem);
        double* red = g + metrics::kMaxWindow;
        ssim_block(blk, a, b, g, red, red + kThreads);
    });
}

int psnr_launch(const metrics::PsnrArgs& a, int64_t blocks, ck_stream_t) {
    return ck_blocks<kThreads>(blocks, kThreads * sizeof(double),
                               [&](auto& blk, int64_t b, void* smem) { psnr_block(blk, a, b, (double*)smem); });
}

// The per-image reduction is a warp's shuffle tree on the device, which the block layer has no counterpart for; the
// emulation build adds the lanes in the same tree.
int reduce_launch(const metrics::ReduceArgs& a, ck_stream_t) {
    for (int64_t i = 0; i < a.n; ++i) {
        double s[metrics::kWarp];
        for (int l = 0; l < metrics::kWarp; ++l) s[l] = a.lane_sum(i, l);
        for (int off = metrics::kWarp / 2; off > 0; off >>= 1)
            for (int l = 0; l < off; ++l) s[l] = dadd_rn(s[l], s[l + off]);
        a.finish_image(i, s[0]);
    }
    a.finish_mean();
    return 0;
}
#else
__global__ void __launch_bounds__(kThreads) metrics_ssim_tile_kernel(const __grid_constant__ metrics::SsimArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ double g[metrics::kMaxWindow];
    __shared__ double red[kThreads];
    ssim_block(DeviceBlock(), a, blockIdx.x, g, red, smem);
}

__global__ void __launch_bounds__(kThreads) metrics_psnr_kernel(const __grid_constant__ metrics::PsnrArgs a) {
    __shared__ double red[kThreads];
    psnr_block(DeviceBlock(), a, blockIdx.x, red);
}

__global__ void __launch_bounds__(kThreads) metrics_reduce_kernel(const __grid_constant__ metrics::ReduceArgs a) {
    const int lane = threadIdx.x % metrics::kWarp, warp = threadIdx.x / metrics::kWarp;
    for (int64_t i = warp; i < a.n; i += kThreads / metrics::kWarp) {
        double s = a.lane_sum(i, lane);
        for (int off = metrics::kWarp / 2; off > 0; off >>= 1) s = dadd_rn(s, __shfl_down_sync(0xffffffffu, s, off));
        if (lane == 0) a.finish_image(i, s);
    }
    __syncthreads();   // the per-image sums in global memory are visible to thread 0
    if (threadIdx.x == 0) a.finish_mean();
}

int ssim_launch(const metrics::SsimArgs& a, int64_t blocks, ck_stream_t s) {
    const int smem = (int)a.smem_bytes();
    if (int e = set_smem(metrics_ssim_tile_kernel, smem)) return e;
    metrics_ssim_tile_kernel<<<(unsigned)blocks, kThreads, smem, s>>>(a);
    return (int)cudaGetLastError();
}

int psnr_launch(const metrics::PsnrArgs& a, int64_t blocks, ck_stream_t s) {
    metrics_psnr_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(a);
    return (int)cudaGetLastError();
}

int reduce_launch(const metrics::ReduceArgs& a, ck_stream_t s) {
    metrics_reduce_kernel<<<1, kThreads, 0, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

constexpr int64_t kMaxBlocks = 0x7fffffff;   // gridDim.x

struct SsimShape {
    int Ho, Wo, tiles_x;
    int64_t tiles, parts, blocks;
};

int ssim_shape(int n, int C, int H, int W, int window, SsimShape* sh) {
    if (n < 1 || C < 1 || H < 1 || W < 1)
        return fail(MIGAN_ERR_INVALID, "ssim: bad batch n=%d C=%d H=%d W=%d (all >= 1)", n, C, H, W);
    if (window < 1 || window > METRICS_MAX_WINDOW)
        return fail(MIGAN_ERR_INVALID, "ssim: window %d outside 1..%d", window, METRICS_MAX_WINDOW);
    const int pad = window / 2;
    sh->Ho = H + 2 * pad - window + 1;
    sh->Wo = W + 2 * pad - window + 1;
    sh->tiles_x = (sh->Wo + metrics::kTileW - 1) / metrics::kTileW;
    sh->tiles = (int64_t)sh->tiles_x * ((sh->Ho + metrics::kTileH - 1) / metrics::kTileH);
    sh->parts = (int64_t)C * sh->tiles;
    sh->blocks = (int64_t)n * sh->parts;
    if (sh->blocks > kMaxBlocks)
        return fail(MIGAN_ERR_INVALID, "ssim: %lld tiles in one call (at most %lld); split the batch", (long long)sh->blocks,
                    (long long)kMaxBlocks);
    return 0;
}

struct PsnrShape {
    int Hv, Wv;
    int64_t chunks, blocks;
};

int psnr_shape(int n, int H, int W, int shave, PsnrShape* sh) {
    if (n < 1 || H < 1 || W < 1) return fail(MIGAN_ERR_INVALID, "psnr: bad batch n=%d H=%d W=%d (all >= 1)", n, H, W);
    if (shave < 0) return fail(MIGAN_ERR_INVALID, "psnr: shave %d < 0", shave);
    sh->Hv = H - 2 * shave;
    sh->Wv = W - 2 * shave;
    if (sh->Hv < 1 || sh->Wv < 1)
        return fail(MIGAN_ERR_INVALID, "psnr: shaving %d pixels from each side of %d x %d leaves an empty region", shave,
                    H, W);
    sh->chunks = (sh->Hv + metrics::kPsnrRows - 1) / metrics::kPsnrRows;
    sh->blocks = (int64_t)n * sh->chunks;
    if (sh->blocks > kMaxBlocks)
        return fail(MIGAN_ERR_INVALID, "psnr: %lld row chunks in one call (at most %lld); split the batch",
                    (long long)sh->blocks, (long long)kMaxBlocks);
    return 0;
}

size_t workspace_bytes(int n, int64_t parts) { return (size_t)(n * parts + n) * sizeof(double); }

int check_workspace(const char* who, const void* ws, size_t have, size_t need) {
    if (!ws) return fail(MIGAN_ERR_INVALID, "%s: null workspace", who);
    if (reinterpret_cast<uintptr_t>(ws) % alignof(double))
        return fail(MIGAN_ERR_INVALID, "%s: workspace not 8-byte aligned", who);
    if (have < need) return fail(MIGAN_ERR_INVALID, "%s: workspace of %zu bytes, %zu needed", who, have, need);
    return 0;
}

}  // namespace

extern "C" {

size_t metrics_ssim_workspace_bytes(int n, int C, int H, int W, int window) {
    SsimShape sh;
    if (ssim_shape(n, C, H, W, window, &sh)) return 0;
    return workspace_bytes(n, sh.parts);
}

int metrics_ssim(const float* img1, const float* img2, int n, int C, int H, int W, const float* taps, int window,
                 float* per_image, float* mean, void* workspace, size_t workspace_bytes_, void* stream) {
    if (!img1 || !img2 || !taps) return fail(MIGAN_ERR_INVALID, "ssim: null img1 / img2 / taps");
    if (!per_image && !mean) return fail(MIGAN_ERR_INVALID, "ssim: per_image and mean are both null");
    SsimShape sh;
    if (int rc = ssim_shape(n, C, H, W, window, &sh)) return rc;
    if (int rc = check_workspace("ssim", workspace, workspace_bytes_, workspace_bytes(n, sh.parts))) return rc;
    double* partial = static_cast<double*>(workspace);
    metrics::SsimArgs a{img1, img2, partial, H, W, sh.Ho, sh.Wo, window, window / 2, sh.tiles_x, sh.tiles, {}};
    for (int k = 0; k < window; ++k) a.taps[k] = taps[k];
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    CUDA_TRY(ssim_launch(a, sh.blocks, s));
    const metrics::ReduceArgs r{partial, partial + n * sh.parts, n, sh.parts, (double)C * sh.Ho * sh.Wo, per_image, mean,
                                nullptr};
    CUDA_TRY(reduce_launch(r, s));
    return 0;
}

size_t metrics_psnr_workspace_bytes(int n, int H, int W, int shave) {
    PsnrShape sh;
    if (psnr_shape(n, H, W, shave, &sh)) return 0;
    return workspace_bytes(n, sh.chunks);
}

int metrics_psnr(const float* pred, const float* gt, int n, int C, int H, int W, int gray, int shave, float rgb_range,
                 double* out, void* workspace, size_t workspace_bytes_, void* stream) {
    if (!pred || !gt || !out) return fail(MIGAN_ERR_INVALID, "psnr: null pred / gt / out");
    if (C < 1) return fail(MIGAN_ERR_INVALID, "psnr: C=%d (>= 1)", C);
    if (gray && C != 3) return fail(MIGAN_ERR_INVALID, "psnr: the gray difference needs C == 3, got C=%d", C);
    if (!(rgb_range > 0.f)) return fail(MIGAN_ERR_INVALID, "psnr: rgb_range %g (> 0)", (double)rgb_range);
    PsnrShape sh;
    if (int rc = psnr_shape(n, H, W, shave, &sh)) return rc;
    if (int rc = check_workspace("psnr", workspace, workspace_bytes_, workspace_bytes(n, sh.chunks))) return rc;
    double* partial = static_cast<double*>(workspace);
    const metrics::PsnrArgs a{pred, gt, partial, C, H, W, shave, sh.Hv, sh.Wv, gray ? 1 : 0, sh.chunks, rgb_range};
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    CUDA_TRY(psnr_launch(a, sh.blocks, s));
    const metrics::ReduceArgs r{partial, partial + n * sh.chunks, n, sh.chunks,
                                (double)(gray ? 1 : C) * sh.Hv * sh.Wv, nullptr, nullptr, out};
    CUDA_TRY(reduce_launch(r, s));
    return 0;
}

}  // extern "C"

// wgmma fused SeparableConv2d kernel: host-side plan + launcher (sepconv_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace migan {

// One resolved launch: tensor maps, tiling and pipeline depths are computed once per
// (batch size, workspace) at plan time and replayed by every forward.  The kernel parameter
// block is opaque here (defined in sepconv_tc.cu).
struct SepconvTcArgs {
    unsigned grid = 0;
    unsigned smem_bytes = 0;
    int num_tiles = 0;
    const void* bound_x = nullptr;     // STEM: the x pointer the input tensor map currently encodes
    alignas(64) unsigned char params_blob[2048];
};

// Optional fused torgb + image path in the epilogue (all output channels in one CTA tile).
struct SepconvTcRgb {
    const float* w;       // [3][cout]
    const float* b;       // [3]
    const float* fir;     // [16][3] taps of the image up-sampling (unused if img_lo == null)
    const float* img_lo;  // [n][3][h/2][w/2] planar or null
    float* img_out;       // [n][3][h][w] planar (may be overridden at launch: the caller's y)
    int store_out;        // 0: do not write the feature map (last block)
};

// Where the depthwise conv's input (or the A operand itself) comes from.  Every tensor is [n, h, w, ...]: h and w need not
// be equal or powers of two (a fully convolutional forward); tiles that reach past the right / bottom edge are zero-filled
// on load and masked on store.
enum SepconvSource {
    SEPCONV_SRC_NHWC = 0,   // in_f32: NHWC fp32 tensor [n, h, w, cin] (TMA tile + halo)
    SEPCONV_SRC_SPLIT = 1,  // a_hi / a_lo: pre-split fp16 operand [n, h, w, cin] loaded by TMA (no prologue)
    SEPCONV_SRC_UP = 2,     // in_f32 = skip tensor [n,h,w,cin]; x = lrelu_agc(up2(up_t) + noise) + skip is rebuilt
                            // in shared memory from up_t [n,h/2,w/2,cin] (the previous layer's raw 1x1 output)
    SEPCONV_SRC_STEM = 3,   // x NCHW [n,4,h,w] (bound at launch); fromrgb + activation recomputed on the halo
};

struct SepconvTcDesc {
    int passes = 3;                 // 3 = fp16 hi/lo split (fp32-faithful), 1 = single fp16 pass
    int source = SEPCONV_SRC_NHWC;
    const float* in_f32 = nullptr;
    const __half* a_hi = nullptr;
    const __half* a_lo = nullptr;
    const float* w9 = nullptr;      // [9][cin] depthwise taps * (64 * sqrt2)
    const float* bias = nullptr;    // [cin]              * (64 * sqrt2)
    const __half* w_hi = nullptr;   // [cout][cin] fp16 hi / lo of w * 2^k
    const __half* w_lo = nullptr;
    float inv_scale = 1.f;
    const float* noise = nullptr;   // [h][noise_pitch] added before the epilogue activation
    float* out = nullptr;           // [n, h, w, cout] NHWC fp32
    int n = 0, h = 0, w = 0, cin = 0, cout = 0, act = 0;
    int noise_pitch = 0;            // row pitch (floats, a multiple of 4) of noise and up_noise
    const SepconvTcRgb* rgb = nullptr;
    // SEPCONV_SRC_UP
    const float* up_t = nullptr;
    const float* up_noise = nullptr;   // [h][noise_pitch] * sqrt2 or null
    float up_taps[16] = {0};           // 4x4 FIR taps * sqrt2 (channel-uniform)
    // SEPCONV_SRC_STEM
    const float* stem_w = nullptr;     // [cin][4] * sqrt2
    const float* stem_b = nullptr;     // [cin]    * sqrt2
};

// Returns nullptr on success, else an error string.
const char* sepconv_tc_plan_ex(SepconvTcArgs* a, const SepconvTcDesc& d);

// What the planner chose for one launch (tests enumerate schedules with it).
struct SepconvTcPlanInfo {
    int n_group, in_stages, a_stages, b_stages, b_resident, dw_global;
    int tile_w, tile_h, tile_n, n_tile, grid, num_tiles, num_candidates;
    int ep_stages, ep_offset, ep_stage_bytes;   // epilogue window ring (0 stages: none) and its place in dynamic smem
    int smem_bytes;                              // dynamic shared memory of the launch
};
// sepconv_tc_plan_ex with the planner's two inputs made explicit, for tests: `sms` SMs for the persistent grid (0: the
// device's minus MIGAN_TC_RESERVE_SMS, as in production) and, if candidate >= 0, the candidate-th layout of the planner's own
// preference list (an error if it does not fit) instead of the first that fits.  a == nullptr plans only: no tensor
// map, no pointer and no CUDA call.
const char* sepconv_tc_plan_debug(SepconvTcArgs* a, const SepconvTcDesc& d, int sms, int candidate, SepconvTcPlanInfo* info);
// Whether a launch with d's shapes and source can fuse torgb, i.e. hold all of cout in one CTA tile (d.rgb and the
// pointers are not read).
bool sepconv_tc_fuses_rgb(const SepconvTcDesc& d);
// Legacy form (plain / pre-split sources, res x res).
const char* sepconv_tc_plan(SepconvTcArgs* a, int passes, const float* in_f32, const __half* a_hi, const __half* a_lo,
                            const float* w9, const float* bias, const __half* w_hi, const __half* w_lo,
                            float inv_scale, const float* noise, float* out, int n, int res, int cin, int cout, int act,
                            const SepconvTcRgb* rgb = nullptr);
// Non-zero after a kernel gave up on a pipeline wait (code | parity << 12 | block << 16); 0 otherwise.
int sepconv_tc_timeout_record(int device);
// img_out_override: the caller's y for the last block; x_nchw: the caller's x for SEPCONV_SRC_STEM launches.
cudaError_t launch_sepconv_tc(SepconvTcArgs& a, cudaStream_t s, float* img_out_override = nullptr, const float* x_nchw = nullptr);

}  // namespace migan

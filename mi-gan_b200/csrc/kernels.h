// Internal launcher interface between the plan executor (migan_abi.cu) and the kernels.
// Activations are NHWC fp32 in HBM ([n, H, W, C], C a multiple of 4, 16-byte aligned);
// the RGB image path is planar NCHW fp32 ([n, 3, H, W]) so the last level is the output.
// H and W are a level's extent: equal powers of two at the model resolution, any sizes in a fully convolutional forward.
// Noise planes are [H][pitch] with pitch >= W a multiple of 4 (16-byte rows for TMA).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "../../include/migan_b200.h"

namespace migan {

// Per-device one-time setup (dynamic shared memory opt-in); called by migan_create.
cudaError_t configure_elementwise();
cudaError_t configure_sepconv_tc();

// ---- CUDA-core kernels (elementwise.cu) ---------------------------------------------
// What a launcher launched, for the stage test hook (migan_debug_stage): rows per thread, the C / G template, the first
// launch's grid and the number of image-group launches.  dry: check the arguments and fill the record, launch nothing.
struct StageLaunch { bool dry = false; int rs = 0, cg = 0, groups = 0; unsigned grid = 0; };

// fromrgb 1x1 (4 -> C0) + bias + lrelu_agc;  x NCHW [n,4,H,W] -> out NHWC [n,H,W,C0]  (H * W a multiple of 4)
cudaError_t launch_stem(const float* x_nchw, const float* w, const float* b, float* out,
                        int n, int H, int W, int C0, cudaStream_t s, StageLaunch* sl = nullptr);
// depthwise 3x3 (pad 1) + bias + lrelu_agc, NHWC -> NHWC.  w9 is tap-major [9][C].
// Writes fp32 (out, if non-null) and/or the scaled fp16 hi/lo split (out_hi/out_lo, if non-null).
cudaError_t launch_dw3x3(const float* in, const float* w9, const float* bias, float* out, __half* out_hi, __half* out_lo,
                         int n, int H, int W, int C, cudaStream_t s, StageLaunch* sl = nullptr);
// depthwise 3x3 + bias + lrelu_agc, then 4x4 FIR stride 2 pad 1 (taps fir16 [16][C]) -> fp32 [n,H/2,W/2,C] (CUDA-core path).
cudaError_t launch_dw3x3_down(const float* in, const float* w9, const float* bias, const float* fir16, float* out_f32,
                              int n, int H, int W, int C, cudaStream_t s, StageLaunch* sl = nullptr);
// Same stage specialised for the tensor-core feed (pre-split fp16 hi/lo output only): w9s / biass are the taps and bias
// pre-multiplied by kActSplitScale * sqrt(2); C = 512, the width of every level a forward runs it at (below 16 x 16).
cudaError_t launch_dw3x3_down_split(const float* in, const float* w9s, const float* biass, const float* fir16,
                                    __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s,
                                    StageLaunch* sl = nullptr);
// TMA-staged variant (W/2 >= 16 and even, H/2 >= 8): a producer warp streams the input rows of a (64-channel, 36-column) slab into a shared-memory
// ring with cp.async.bulk.tensor (out-of-image rows / columns arrive zero-filled), so the row walk never waits on global
// memory.  `desc` = 128-byte CUtensorMap of the input made by make_down_tensor_map (host, once per plan).
struct alignas(64) DownTensorMap { unsigned char bytes[128]; };
const char* make_down_tensor_map(DownTensorMap* desc, const float* in, int n, int H, int W, int C);   // sepconv_tc.cu (driver entry point lives there)
cudaError_t launch_dw3x3_down_tma(const DownTensorMap& desc, const float* w9s, const float* biass, const float* fir16,
                                  __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s,
                                  StageLaunch* sl = nullptr);
// 2x polyphase FIR up-sampling of the raw 1x1-conv output + noise + lrelu_agc + skip add.
// t [n,h,w,C] -> out [n,2h,2w,C]; fir16 [16][C] (gain included); noise [2h][noise_pitch] (already
// multiplied by noise_strength) or null; skip [n,2h,2w,C] or null (added AFTER the activation).
cudaError_t launch_up2(const float* t, const float* fir16, const float* noise, int noise_pitch, const float* skip,
                       float* out, int n, int h, int w, int C, cudaStream_t s, StageLaunch* sl = nullptr);
// img_out[n,3,h,w] = up2(img_lo[n,3,h/2,w/2]) + torgb(x[n,h,w,C]) + b;  img_lo may be null (b4).
cudaError_t launch_torgb(const float* x, const float* w, const float* b, const float* img_lo,
                         const float* fir16x3, float* img_out, int n, int h, int wd, int C, cudaStream_t s,
                         StageLaunch* sl = nullptr);
cudaError_t launch_add(float* x, const float* y, int64_t numel, cudaStream_t s, StageLaunch* sl = nullptr);
// Noise planes of a fully convolutional forward, all in one launch: dst[y][x] = src[y % r][x % r] for y < H, x < W (rows
// `pitch` floats apart, padding columns zero); src = a level's r x r plane as uploaded (noise_const * noise_strength [* sqrt 2]).
struct NoiseTile { const float* src; float* dst; int r, H, W, pitch; };
constexpr int kMaxNoiseTiles = 32;
struct NoiseTileBatch { NoiseTile t[kMaxNoiseTiles]; int count; };
cudaError_t launch_noise_tile(const NoiseTileBatch& b, cudaStream_t s, StageLaunch* sl = nullptr);
cudaError_t launch_nhwc_to_nchw(const float* in, float* out, int n, int H, int W, int C, cudaStream_t s);
cudaError_t launch_split_f16(const float* in, __half* hi, __half* lo, float scale, int64_t numel, cudaStream_t s);

// ---- fp32 CUDA-core GEMM for the 1x1 conv (gemm_simt.cu) ----------------------------
// out[p][n] = epilogue( sum_k A[p][k] * Bt[k][n] ), A [P][K], Bt [K][N], out [P][N].
// epilogue: + noise (if non-null; pixel p = image pixel (y, x) of [H][W] reads noise[y * noise_pitch + x]) then lrelu_agc (if act).
cudaError_t launch_pw_gemm_simt(const float* A, const float* Bt, float* out, int64_t P, int K, int N,
                                const float* noise, int H, int W, int noise_pitch, int act, cudaStream_t s);

// ---- standalone ops (ops.cu) ---------------------------------------------------------
cudaError_t launch_upfirdn2d(const float* x, const float* f, float* y, int n, int c, int h, int w,
                             int fh, int fw, int upx, int upy, int downx, int downy,
                             int padx0, int padx1, int pady0, int pady1, int flip, float gain,
                             int oh, int ow, cudaStream_t s);
cudaError_t launch_bias_act(const float* x, const float* b, float* y, int64_t numel, int64_t step_b, int size_b,
                            int act, float alpha, float gain, float clamp, cudaStream_t s);

// ---- uint8 pre/post-processing (prepost.cu): demo.py:56-66 and :135-142 around the forward ------
int launch_preprocess_u8(const uint8_t* img_hwc, const uint8_t* mask_hw, float* x_nchw, int n, int H, int W, cudaStream_t s);
int launch_postprocess_u8(const float* y_nchw, const uint8_t* img_hwc, const uint8_t* mask_hw, uint8_t* out_hwc, int n, int H, int W,
                          cudaStream_t s);

}  // namespace migan

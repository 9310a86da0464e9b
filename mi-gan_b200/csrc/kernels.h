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
// fromrgb 1x1 (4 -> C0) + bias + lrelu_agc;  x NCHW [n,4,H,W] -> out NHWC [n,H,W,C0]  (H * W a multiple of 4)
cudaError_t launch_stem(const float* x_nchw, const float* w, const float* b, float* out,
                        int n, int H, int W, int C0, cudaStream_t s);
// depthwise 3x3 (pad 1) + bias + lrelu_agc, NHWC -> NHWC.  w9 is tap-major [9][C].
// Writes fp32 (out, if non-null) and/or the scaled fp16 hi/lo split (out_hi/out_lo, if non-null).
cudaError_t launch_dw3x3(const float* in, const float* w9, const float* bias, float* out, __half* out_hi, __half* out_lo,
                         int n, int H, int W, int C, cudaStream_t s);
// depthwise 3x3 + bias + lrelu_agc, then 4x4 FIR stride 2 pad 1 (taps fir16 [16][C]).
// Writes fp32 [n,H/2,W/2,C] to out_f32 (if non-null) and/or the scaled fp16 hi/lo split
// (if out_hi non-null) that the wgmma GEMM consumes directly through TMA.
cudaError_t launch_dw3x3_down(const float* in, const float* w9, const float* bias, const float* fir16,
                              float* out_f32, __half* out_hi, __half* out_lo,
                              int n, int H, int W, int C, cudaStream_t s);
// Same stage specialised for the tensor-core feed (pre-split fp16 hi/lo output only): w9s / biass are the taps and bias
// pre-multiplied by kActSplitScale * sqrt(2); C in {64, 128, 256, 512}.
cudaError_t launch_dw3x3_down_split(const float* in, const float* w9s, const float* biass, const float* fir16,
                                    __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s);
// TMA-staged variant (W/2 >= 16 and even): a producer warp streams the input rows of a (64-channel, 36-column) slab into a shared-memory
// ring with cp.async.bulk.tensor (out-of-image rows / columns arrive zero-filled), so the row walk never waits on global
// memory.  `desc` = 128-byte CUtensorMap of the input made by make_down_tensor_map (host, once per plan).
struct alignas(64) DownTensorMap { unsigned char bytes[128]; };
const char* make_down_tensor_map(DownTensorMap* desc, const float* in, int n, int H, int W, int C);   // sepconv_tc.cu (driver entry point lives there)
cudaError_t launch_dw3x3_down_tma(const DownTensorMap& desc, const float* w9s, const float* biass, const float* fir16,
                                  __half* out_hi, __half* out_lo, int n, int H, int W, int C, cudaStream_t s);
// 2x polyphase FIR up-sampling of the raw 1x1-conv output + noise + lrelu_agc + skip add.
// t [n,h,w,C] -> out [n,2h,2w,C]; fir16 [16][C] (gain included); noise [2h][noise_pitch] (already
// multiplied by noise_strength) or null; skip [n,2h,2w,C] or null (added AFTER the activation).
cudaError_t launch_up2(const float* t, const float* fir16, const float* noise, int noise_pitch, const float* skip,
                       float* out, int n, int h, int w, int C, cudaStream_t s);
// img_out[n,3,h,w] = up2(img_lo[n,3,h/2,w/2]) + torgb(x[n,h,w,C]) + b;  img_lo may be null (b4).
cudaError_t launch_torgb(const float* x, const float* w, const float* b, const float* img_lo,
                         const float* fir16x3, float* img_out, int n, int h, int wd, int C, cudaStream_t s);
cudaError_t launch_add(float* x, const float* y, int64_t numel, cudaStream_t s);
// Noise planes of a fully convolutional forward, all in one launch: dst[y][x] = src[y % r][x % r] for y < H, x < W (rows
// `pitch` floats apart, padding columns zero); src = a level's r x r plane as uploaded (noise_const * noise_strength [* sqrt 2]).
struct NoiseTile { const float* src; float* dst; int r, H, W, pitch; };
constexpr int kMaxNoiseTiles = 32;
struct NoiseTileBatch { NoiseTile t[kMaxNoiseTiles]; int count; };
cudaError_t launch_noise_tile(const NoiseTileBatch& b, cudaStream_t s);
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
// feathered composite of the ONNX pipeline (create_onnx_pipeline.py:233-245): NCHW uint8 image / mask, 25 smoothing taps (host array)
int launch_feather_composite(const float* y_nchw, const uint8_t* img_nchw, const uint8_t* mask_n1hw, uint8_t* out_nchw, int n, int H, int W,
                             const float* k25_host, cudaStream_t s);
int launch_preprocess_u8(const uint8_t* img_hwc, const uint8_t* mask_hw, float* x_nchw, int n, int H, int W, cudaStream_t s);
int launch_postprocess_u8(const float* y_nchw, const uint8_t* img_hwc, const uint8_t* mask_hw, uint8_t* out_hwc, int n, int H, int W,
                          cudaStream_t s);



// ---- arbitrary-resolution crop pipeline (pipeline.cu): scripts/create_onnx_pipeline.py:121-264 ------
size_t pipeline_scratch_bytes(int H, int W, int res);
int launch_resize_nearest_u8(const uint8_t* in, int H, int W, uint8_t* out, int oh, int ow, cudaStream_t s);
int launch_hole_flags(const uint8_t* mask, int H, int W, uint8_t* flags, cudaStream_t s);
void crop_box_from_flags(const uint8_t* flags_host, int H, int W, int res, int padding, int* box4);
int launch_pipeline_preprocess(const uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res, float* x,
                               void* scratch, cudaStream_t s);
int launch_pipeline_postprocess(const float* y, uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res,
                                const float* k25_host, void* scratch, cudaStream_t s);
// batches of 1..MIGAN_PIPE_MAX_BATCH requests of any sizes, one launch per stage
size_t pipeline_batch_scratch_bytes(const migan_pipe_request* reqs, int n, int res);
int check_pipe_batch(const migan_pipe_request* reqs, int n, int res, bool boxes, char* msg, size_t len);
int launch_hole_flags_batch(const migan_pipe_request* reqs, int n, uint8_t* flags, cudaStream_t s);
int launch_pipeline_preprocess_batch(const migan_pipe_request* reqs, int n, int res, float* x, void* scratch, cudaStream_t s);
int launch_pipeline_postprocess_batch(const float* y, const migan_pipe_request* reqs, int n, int res, const float* k25_host,
                                      void* scratch, cudaStream_t s);
// the same batches with the crop windows planned on the device from the flags (no host round trip)
int check_pipe_planned(const migan_pipe_request* reqs, int n, int res, char* msg, size_t len);
size_t pipeline_batch_scratch_bound(const migan_pipe_request* reqs, int n, int res);
int launch_pipeline_plan_batch(const migan_pipe_request* reqs, int n, int res, int padding, const uint8_t* flags, int* boxes,
                               void* scratch, cudaStream_t s);
int launch_pipeline_preprocess_planned(const migan_pipe_request* reqs, int n, int res, float* x, void* scratch, cudaStream_t s);
int launch_pipeline_postprocess_planned(const float* y, const migan_pipe_request* reqs, int n, int res, const float* k25_host,
                                        void* scratch, cudaStream_t s);

// ---- the reference demo's request path at any photo size (demo_resize.cu): scripts/demo.py:26-66, :120-143 ------
int demo_resized_size(int w, int h, int max_size, int* ow, int* oh);
int check_demo_batch(const migan_demo_request* reqs, int n, int res, char* msg, size_t len);
size_t demo_scratch_bytes(const migan_demo_request* reqs, int n, int res);
int launch_demo_preprocess(const migan_demo_request* reqs, int n, int res, float* x, void* scratch, cudaStream_t s);
// the evaluation batch (evaluate_fid_lpips.py InferenceDataset + :246-249) on the same stages
int check_eval_batch(const migan_demo_request* reqs, int n, int res, char* msg, size_t len);
size_t eval_scratch_bytes(const migan_demo_request* reqs, int n, int res);
int launch_eval_preprocess(const migan_demo_request* reqs, int n, int res, float* x, float* img, void* scratch, cudaStream_t s);
int launch_eval_composite(const float* x, const float* y, int n, int res, float* real, float* composed, cudaStream_t s);
int launch_demo_postprocess(const float* y, const migan_demo_request* reqs, int n, int res, void* scratch, cudaStream_t s);

// ---- full-resolution request path (fullres.cu): reflect padding and the composite around migan_forward_hw ------
int check_fullres_batch(const migan_fullres_request* reqs, int n, bool pre, char* msg, size_t len);
int launch_fullres_preprocess(const migan_fullres_request* reqs, int n, cudaStream_t s);
int launch_fullres_postprocess(const migan_fullres_request* reqs, int n, cudaStream_t s);
// the same kernels on windows of a photo (the whole photo is the window (0, 0, H, W))
int check_window_batch(const migan_window_request* reqs, int n, bool pre, char* msg, size_t len);
int launch_window_preprocess(const migan_window_request* reqs, int n, cudaStream_t s);
int launch_window_postprocess(const migan_window_request* reqs, int n, cudaStream_t s);

// ---- hole-window request path (holewin.cu): hole cells on the device, the window planner on the host ------
int check_hole_cells(const migan_cells_request* reqs, int n, int res, char* msg, size_t len);
size_t hole_cells_bytes(const migan_cells_request* reqs, int n, int res);
int launch_hole_cells(const migan_cells_request* reqs, int n, int res, uint8_t* cells, cudaStream_t s);
int hole_windows_max(int H, int W, int res, int* max_windows, char* msg, size_t len);
int hole_windows(const uint8_t* cells_host, int H, int W, int res, int margin, int* win4, int max_windows, int* count, char* msg,
                 size_t len);

// ---- free-form masks of the evaluation protocol (masks.cu): numpy's stream on the host, the rasterizer on the device ----
void np_seed(migan_np_random* st, uint32_t seed);
int check_mask_size(int s, int n_att, char* msg, size_t len);
int mask_plan(migan_np_random* st, int s, int n_att, migan_mask_record* recs, migan_np_random* states, char* msg, size_t len);
int launch_mask_raster(const migan_mask_record* recs, int n_att, int s, uint8_t* attempts, int* holes, cudaStream_t s_);
int launch_mask_compact(const uint8_t* attempts, const int* holes, int n_att, int s, int n, uint8_t* out, cudaStream_t s_);


// ---- training snapshot -> inference filters (reparam.cu): scripts/export_inference_model.py:18-27 ------
int launch_reparam_filter(const float* const* w_dev, int k, int cout, int64_t fan, float* out, cudaStream_t s);

}  // namespace migan

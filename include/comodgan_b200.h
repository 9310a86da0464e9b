/* comodgan_b200.h -- C ABI of the H100-native Co-Mod-GAN generator forward and of conv2d_resample.
 *
 * Same shared library and conventions as migan_b200.h (return 0 / non-zero code, comodgan_last_error(), fp32
 * device pointers, `stream` = cudaStream_t as void*, no CPU fallback).  Reference interfaces replaced
 * (file:line in /root/reference):
 *
 *   comodgan_create / _destroy        Generator(Mapping(num_ws), Encoder(resolution), Synthesis(resolution))
 *                                     scripts/demo.py:95-100; lib/model_zoo/comodgan.py:113-204, 346-396, 424-435
 *   comodgan_set_weight / _finalize   load_state_dict (scripts/demo.py:110): key names + shapes = the reference
 *                                     state_dict (180 entries, 79.35 M values @256)
 *   comodgan_forward                  Generator.forward(x, z, c=None, truncation_psi, truncation_cutoff, noise_mode)
 *                                     lib/model_zoo/comodgan.py:438-455 (eval mode, fp32)
 *   b200_conv2d_resample              conv2d_resample(x, w, f, up, down, padding, groups, flip_weight, flip_filter)
 *                                     torch_utils/ops/conv2d_resample.py:59-154 (all six branches)
 */
#ifndef COMODGAN_B200_H_
#define COMODGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COMODGAN_NOISE_NONE 0
#define COMODGAN_NOISE_CONST 1
#define COMODGAN_NOISE_RANDOM 2   /* caller supplies the N(0,1) planes (the reference draws them with torch.randn) */

typedef struct comodgan_ctx comodgan_ctx;

const char* comodgan_last_error(void);

/* resolution: power of two >= 8 (ValueError in the reference otherwise, comodgan.py:132-134, 360-362);
 * num_ws = 2*log2(resolution) - 2 (14 @256, 16 @512, comodgan.py:371-374).  device < 0: description only. */
int comodgan_create(int resolution, int device, comodgan_ctx** out);
int comodgan_destroy(comodgan_ctx* ctx);

int comodgan_num_weights(const comodgan_ctx* ctx);
int comodgan_weight_info(const comodgan_ctx* ctx, int index, const char** name, int* ndim, int64_t shape[4]);
/* HOST pointer, fp32, contiguous, reference layout. */
int comodgan_set_weight(comodgan_ctx* ctx, const char* name, const float* host_data, int64_t numel);
/* Checks every key was given; folds the equalised-lr gains, the demodulation pre-normalisation
 * (stylegan.py:145) and the NCHW<->NHWC permutations of the two bottleneck dense layers into the packed GEMM operands. */
int comodgan_finalize_weights(comodgan_ctx* ctx);

size_t comodgan_workspace_bytes(const comodgan_ctx* ctx, int n);

/* Number of float planes comodgan_forward reads from `noise` in COMODGAN_NOISE_RANDOM mode, and their sizes: plane i
 * (forward order: b4.conv, b8.conv0, b8.conv1, ...) is [n, r_i, r_i]. */
int comodgan_num_noise_planes(const comodgan_ctx* ctx);
int comodgan_noise_plane_res(const comodgan_ctx* ctx, int index);

/* y[n,3,R,R] = G(x[n,4,R,R], z[n,512]).  truncation_cutoff < 0 = None (all ws).  noise: device pointer to the
 * concatenated planes (RANDOM mode only, else NULL).  Asynchronous on `stream`. */
int comodgan_forward(comodgan_ctx* ctx, const float* x, const float* z, float* y, int n,
                     float truncation_psi, int truncation_cutoff, int noise_mode, const float* noise,
                     void* workspace, size_t workspace_bytes, void* stream);

int comodgan_last_launch_count(const comodgan_ctx* ctx);

/* Debug/test tap (see migan_set_tap): copy the named intermediate, as NCHW fp32, into dst during the next forwards.
 * Names follow oracle/comodgan_oracle.py ("encoder.b256.conv0.out", "synthesis.b64.img", "mapping.ws" ...). */
int comodgan_set_tap(comodgan_ctx* ctx, const char* name, float* dst);

/* conv2d_resample on NCHW device tensors: x[n,cin,h,w], w[cout,cin/groups,kh,kw], f[fh,fw] (fh = fw = 0: no filter, f ignored);
 * padding = [px0, px1, py0, py1] with respect to the up-sampled image.  out_h/out_w receive the output size
 * (either may be NULL).  y == NULL: only compute the output size and the workspace requirement (no device work). */
int b200_conv2d_resample(const float* x, const float* w, const float* f, float* y,
                         int n, int cin, int h, int wd, int cout, int kh, int kw, int fh, int fw,
                         int up, int down, int px0, int px1, int py0, int py1, int groups,
                         int flip_weight, int flip_filter,
                         void* workspace, size_t workspace_bytes, size_t* workspace_needed,
                         int* out_h, int* out_w, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COMODGAN_B200_H_ */

/* lpips_b200.h -- C ABI of the H100-native LPIPS distance (lpips.LPIPS(net="alex", version="0.1")).
 *
 * Same shared library and conventions as inception_b200.h (return 0 / non-zero MIGAN_ERR_* code, fp32 device pointers,
 * `stream` = cudaStream_t as void*, no CPU fallback); the error message is migan_last_error()'s.
 *
 *   lpips_create / _destroy        LPIPS 0.1 on AlexNet features[0:12], linear layers on, not spatial
 *   lpips_set_weight / _finalize   load_state_dict of lpips.LPIPS(net="alex").state_dict(): scaling_layer.shift / .scale,
 *                                  net.slice{1..5}.{0,3,6,8,10}.weight / .bias, lin{0..4}.model.1.weight (17 entries)
 *   lpips_forward                  model(in0, in1, normalize=...) for n image pairs, and the five layer terms
 */
#ifndef LPIPS_B200_H_
#define LPIPS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LPIPS_LAYERS 5
/* The smallest H and W AlexNet features[0:12] takes: 31 leaves one pixel after the second max pool, 30 none. */
#define LPIPS_MIN_SIZE 31

typedef struct lpips_ctx lpips_ctx;

/* device < 0: description only (weight spec, launch plan). */
int lpips_create(int device, lpips_ctx** out);
int lpips_destroy(lpips_ctx* ctx);

int lpips_num_weights(const lpips_ctx* ctx);
int lpips_weight_info(const lpips_ctx* ctx, int index, const char** name, int* ndim, int64_t shape[4]);
/* HOST pointer, fp32, contiguous, the lpips state_dict layout. */
int lpips_set_weight(lpips_ctx* ctx, const char* name, const float* host_data, int64_t numel);
/* Checks every key was given and packs the TF32 hi / lo operands of the five convolutions. */
int lpips_finalize_weights(lpips_ctx* ctx);

/* Device bytes lpips_forward needs for n pairs of H x W (0 on bad arguments). */
size_t lpips_workspace_bytes(const lpips_ctx* ctx, int n, int H, int W);
/* out[n] (fp32, device) = LPIPS(in0[i], in1[i]) of in0, in1 [n][3][H][W] (fp32 NCHW, device, H, W >= LPIPS_MIN_SIZE);
 * normalize != 0 maps [0, 1] inputs to [-1, 1] first.  per_layer[5][n] (device, or NULL) receives the five layer terms
 * whose sum out is.  The two inputs run as one batch of 2n images; pair i's value does not depend on n or on i.
 * Asynchronous on `stream`. */
int lpips_forward(lpips_ctx* ctx, const float* in0, const float* in1, int n, int H, int W, int normalize, float* out,
                  float* per_layer, void* workspace, size_t workspace_bytes, void* stream);
int lpips_last_launch_count(const lpips_ctx* ctx);

/* The forward's launches for n pairs of H x W, one per line ("<kind> <name> key=value ..."), written to buf (NUL
 * terminated, truncated to cap bytes); returns the full length, or minus an error code.  Works on a description-only
 * context. */
int lpips_launch_plan(const lpips_ctx* ctx, int n, int H, int W, char* buf, int cap);

/* ---- the input stage on its own -------------------------------------------------------------------------------------
 * y[2n][H][W][4] (NHWC, device): image i of in0, then image i of in1, each channel c mapped to
 * ((normalize ? 2x - 1 : x) - shift[c]) / scale[c]; channel 3 = 0.  shift, scale: 3 host floats. */
int lpips_input(const float* in0, const float* in1, int n, int H, int W, int normalize, const float* shift,
                const float* scale, float* y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LPIPS_B200_H_ */

/* inception_b200.h -- C ABI of the H100-native FID InceptionV3 feature extractor and of the feature statistics.
 *
 * Same shared library and conventions as migan_b200.h (return 0 / non-zero MIGAN_ERR_* code, fp32 device pointers,
 * `stream` = cudaStream_t as void*, no CPU fallback); the error message is migan_last_error()'s.
 *
 *   inception_create / _destroy        pytorch_fid InceptionV3([3]) with resize_input, normalize_input and the FID
 *                                      Inception blocks (fid_inception_v3(): torchvision Inception3, 1008 classes, no
 *                                      aux logits, FID variants of Mixed_5b..5d, 6b..6e, 7b, 7c)
 *   inception_set_weight / _finalize   load_state_dict of pt_inception-2015-12-05: torchvision Inception3 key names
 *                                      and shapes (472 entries besides num_batches_tracked, fc.* accepted and unused)
 *   inception_features                 model(x)[0].view(n, 2048): the 2048-d pool3 features of x[n,3,H,W] in [0, 1]
 *   fid_stats_update                   the float64 running sums behind np.mean / np.cov(rowvar=False) of the features
 */
#ifndef INCEPTION_B200_H_
#define INCEPTION_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define INCEPTION_FEATURES 2048
#define INCEPTION_SIZE 299

typedef struct inception_ctx inception_ctx;

/* device < 0: description only (weight spec, launch plan). */
int inception_create(int device, inception_ctx** out);
int inception_destroy(inception_ctx* ctx);

int inception_num_weights(const inception_ctx* ctx);
int inception_weight_info(const inception_ctx* ctx, int index, const char** name, int* ndim, int64_t shape[4]);
/* HOST pointer, fp32, contiguous, torchvision layout.  Keys ending in "num_batches_tracked" are accepted and ignored. */
int inception_set_weight(inception_ctx* ctx, const char* name, const float* host_data, int64_t numel);
/* Checks every key was given, folds each BatchNorm2d(eps=0.001) into its convolution in double (w * g / sqrt(var + eps),
 * b - mean * g / sqrt(var + eps), each rounded once to fp32) and packs the TF32 hi / lo operands of the convolutions. */
int inception_finalize_weights(inception_ctx* ctx);

/* Device bytes inception_features needs for n images of H x W (0 on bad arguments). */
size_t inception_workspace_bytes(const inception_ctx* ctx, int n, int H, int W);
/* feats[n][2048] (fp32, device) = pool3 features of x[n][3][H][W] (fp32 NCHW in [0, 1], device, any H, W >= 1).
 * Asynchronous on `stream`. */
int inception_features(inception_ctx* ctx, const float* x, int n, int H, int W, float* feats, void* workspace,
                       size_t workspace_bytes, void* stream);
int inception_last_launch_count(const inception_ctx* ctx);

/* The forward's launches for n images of H x W, one per line ("<kind> <name> key=value ..."), written to buf (NUL
 * terminated, truncated to cap bytes); returns the full length.  Works on a description-only context. */
int inception_launch_plan(const inception_ctx* ctx, int n, int H, int W, char* buf, int cap);

/* ---- kernels on their own (device pointers, NHWC fp32 unless stated) ----------------------------------------------- */
/* y[n][299][299][4] = 2 * bilinear(x[n][3][H][W] -> 299 x 299, align_corners=False, no antialias) - 1; channel 3 = 0. */
int inception_resize(const float* x, int n, int H, int W, float* y, void* stream);
#define INCEPTION_POOL_MAX_S2 0     /* max 3x3, stride 2, no padding */
#define INCEPTION_POOL_AVG_S1 1     /* average 3x3, stride 1, padding 1, count_include_pad=False */
#define INCEPTION_POOL_MAX_S1 2     /* max 3x3, stride 1, padding 1 */
/* y[n][OH][OW][ct] channels [c0, c0 + C) = pool(x[n][H][W][C]); the other channels are left untouched. */
int inception_pool(int kind, const float* x, int n, int H, int W, int C, float* y, int ct, int c0, void* stream);
/* y[n][OH][OW][ct] channels [c0, c0 + cout) = relu(conv2d(x[n][H][W][cin], w[cout][cin][kh][kw], stride, (ph, pw)) +
 * bias) on the tensor-core kernel (TF32 hi / lo, three passes).  cin a multiple of 4.  The packed operands go to the
 * workspace; workspace == NULL: only report its size in *workspace_needed. */
int inception_conv2d(const float* x, int n, int H, int W, int cin, const float* w, const float* bias, int cout, int kh,
                     int kw, int stride, int ph, int pw, float* y, int ct, int c0, void* workspace, size_t workspace_bytes,
                     size_t* workspace_needed, void* stream);

/* ---- feature statistics --------------------------------------------------------------------------------------------
 * Running float64 sums over feature rows x[n][dim] (fp32, device): shift[dim] (set to the mean of the first batch when
 * first != 0), sum[dim] += sum_i (x_i - shift), sumsq[dim][dim] += sum_i (x_i - shift)(x_i - shift)^T.  Then
 * mean = shift + sum / N and cov = (sumsq - sum sum^T / N) / (N - 1). */
int fid_stats_update(const float* x, int n, int dim, double* shift, double* sum, double* sumsq, int first, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* INCEPTION_B200_H_ */

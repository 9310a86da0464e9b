/* metrics_b200.h -- C ABI of the H100-native SSIM and PSNR evaluators (the reference's lib/evaluator/eva_ssim.py and
 * eva_psnr.py arithmetic).
 *
 * Same shared library and conventions as lpips_b200.h (return 0 / non-zero MIGAN_ERR_* code, fp32 device pointers
 * unless stated, `stream` = cudaStream_t as void*, no CPU fallback); the error message is migan_last_error()'s.  The
 * functions are stateless: there are no weights.  Each call is two launches, a partial-sum kernel and one per-image
 * reduction; an image's value does not depend on n or on its position in the batch.
 */
#ifndef METRICS_B200_H_
#define METRICS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define METRICS_MAX_WINDOW 31

/* ---- SSIM (pytorch-ssim's compute_ssim) ------------------------------------------------------------------------------
 * img1, img2 [n][C][H][W]; taps: `window` host floats, the 1-D Gaussian taps (the 2-D window is their outer product,
 * taken in double); zero padding window / 2, so the map is H' x W' = (H + 2 (window / 2) - window + 1) x (the same in
 * W).  per_image[n] (fp32, device, or NULL): the mean of image i's C x H' x W' map; mean (one fp32, device, or NULL):
 * the mean over the whole [n][C][H'][W'] map.  At least one of the two.  Window sums and the map in double.
 * 1 <= window <= METRICS_MAX_WINDOW.  Asynchronous on `stream`. */
size_t metrics_ssim_workspace_bytes(int n, int C, int H, int W, int window);   /* 0 on bad arguments */
int metrics_ssim(const float* img1, const float* img2, int n, int C, int H, int W, const float* taps, int window,
                 float* per_image, float* mean, void* workspace, size_t workspace_bytes, void* stream);

/* ---- PSNR (psnr_evaluator.add_batch, per image) ----------------------------------------------------------------------
 * pred, gt [n][C][H][W]; diff = (pred - gt) / rgb_range in fp32; `shave` pixels dropped from each side of H and W
 * (0: the whole image); gray != 0 (C == 3): the gray difference sum_c diff_c * coef_c, coef = [65.738, 129.057,
 * 25.064] / 256, in double.  out[n] (double, device) = -10 log10(mean of the squared (gray) differences), +inf for
 * identical images.  The region (H - 2 shave) x (W - 2 shave) must not be empty.  Asynchronous on `stream`. */
size_t metrics_psnr_workspace_bytes(int n, int H, int W, int shave);           /* 0 on bad arguments */
int metrics_psnr(const float* pred, const float* gt, int n, int C, int H, int W, int gray, int shave, float rgb_range,
                 double* out, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* METRICS_B200_H_ */

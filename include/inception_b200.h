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
 *   fid_stats_update_binned            the same sums for up to 32 bins of rows at once (statistics per hole size)
 *   fid_stats_mean_cov                 the mean and covariance from those sums, on the device
 *   fid_frechet_distance               the Fréchet distance of two (mu, sigma) on the device (float64 eigensolver)
 *   ids_scores                         P-IDS and U-IDS of paired real / fake features (float64 finite-Newton SVM)
 *   kid_subset_terms                   the per-subset kernel sums of the kernel Inception distance (float64 DMMA)
 *   prdc_counts                        the counts behind precision, recall, density and coverage (float64 DMMA)
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
/* fid_stats_update for nbins (1..FID_STATS_MAX_BINS) sets of sums at once, all on the device: row r of x[n][dim] goes to
 * bin[r] (int32 [n]; -1, or any value outside [0, nbins): no bin), and bin b holds shift[b][dim], sum[b][dim],
 * sumsq[b][dim][dim] and count[b] (int64).  Bitwise, every bin ends as if fid_stats_update had run on its rows x[bin == b]
 * in row order, with first = (count[b] == 0), for every call that gives it a row; nothing of a bin changes otherwise.
 * No host synchronisation: the bin counts stay on the device. */
#define FID_STATS_MAX_BINS 32
int fid_stats_update_binned(const float* x, const int* bin, int n, int dim, int nbins, double* shift, double* sum,
                            double* sumsq, int64_t* count, void* stream);
/* mu[dim] = shift + sum / count and sigma[dim][dim] = (sumsq - sum sum^T / count) / (count - 1) from the sums above
 * (float64, device), each operation rounded on its own: bitwise what FeatureStatistics.mean_cov() computes on the host.
 * count >= 2.  Asynchronous on `stream`. */
int fid_stats_mean_cov(const double* shift, const double* sum, const double* sumsq, int64_t count, int dim, double* mu,
                       double* sigma, void* stream);

/* ---- Fréchet distance ----------------------------------------------------------------------------------------------
 * FID = ||mu1 - mu2||^2 + tr S1 + tr S2 - 2 tr sqrt(S1 S2) in float64 for covariances S1, S2 [dim][dim] (device,
 * symmetric positive semi-definite; each is symmetrised once as (S + S^T) / 2).  tr sqrt(S1 S2) is the sum of
 * sqrt(max(lambda, 0)) over the eigenvalues of D^1/2 V^T S2 V D^1/2, S1 = V D V^T (negative d clamped to 0): two
 * block-Jacobi eigensolves on the device, no non-symmetric product.  No atomics and fixed-order sums: the same inputs
 * give the same bytes on every run.
 *
 * out_host[4] (HOST) = {||mu1 - mu2||^2, tr S1, tr S2, tr sqrt(S1 S2)}; FID = out[0] + out[1] + out[2] - 2 out[3].
 * sweeps_host (HOST, may be NULL) receives the Jacobi sweeps of the two eigensolves (int[2]).
 * SYNCHRONOUS on `stream`: the solver reads a convergence value back once per sweep, and the call returns with the
 * result on the host.  Refused with MIGAN_ERR_INVALID: dim outside 1..FID_FRECHET_MAX_DIM, null pointers, non-finite
 * input, no convergence within 40 sweeps; with MIGAN_ERR_WORKSPACE: a workspace that is short or not 256-byte aligned. */
#define FID_FRECHET_MAX_DIM 4096
/* Device bytes fid_frechet_distance needs (about 4 N^2 doubles, N = dim rounded up to 64); 0 on bad arguments. */
size_t fid_frechet_workspace_bytes(int dim);
int fid_frechet_distance(const double* mu1, const double* sigma1, const double* mu2, const double* sigma2, int dim,
                         double out_host[4], int* sweeps_host, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Inception discriminative scores (P-IDS, U-IDS) ------------------------------------------------------------------
 * The linear SVM of sklearn.svm.LinearSVC(dual=False) on paired rows real[n][dim] (label +1) and fake[n][dim] (label
 * -1): the minimiser b* = (w, intercept) of f(b) = 1/2 |b|^2 + C sum_i max(0, 1 - y_i b.[x_i, 1])^2 with C = 1 (the
 * intercept regularised as a weight on a constant feature, as liblinear does), found to float64 rounding by the finite
 * Newton method on the device (Gram on fp64 DMMA tiles, blocked Cholesky, exact line search).  With o_i = b*.[x_i, 1]:
 *   U-IDS = (#{real: o <= 0} + #{fake: o > 0}) / 2n      P-IDS = #{i: o_fake,i > o_real,i} / n.
 * The features are read as stored (dtype IDS_FLOAT32 or IDS_FLOAT64, device, row-major) and promoted exactly to float64.
 * No atomics and fixed-order sums: the same inputs give the same bytes on every run and on any stream.
 *
 * coef (device, float64 [dim]) = w.  out_host[5] (HOST) = {P-IDS, U-IDS, intercept, f(b*), |grad f(b*)| / |grad f(0)|}.
 * iterations_host[2] (HOST) = {Newton iterations, the rule that ended the solve: IDS_STOP_ACTIVE_SET (the active set at
 * the Newton point equals the one it was solved on, so it is the minimiser) or IDS_STOP_GRADIENT (relative gradient
 * <= 1e-12)}.  SYNCHRONOUS on `stream`: the host reads a small status back once per Newton iteration.  Refused with
 * MIGAN_ERR_INVALID: null pointers, n < 1, dim outside 1..IDS_MAX_DIM, n x 2 x (dim + 1) >= 2^31, an unknown dtype,
 * non-finite features, a workspace that is short or not 256-byte aligned, no convergence in 100 iterations (the
 * message gives the last active-set change). */
#define IDS_MAX_DIM 4096
#define IDS_FLOAT32 0
#define IDS_FLOAT64 1
#define IDS_STOP_ACTIVE_SET 1
#define IDS_STOP_GRADIENT 2
/* Device bytes ids_scores needs; 0 on bad arguments. */
size_t ids_workspace_bytes(int64_t n, int dim);
int ids_scores(const void* real, const void* fake, int64_t n, int dim, int dtype, double* coef, double out_host[5],
               int iterations_host[2], void* workspace, size_t workspace_bytes, void* stream);

/* ---- Kernel Inception distance (KID) ---------------------------------------------------------------------------------
 * The kernel sums behind the unbiased MMD^2 estimate of Binkowski et al. 2018 under the cubic polynomial kernel
 * k(u, v) = t t t, t = (u.v) / dim + 1, in float64, on num_subsets = S subsets of m rows.  Subset s takes the fake rows
 * fake_idx_host[s][0..m) of fake[n_fake][dim] (X) and the real rows real_idx_host[s][0..m) of real[n_real][dim] (Y):
 *   terms[s][0] = Sxx = sum_{i != j} k(x_i, x_j)   terms[s][1] = Syy = sum_{i != j} k(y_i, y_j)
 *   terms[s][2] = Sxy = sum_{i, j} k(x_i, y_j)
 * and its estimate is ((Sxx + Syy) / (m - 1) - 2 Sxy / m) / m; the caller draws the subsets and finishes the mean.
 * The features are read as stored (dtype IDS_FLOAT32 or IDS_FLOAT64, device, row-major) and promoted exactly to float64;
 * the Gram products run on 64 x 64 fp64 DMMA tiles, the rows gathered through the index tables.  No atomics and sums in
 * an order fixed by the shapes: the same inputs give the same bytes on every run and on any stream.
 *
 * real_idx_host, fake_idx_host: HOST int32 [S][m], checked on the host (each entry in range, the m entries of a subset
 * distinct) and copied into the workspace on `stream`; they may be freed when the call returns.  terms: device float64
 * [S][3].  ASYNCHRONOUS on `stream`: nothing is read back.  Refused with MIGAN_ERR_INVALID: null pointers, S < 1,
 * m < 2, m above n_real or n_fake, n_real or n_fake >= 2^31, dim outside 1..KID_MAX_DIM, an unknown dtype, an index out
 * of range or repeated within a subset, S x m or the tile grid reaching 2^31; with MIGAN_ERR_WORKSPACE: a workspace that
 * is short or not 256-byte aligned.  Non-finite features are not checked here: they make the sums non-finite. */
#define KID_MAX_DIM 4096
/* Device bytes kid_subset_terms needs (the index tables and S x 3 x ceil(m / 64)^2 tile partials); 0 on bad arguments. */
size_t kid_workspace_bytes(int num_subsets, int m);
int kid_subset_terms(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype,
                     const int32_t* real_idx_host, const int32_t* fake_idx_host, int num_subsets, int m, double* terms,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- Precision, recall, density and coverage -------------------------------------------------------------------------
 * The k-nearest-neighbour manifold metrics of Kynkaanniemi et al. 2019 and Naeem et al. 2020 between real[n_real][dim]
 * (Y) and fake[n_fake][dim] (X), on squared Euclidean distances in float64.  r_i is the (k + 1)-th smallest of
 * {|Y_i - Y_j|^2 : j = 1..n_real}, row i itself included (so duplicate rows count as neighbours), s_j the same within X,
 * and every comparison is `<=`:
 *   out_counts[0] = #{j : exists i, |X_j - Y_i|^2 <= r_i}        precision = out_counts[0] / n_fake
 *   out_counts[1] = #{i : exists j, |Y_i - X_j|^2 <= s_j}        recall    = out_counts[1] / n_real
 *   out_counts[2] = sum_j #{i : |X_j - Y_i|^2 <= r_i}            density   = out_counts[2] / (k n_fake)
 *   out_counts[3] = #{i : min_j |Y_i - X_j|^2 <= r_i}            coverage  = out_counts[3] / n_real
 * The features are read as stored (dtype IDS_FLOAT32 or IDS_FLOAT64, device, row-major) and promoted exactly to float64.
 * |a - b|^2 = max(0, |a|^2 + |b|^2 - 2 a.b) with every term from 64 x 64 fp64 DMMA tiles in one column order, so
 * identical rows are at distance exactly 0.  No N x N or N x M matrix is formed: three passes keep per-row lists of the
 * k + 1 smallest values, per-row counters and per-row flags.  The same inputs give the same bytes on every run, on any
 * stream and for any order of the rows.
 *
 * out_counts: device int64 [4].  ASYNCHRONOUS on `stream`: nothing is read back.  Refused with MIGAN_ERR_INVALID: null
 * pointers, k outside 1..PRDC_MAX_K, k + 1 above n_real or n_fake, n_real or n_fake >= 2^31, dim outside
 * 1..PRDC_MAX_DIM, an unknown dtype; with MIGAN_ERR_WORKSPACE: a workspace that is short or not 256-byte aligned.
 * Non-finite features are not checked here.
 *
 * prdc_real_radii computes the real side alone (|Y_i|^2 and r_i) into the start of the workspace, and
 * prdc_counts_with_real_radii then scores a fake set against them without recomputing them: the same counts as
 * prdc_counts, for any number of fake sets against one real set, as long as the workspace is not used for anything
 * else in between and is sized for the largest n_fake.  prdc_counts is the two calls in turn. */
#define PRDC_MAX_DIM 4096
#define PRDC_MAX_K 32
/* Device bytes prdc_counts needs; 0 on bad arguments.  With T(n) = ceil(n / 64), S(n) = min(8, T(n)),
 * L = max(n_real, n_fake) and each region rounded up to 256 bytes: 8 n_real twice (norms, radii), 8 n_fake twice,
 * 2048 (k + 1) T(L) S(L) (the neighbour lists), 256 S(n_real) T(n_fake) (the per-row counters), 4 n_real twice (the
 * flags) and 16 (T(n_real) + T(n_fake)) (the partial totals). */
size_t prdc_workspace_bytes(int64_t n_real, int64_t n_fake, int dim, int k);
int prdc_counts(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype, int k,
                int64_t* out_counts, void* workspace, size_t workspace_bytes, void* stream);
int prdc_real_radii(const void* real, int64_t n_real, int dim, int dtype, int k, void* workspace,
                    size_t workspace_bytes, void* stream);
int prdc_counts_with_real_radii(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype,
                                int k, int64_t* out_counts, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* INCEPTION_B200_H_ */

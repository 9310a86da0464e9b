// C ABI of precision, recall, density and coverage (include/inception_b200.h): prdc_workspace_bytes, prdc_counts,
// prdc_real_radii and prdc_counts_with_real_radii.  Argument checks, workspace layout and the launches; the arithmetic
// is prdc_kernels.cuh's.  The tile kernel runs its phases with a block's threads at once, and the emulation build
// (MIGAN_EMULATE) runs the same phases with the threads of a block in turn.  It is not written over portable.cuh's
// block layer: that way nvcc keeps its tile indices in uniform registers, and its radius passes run 3-5% slower on an
// H100 (80 GB HBM3, 700 W).
//
// Workspace (each region 256-byte aligned), the real side first so that it does not move with n_fake:
//   |Y|^2 and r (n_real doubles each), the coverage and recall flags (n_real ints each), the neighbour lists
//   (T(L) x S(L) x (k + 1) x 256 doubles, L = max(n_real, n_fake), shared by the two radius passes), |X|^2 and s (n_fake
//   doubles each), the per-row counters (S(n_real) x T(n_fake) x 64 ints), the partial totals
//   ((T(n_fake) + T(n_real)) x 2 int64).
#include <string.h>

#include <vector>

#include "../../include/inception_b200.h"
#include "abi_error.h"
#include "prdc_kernels.cuh"

namespace {
using prdc::kG;
using prdc::kThreads;
using prdc::kTileDoubles;
using migan::fail;

static_assert(prdc::kMaxDim == PRDC_MAX_DIM && prdc::kMaxK == PRDC_MAX_K, "one cap");
static_assert(IDS_FLOAT32 == 0 && IDS_FLOAT64 == 1, "the dtype codes of ids_scores");

size_t pass_smem(const prdc::PassArgs& a) { return (2 * (size_t)kTileDoubles + a.extra_doubles()) * sizeof(double); }

#ifdef MIGAN_EMULATE
int pass_launch(const prdc::PassArgs& a, ck_stream_t) {
    const int64_t blocks = a.blocks();
#pragma omp parallel for schedule(dynamic)
    for (int64_t b = 0; b < blocks; ++b) {
        std::vector<double> Xs(kTileDoubles), Ys(kTileDoubles), ex(a.extra_doubles() + 1);
        std::vector<prdc::Acc> c(kThreads);
        for (int t = 0; t < kThreads; ++t) a.begin(t, ex.data());
        for (int jt = a.first(b); jt < a.last(b); ++jt) {
            for (int t = 0; t < kThreads; ++t) frechet::acc_zero(c[t]);
            for (int k0 = 0; k0 < a.A.d; k0 += kG) {
                for (int t = 0; t < kThreads; ++t) a.stage(b, jt, t, k0, Xs.data(), Ys.data());
                for (int t = 0; t < kThreads; ++t) a.product(t, c[t], Xs.data(), Ys.data());
            }
            for (int t = 0; t < kThreads; ++t) a.epilogue(b, jt, t, c[t], ex.data());
            for (int t = 0; t < kThreads; ++t) a.flush(jt, t, ex.data());
        }
        for (int t = 0; t < kThreads; ++t) a.end(b, t, ex.data());
    }
    return 0;
}
#else
__global__ void __launch_bounds__(kThreads) prdc_pass_kernel(const __grid_constant__ prdc::PassArgs a) {
    extern __shared__ __align__(16) double smem[];
    double* Xs = smem;
    double* Ys = Xs + kTileDoubles;
    double* ex = Ys + kTileDoubles;
    const int64_t b = blockIdx.x;
    const int t = threadIdx.x;
    a.begin(t, ex);
    for (int jt = a.first(b); jt < a.last(b); ++jt) {
        prdc::Acc c;
        frechet::acc_zero(c);
        for (int k0 = 0; k0 < a.A.d; k0 += kG) {
            a.stage(b, jt, t, k0, Xs, Ys);
            __syncthreads();
            a.product(t, c, Xs, Ys);
            __syncthreads();
        }
        a.epilogue(b, jt, t, c, ex);
        __syncthreads();
        a.flush(jt, t, ex);   // the next tile's panel barriers order its zeroing before the next epilogue
    }
    __syncthreads();
    a.end(b, t, ex);
}

int pass_launch(const prdc::PassArgs& a, ck_stream_t s) {
    const size_t smem = pass_smem(a);
    if (int e = set_smem(prdc_pass_kernel, smem)) return e;
    prdc_pass_kernel<<<(unsigned)a.blocks(), kThreads, smem, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

struct Layout {
    size_t norm_y, r_y, cov, rec, lists, real_total, norm_x, r_x, counts, part, total;
};

Layout layout(int64_t N, int64_t M, int k) {
    const int64_t L = N > M ? N : M;
    const size_t tl = (size_t)prdc::tiles_of(L), tm = (size_t)prdc::tiles_of(M), tn = (size_t)prdc::tiles_of(N);
    Layout W;
    W.norm_y = 0;
    W.r_y = W.norm_y + align256((size_t)N * sizeof(double));
    W.cov = W.r_y + align256((size_t)N * sizeof(double));
    W.rec = W.cov + align256((size_t)N * sizeof(int));
    W.lists = W.rec + align256((size_t)N * sizeof(int));
    // what prdc_real_radii uses: the lists of the real pass alone
    W.real_total = W.lists + align256(tn * prdc::splits_of((int)tn) * (k + 1) * kThreads * sizeof(double));
    W.norm_x = W.lists + align256(tl * prdc::splits_of((int)tl) * (k + 1) * kThreads * sizeof(double));
    W.r_x = W.norm_x + align256((size_t)M * sizeof(double));
    W.counts = W.r_x + align256((size_t)M * sizeof(double));
    W.part = W.counts + align256((size_t)prdc::splits_of((int)tn) * tm * kG * sizeof(int));
    W.total = W.part + align256((tm + tn) * 2 * sizeof(int64_t));
    return W;
}

bool big(int64_t n) { return n >= ((int64_t)1 << 31); }

// The checks shared by the entry points; n_fake < 0 for prdc_real_radii, which has no fake side.
int check_args(const char* fn, const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype,
               int k, const void* out, const void* workspace) {
    if (!real || (n_fake >= 0 && (!fake || !out)) || !workspace)
        return fail(MIGAN_ERR_INVALID, "%s: null real / fake / out_counts / workspace", fn);
    if (k < 1 || k > prdc::kMaxK) return fail(MIGAN_ERR_INVALID, "%s: k %d outside 1..%d", fn, k, prdc::kMaxK);
    if (big(n_real) || big(n_fake))
        return fail(MIGAN_ERR_INVALID, "%s: %lld real / %lld fake rows reach 2^31", fn, (long long)n_real,
                    (long long)n_fake);
    if (k + 1 > n_real || (n_fake >= 0 && k + 1 > n_fake))
        return fail(MIGAN_ERR_INVALID, "%s: k + 1 = %d neighbours from %lld real and %lld fake rows", fn, k + 1,
                    (long long)n_real, (long long)n_fake);
    if (dim < 1 || dim > prdc::kMaxDim)
        return fail(MIGAN_ERR_INVALID, "%s: dim %d outside 1..%d", fn, dim, prdc::kMaxDim);
    if (dtype != IDS_FLOAT32 && dtype != IDS_FLOAT64)
        return fail(MIGAN_ERR_INVALID, "%s: dtype %d is neither IDS_FLOAT32 nor IDS_FLOAT64", fn, dtype);
    if (reinterpret_cast<uintptr_t>(workspace) % 256)
        return fail(MIGAN_ERR_WORKSPACE, "%s: workspace not 256-byte aligned", fn);
    return MIGAN_OK;
}

int short_workspace(const char* fn, size_t have, size_t need) {
    return fail(MIGAN_ERR_WORKSPACE, "%s: workspace of %zu bytes, %zu needed", fn, have, need);
}

prdc::PassArgs pass(prdc::Rows A, prdc::Rows B, int64_t nA, int64_t nB, int mode, int k) {
    prdc::PassArgs a;
    memset(&a, 0, sizeof(a));
    a.A = A;
    a.B = B;
    a.nA = (int)nA;
    a.nB = (int)nB;
    a.mode = mode;
    a.K1 = k + 1;
    return a;
}

// |rows|^2 into norms, then the (k + 1)-th smallest distance of each row within its set into r.
int radii(prdc::Rows rows, int64_t n, int k, double* norms, double* r, double* lists, ck_stream_t s) {
    prdc::PassArgs a = pass(rows, rows, n, n, prdc::kNorms, k);
    a.norms = norms;
    if (int e = pass_launch(a, s)) return e;
    a = pass(rows, rows, n, n, prdc::kRadii, k);
    a.normA = a.normB = norms;
    a.lists = lists;
    if (int e = pass_launch(a, s)) return e;
    return (int)comod::ck_launch(prdc::RadiusK{lists, r, k + 1, a.splits()}, n, s);
}

int real_side(const void* real, int64_t n_real, int dim, int dtype, int k, char* ws, const Layout& W, ck_stream_t s) {
    const prdc::Rows Y{real, dim, dtype == IDS_FLOAT64};
    return radii(Y, n_real, k, reinterpret_cast<double*>(ws + W.norm_y), reinterpret_cast<double*>(ws + W.r_y),
                 reinterpret_cast<double*>(ws + W.lists), s);
}

int fake_side(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype, int k,
              int64_t* out, char* ws, const Layout& W, ck_stream_t s) {
    const int fp64 = dtype == IDS_FLOAT64;
    const prdc::Rows X{fake, dim, fp64}, Y{real, dim, fp64};
    double* norm_x = reinterpret_cast<double*>(ws + W.norm_x);
    double* r_x = reinterpret_cast<double*>(ws + W.r_x);
    int* cov = reinterpret_cast<int*>(ws + W.cov);
    int* rec = reinterpret_cast<int*>(ws + W.rec);
    int* counts = reinterpret_cast<int*>(ws + W.counts);
    int64_t* part = reinterpret_cast<int64_t*>(ws + W.part);
    CUDA_TRY(radii(X, n_fake, k, norm_x, r_x, reinterpret_cast<double*>(ws + W.lists), s));
    CUDA_TRY(comod::ck_launch(prdc::ZeroK{cov, rec}, n_real, s));
    prdc::PassArgs a = pass(X, Y, n_fake, n_real, prdc::kCross, k);
    a.normA = norm_x;
    a.normB = reinterpret_cast<const double*>(ws + W.norm_y);
    a.rA = r_x;
    a.rB = reinterpret_cast<const double*>(ws + W.r_y);
    a.counts = counts;
    a.cov = cov;
    a.rec = rec;
    CUDA_TRY(pass_launch(a, s));
    const int64_t items = prdc::tiles_of(n_fake) + prdc::tiles_of(n_real);
    CUDA_TRY(comod::ck_launch(prdc::TotalsPartK{counts, cov, rec, part, (int)n_fake, (int)n_real, a.splits()}, items,
                              s));
    CUDA_TRY(comod::ck_launch(prdc::TotalsK{part, out, (int)n_fake, (int)n_real}, 1, s));
    return 0;
}

}  // namespace

extern "C" {

size_t prdc_workspace_bytes(int64_t n_real, int64_t n_fake, int dim, int k) {
    if (k < 1 || k > prdc::kMaxK || dim < 1 || dim > prdc::kMaxDim || big(n_real) || big(n_fake) || k + 1 > n_real ||
        k + 1 > n_fake)
        return 0;
    return layout(n_real, n_fake, k).total;
}

int prdc_real_radii(const void* real, int64_t n_real, int dim, int dtype, int k, void* workspace,
                    size_t workspace_bytes, void* stream) {
    const char* fn = "prdc_real_radii";
    if (int rc = check_args(fn, real, n_real, nullptr, -1, dim, dtype, k, nullptr, workspace)) return rc;
    const Layout W = layout(n_real, 0, k);
    if (workspace_bytes < W.real_total) return short_workspace(fn, workspace_bytes, W.real_total);
    CUDA_TRY(real_side(real, n_real, dim, dtype, k, static_cast<char*>(workspace), W,
                       static_cast<ck_stream_t>(stream)));
    return 0;
}

int prdc_counts_with_real_radii(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype,
                                int k, int64_t* out_counts, void* workspace, size_t workspace_bytes, void* stream) {
    const char* fn = "prdc_counts_with_real_radii";
    if (int rc = check_args(fn, real, n_real, fake, n_fake, dim, dtype, k, out_counts, workspace)) return rc;
    const Layout W = layout(n_real, n_fake, k);
    if (workspace_bytes < W.total) return short_workspace(fn, workspace_bytes, W.total);
    CUDA_TRY(fake_side(real, n_real, fake, n_fake, dim, dtype, k, out_counts, static_cast<char*>(workspace), W,
                       static_cast<ck_stream_t>(stream)));
    return 0;
}

int prdc_counts(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype, int k,
                int64_t* out_counts, void* workspace, size_t workspace_bytes, void* stream) {
    const char* fn = "prdc_counts";
    if (int rc = check_args(fn, real, n_real, fake, n_fake, dim, dtype, k, out_counts, workspace)) return rc;
    const Layout W = layout(n_real, n_fake, k);
    if (workspace_bytes < W.total) return short_workspace(fn, workspace_bytes, W.total);
    char* ws = static_cast<char*>(workspace);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    CUDA_TRY(real_side(real, n_real, dim, dtype, k, ws, W, s));
    CUDA_TRY(fake_side(real, n_real, fake, n_fake, dim, dtype, k, out_counts, ws, W, s));
    return 0;
}

}  // extern "C"

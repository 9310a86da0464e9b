// C ABI of the Fréchet distance (include/inception_b200.h): fid_stats_mean_cov, fid_frechet_workspace_bytes and
// fid_frechet_distance.  Argument checks, workspace layout, the eigensolver's sweep loop and the launches; the
// arithmetic is frechet_kernels.cuh's.  Each block kernel is one body over portable.cuh's block layer: the kernel runs
// it with a block's threads at once, and the emulation build (MIGAN_EMULATE) runs the same body on the host.
//
// Workspace (N = dim rounded up to a multiple of 64, each region 256-byte aligned): A, V, B, W (N x N doubles each),
// the pair factors (N / 64 of 64 x 64), sqrt(d) (N), the column partials of the norm (2N), 8 scalars.
#include <math.h>
#include <string.h>

#include "../../include/inception_b200.h"
#include "abi_error.h"
#include "frechet_kernels.cuh"

namespace {
using frechet::kG;
using frechet::kLd;
using frechet::kThreads;
using frechet::kTileDoubles;
using migan::fail;

constexpr int kMaxSweeps = 40;
static_assert(frechet::kMaxDim == FID_FRECHET_MAX_DIM, "one cap");
constexpr size_t kPairSmem = (2 * kTileDoubles + 4 * frechet::kB) * sizeof(double);
constexpr size_t kUpdateSmem = 3 * kTileDoubles * sizeof(double);
constexpr size_t kGemmSmem = 2 * kTileDoubles * sizeof(double);

// Block k of the pair kernel: the subproblem of block pair k, rotated until an inner step rotates nothing.
template <class B>
CK_D void pair_block(const B& blk, const frechet::PairArgs& a, int k, double* smem) {
    double* S = smem;
    double* J = S + kTileDoubles;
    double* cs = J + kTileDoubles;
    blk.each([&](int t) { a.load(k, t, S, J); });
    blk.sync();
    for (int sweep = 0; sweep < frechet::kMaxInner; ++sweep) {
        int rotated = 0;
        for (int step = 0; step < kG - 1; ++step) {
            if (!blk.any([&](int t) { return t < frechet::kB ? a.rot(step, t, S, cs) : 0; })) continue;
            blk.each([&](int t) { a.apply(step, t, S, J, cs); });
            rotated = 1;
            blk.sync();
        }
        if (!rotated) break;
    }
    blk.each([&](int t) { a.store(k, t, S, J); });
}

template <class B>
CK_D void update_block(const B& blk, const frechet::UpdateArgs& a, int64_t b, double* smem) {
    double* X = smem;
    double* P = X + kTileDoubles;
    double* R = P + kTileDoubles;
    blk.each([&](int t) { a.load(b, t, X, P, R); });
    blk.sync();
    frechet::Accs<B> c;
    blk.each([&](int t) { a.right(t, c[t], X, P); });
    blk.sync();
    blk.each([&](int t) { a.after_right(b, t, c[t], X); });
    if (b >= a.tilesA) return;
    blk.sync();
    blk.each([&](int t) { a.left(b, t, c[t], X, R); });
}

template <class B>
CK_D void gemm_block(const B& blk, const frechet::GemmArgs& a, int64_t b, double* smem) {
    double* Xs = smem;
    double* Ys = Xs + kTileDoubles;
    frechet::Accs<B> c;
    frechet::panel_product(blk, c, a.N, Xs, Ys, a, b);
    blk.each([&](int t) { a.store(b, t, c[t]); });
}

int64_t gemm_blocks(const frechet::GemmArgs& a) { return (int64_t)(a.N / kG) * (a.N / kG); }

#ifdef MIGAN_EMULATE
int pair_launch(const frechet::PairArgs& a, int blocks, ck_stream_t) {
    return ck_blocks<kThreads>(blocks, kPairSmem,
                               [&](auto& blk, int64_t k, void* smem) { pair_block(blk, a, (int)k, (double*)smem); });
}

int update_launch(const frechet::UpdateArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(a.blocks(), kUpdateSmem,
                               [&](auto& blk, int64_t b, void* smem) { update_block(blk, a, b, (double*)smem); });
}

int gemm_launch(const frechet::GemmArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(gemm_blocks(a), kGemmSmem,
                               [&](auto& blk, int64_t b, void* smem) { gemm_block(blk, a, b, (double*)smem); });
}
#else
__global__ void __launch_bounds__(kThreads) frechet_pair_kernel(const __grid_constant__ frechet::PairArgs a) {
    extern __shared__ __align__(16) double smem[];
    pair_block(DeviceBlock(), a, blockIdx.x, smem);
}

__global__ void __launch_bounds__(kThreads) frechet_update_kernel(const __grid_constant__ frechet::UpdateArgs a) {
    extern __shared__ __align__(16) double smem[];
    update_block(DeviceBlock(), a, blockIdx.x, smem);
}

__global__ void __launch_bounds__(kThreads) frechet_gemm_kernel(const __grid_constant__ frechet::GemmArgs a) {
    extern __shared__ __align__(16) double smem[];
    gemm_block(DeviceBlock(), a, blockIdx.x, smem);
}

int pair_launch(const frechet::PairArgs& a, int blocks, ck_stream_t s) {
    if (int e = set_smem(frechet_pair_kernel, kPairSmem)) return e;
    frechet_pair_kernel<<<blocks, kThreads, kPairSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int update_launch(const frechet::UpdateArgs& a, ck_stream_t s) {
    if (int e = set_smem(frechet_update_kernel, kUpdateSmem)) return e;
    frechet_update_kernel<<<(unsigned)a.blocks(), kThreads, kUpdateSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int gemm_launch(const frechet::GemmArgs& a, ck_stream_t s) {
    if (int e = set_smem(frechet_gemm_kernel, kGemmSmem)) return e;
    frechet_gemm_kernel<<<(unsigned)gemm_blocks(a), kThreads, kGemmSmem, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

int padded(int dim) { return (dim + kG - 1) / kG * kG; }

struct Layout {
    size_t A, V, B, W, J, sd, part, scal, total;
};

Layout layout(int dim) {
    const size_t N = (size_t)padded(dim), mat = align256(N * N * sizeof(double));
    Layout L;
    L.A = 0;
    L.V = L.A + mat;
    L.B = L.V + mat;
    L.W = L.B + mat;
    L.J = L.W + mat;
    L.sd = L.J + align256(N / kG * kG * kG * sizeof(double));
    L.part = L.sd + align256(N * sizeof(double));
    L.scal = L.part + align256(2 * N * sizeof(double));
    L.total = L.scal + align256(8 * sizeof(double));
    return L;
}

int check_dim(const char* who, int dim) {
    if (dim < 1 || dim > frechet::kMaxDim)
        return fail(MIGAN_ERR_INVALID, "%s: dim %d outside 1..%d", who, dim, frechet::kMaxDim);
    return 0;
}

// Block-Jacobi sweeps on A (and V when given) until off(A) <= dim 2^-53 ||A||_F; the sweeps taken in *sweeps.
int solve(double* A, double* V, double* J, double* part, double* scal, int dim, int N, int* sweeps, ck_stream_t s) {
    const int nb = N / frechet::kB, groups = nb / 2;
    const double tol = (double)dim * frechet::kEps;
    for (int sweep = 0;; ++sweep) {
        CUDA_TRY(comod::ck_launch(frechet::ColNormK{A, part, N}, N, s));
        CUDA_TRY(comod::ck_launch(frechet::NormSumK{part, scal, N}, 1, s));
        double norm[2];
        CUDA_TRY(to_host(norm, scal, sizeof(norm), s));
        if (!isfinite(norm[1])) return fail(MIGAN_ERR_INVALID, "frechet: the covariances are not finite");
        if (norm[0] <= tol * tol * norm[1]) {
            *sweeps = sweep;
            return 0;
        }
        if (sweep == kMaxSweeps)
            return fail(MIGAN_ERR_INVALID, "frechet: the eigensolver did not converge in %d sweeps (off/norm %.3g)",
                        kMaxSweeps, sqrt(norm[0] / norm[1]));
        for (int r = 0; r < nb - 1; ++r) {
            CUDA_TRY(pair_launch(frechet::PairArgs{A, J, N, nb, r}, groups, s));
            CUDA_TRY(update_launch(frechet::UpdateArgs{A, V, J, N, nb, r, groups * (groups + 1) / 2}, s));
        }
    }
}

}  // namespace

extern "C" {

int fid_stats_mean_cov(const double* shift, const double* sum, const double* sumsq, int64_t count, int dim, double* mu,
                       double* sigma, void* stream) {
    if (!shift || !sum || !sumsq || !mu || !sigma) return fail(MIGAN_ERR_INVALID, "fid_stats_mean_cov: null argument");
    if (dim < 1 || dim > 65536) return fail(MIGAN_ERR_INVALID, "fid_stats_mean_cov: dim %d outside 1..65536", dim);
    if (count < 2) return fail(MIGAN_ERR_INVALID, "fid_stats_mean_cov: needs at least 2 rows, has %lld", (long long)count);
    CUDA_TRY(comod::ck_launch(frechet::MeanCovK{shift, sum, sumsq, mu, sigma, dim, (double)count}, (int64_t)dim * dim,
                              static_cast<ck_stream_t>(stream)));
    return 0;
}

size_t fid_frechet_workspace_bytes(int dim) {
    if (dim < 1 || dim > frechet::kMaxDim) return 0;
    return layout(dim).total;
}

int fid_frechet_distance(const double* mu1, const double* sigma1, const double* mu2, const double* sigma2, int dim,
                         double out[4], int* sweeps, void* workspace, size_t workspace_bytes, void* stream) {
    if (!mu1 || !sigma1 || !mu2 || !sigma2 || !out)
        return fail(MIGAN_ERR_INVALID, "fid_frechet_distance: null mu1 / sigma1 / mu2 / sigma2 / out");
    if (int rc = check_dim("fid_frechet_distance", dim)) return rc;
    const Layout L = layout(dim);
    if (!workspace) return fail(MIGAN_ERR_INVALID, "fid_frechet_distance: null workspace");
    if (reinterpret_cast<uintptr_t>(workspace) % 256)
        return fail(MIGAN_ERR_WORKSPACE, "fid_frechet_distance: workspace not 256-byte aligned");
    if (workspace_bytes < L.total)
        return fail(MIGAN_ERR_WORKSPACE, "fid_frechet_distance: workspace of %zu bytes, %zu needed", workspace_bytes,
                    L.total);
    char* ws = static_cast<char*>(workspace);
    double* A = reinterpret_cast<double*>(ws + L.A);
    double* V = reinterpret_cast<double*>(ws + L.V);
    double* B = reinterpret_cast<double*>(ws + L.B);
    double* W = reinterpret_cast<double*>(ws + L.W);
    double* J = reinterpret_cast<double*>(ws + L.J);
    double* sd = reinterpret_cast<double*>(ws + L.sd);
    double* part = reinterpret_cast<double*>(ws + L.part);
    double* scal = reinterpret_cast<double*>(ws + L.scal);
    const int N = padded(dim);
    const int64_t NN = (int64_t)N * N;
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    int sw[2] = {0, 0};

    // S1 = V D V^T
    CUDA_TRY(comod::ck_launch(frechet::LoadK{sigma1, A, V, dim, N}, NN, s));
    CUDA_TRY(comod::ck_launch(frechet::LoadK{sigma2, B, nullptr, dim, N}, NN, s));
    if (int rc = solve(A, V, J, part, scal, dim, N, &sw[0], s)) return rc;
    // M = D^1/2 (V^T S2 V) D^1/2, then its eigenvalues
    CUDA_TRY(comod::ck_launch(frechet::CutoffK{A, scal + 4, dim, N}, 1, s));
    CUDA_TRY(comod::ck_launch(frechet::SqrtDiagK{A, scal + 4, sd, N}, N, s));
    CUDA_TRY(gemm_launch(frechet::GemmArgs{B, V, W, N}, s));   // W = S2^T V = S2 V
    CUDA_TRY(gemm_launch(frechet::GemmArgs{V, W, B, N}, s));   // B = V^T S2 V
    CUDA_TRY(comod::ck_launch(frechet::ScaleK{B, sd, A, N}, NN, s));
    if (int rc = solve(A, nullptr, J, part, scal, dim, N, &sw[1], s)) return rc;
    CUDA_TRY(comod::ck_launch(frechet::ResultK{mu1, sigma1, mu2, sigma2, A, scal, dim, N}, 1, s));
    CUDA_TRY(to_host(out, scal, 4 * sizeof(double), s));
    if (sweeps) {
        sweeps[0] = sw[0];
        sweeps[1] = sw[1];
    }
    return 0;
}

}  // extern "C"

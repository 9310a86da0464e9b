// C ABI of the Inception discriminative scores (include/inception_b200.h): ids_workspace_bytes and ids_scores.
// Argument checks, workspace layout, the finite Newton loop and the launches; the arithmetic is ids_kernels.cuh's.  Each
// block kernel is one body over portable.cuh's block layer, run with a block's threads at once on the device and on the
// host in the emulation build (MIGAN_EMULATE).
//
// Workspace (M = 2n rows, Dp = dim + 1 rounded up to 64, H = chunks of 256 rows; each region 256-byte aligned):
// b, b~, g, r (Dp each), o, ob (M), the active list (M ints), the chunk partials (3H) and offsets (H ints), the margin
// lane partials (32 M), the gradient's column partials (2 H Dp), G (Dp x Dp), 16 status scalars.
#include <math.h>
#include <string.h>

#include "../../include/inception_b200.h"
#include "abi_error.h"
#include "ids_kernels.cuh"

namespace {
using ids::kG;
using ids::kLd;
using ids::kThreads;
using ids::kTileDoubles;
using migan::fail;

constexpr int kMaxIter = 100;
constexpr double kGradTol = 1e-12;
static_assert(ids::kMaxDim == IDS_MAX_DIM, "one cap");
constexpr size_t kTileSmem = 2 * kTileDoubles * sizeof(double);
constexpr size_t kDiagSmem = kTileDoubles * sizeof(double);
constexpr size_t kLineSmem = 3 * kThreads * sizeof(double);

template <class B>
CK_D void gram_block(const B& blk, const ids::GramArgs& a, int64_t b, double* smem) {
    double* Xs = smem;
    double* Ys = Xs + kTileDoubles;
    ids::Accs<B> c;
    frechet::panel_product(blk, c, a.count(), Xs, Ys, a, b);
    blk.each([&](int t) { a.store(b, t, c[t]); });
}

template <class B>
CK_D void diag_block(const B& blk, const ids::CholArgs& a, double* S) {
    blk.each([&](int t) { a.diag_load(t, S); });
    blk.sync();
    for (int j = 0; j < kG; ++j) {
        blk.each([&](int t) { a.diag_scale(j, t, S); });
        blk.sync();
        blk.each([&](int t) { a.diag_update(j, t, S); });
        blk.sync();
    }
    blk.each([&](int t) { a.diag_store(t, S); });
}

template <class B>
CK_D void panel_block(const B& blk, const ids::CholArgs& a, int b, double* smem) {
    double* L = smem;
    double* P = L + kTileDoubles;
    blk.each([&](int t) { a.panel_load(b, t, L, P); });
    blk.sync();
    blk.each([&](int t) { a.panel_solve(t, L, P); });
    blk.sync();
    blk.each([&](int t) { a.panel_store(b, t, P); });
}

template <class B>
CK_D void trail_block(const B& blk, const ids::CholArgs& a, int64_t b, double* smem) {
    double* Xs = smem;
    double* Ys = Xs + kTileDoubles;
    blk.each([&](int t) { a.trail_stage(b, t, Xs, Ys); });
    blk.sync();
    ids::Accs<B> c;
    blk.each([&](int t) {
        a.trail_product(b, t, c[t], Xs, Ys);
        a.trail_store(b, t, c[t]);
    });
}

template <class B>
CK_D void solve_block(const B& blk, const ids::SolveArgs& a, double* smem) {
    double* z = smem;
    double* w = z + a.Dp;
    blk.each([&](int t) { a.load(t, z); });
    blk.sync();
    for (int j = 0; j < a.Dp; ++j) {
        blk.each([&](int t) { a.forward(j, t, z, w); });
        blk.sync();
    }
    for (int j = a.Dp - 1; j >= 0; --j) {
        blk.each([&](int t) { a.backward(j, t, w); });
        blk.sync();
    }
}

template <class B>
CK_D void line_block(const B& blk, const ids::LineArgs& a, double* part) {
    if (a.scal[ids::kMismatch] == 0.0) {
        blk.each([&](int t) {
            if (t == 0) a.scal[ids::kStep] = 1.0;
        });
        return;
    }
    double s[3];
    blk.each([&](int t) { a.dir_part(t, part); });
    blk.sync();
    ids::sum_parts(part, s);
    blk.sync();
    ids::LineSearch ls;
    ls.start(s);
    for (;;) {
        blk.each([&](int t) { a.row_part(t, ls.eval_lo(), ls.hi, ls.mid(), part); });
        blk.sync();
        ids::sum_parts(part, s);
        blk.sync();
        if (ls.next(s)) break;   // every thread takes the same decision from the same sums
    }
    blk.each([&](int t) {
        if (t == 0) a.scal[ids::kStep] = ls.t;
    });
}

size_t solve_smem(const ids::SolveArgs& a) { return 2 * (size_t)a.Dp * sizeof(double); }

#ifdef MIGAN_EMULATE
int gram_launch(const ids::GramArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(a.tiles(), kTileSmem,
                               [&](auto& blk, int64_t b, void* smem) { gram_block(blk, a, b, (double*)smem); });
}

int diag_launch(const ids::CholArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(1, kDiagSmem, [&](auto& blk, int64_t, void* smem) { diag_block(blk, a, (double*)smem); });
}

int panel_launch(const ids::CholArgs& a, int blocks, ck_stream_t) {
    return ck_blocks<kThreads>(blocks, kTileSmem,
                               [&](auto& blk, int64_t b, void* smem) { panel_block(blk, a, (int)b, (double*)smem); });
}

int trail_launch(const ids::CholArgs& a, int64_t blocks, ck_stream_t) {
    return ck_blocks<kThreads>(blocks, kTileSmem,
                               [&](auto& blk, int64_t b, void* smem) { trail_block(blk, a, b, (double*)smem); });
}

int solve_launch(const ids::SolveArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(1, solve_smem(a),
                               [&](auto& blk, int64_t, void* smem) { solve_block(blk, a, (double*)smem); });
}

int line_launch(const ids::LineArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(1, kLineSmem, [&](auto& blk, int64_t, void* smem) { line_block(blk, a, (double*)smem); });
}
#else
__global__ void __launch_bounds__(kThreads) ids_gram_kernel(const __grid_constant__ ids::GramArgs a) {
    extern __shared__ __align__(16) double smem[];
    gram_block(DeviceBlock(), a, blockIdx.x, smem);
}

__global__ void __launch_bounds__(kThreads) ids_diag_kernel(const __grid_constant__ ids::CholArgs a) {
    extern __shared__ __align__(16) double smem[];
    diag_block(DeviceBlock(), a, smem);
}

__global__ void __launch_bounds__(kThreads) ids_panel_kernel(const __grid_constant__ ids::CholArgs a) {
    extern __shared__ __align__(16) double smem[];
    panel_block(DeviceBlock(), a, blockIdx.x, smem);
}

__global__ void __launch_bounds__(kThreads) ids_trail_kernel(const __grid_constant__ ids::CholArgs a) {
    extern __shared__ __align__(16) double smem[];
    trail_block(DeviceBlock(), a, blockIdx.x, smem);
}

__global__ void __launch_bounds__(kThreads) ids_solve_kernel(const __grid_constant__ ids::SolveArgs a) {
    extern __shared__ __align__(16) double smem[];
    solve_block(DeviceBlock(), a, smem);
}

__global__ void __launch_bounds__(kThreads) ids_line_kernel(const __grid_constant__ ids::LineArgs a) {
    extern __shared__ __align__(16) double smem[];
    line_block(DeviceBlock(), a, smem);
}

int gram_launch(const ids::GramArgs& a, ck_stream_t s) {
    if (int e = set_smem(ids_gram_kernel, kTileSmem)) return e;
    ids_gram_kernel<<<(unsigned)a.tiles(), kThreads, kTileSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int diag_launch(const ids::CholArgs& a, ck_stream_t s) {
    ids_diag_kernel<<<1, kThreads, kDiagSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int panel_launch(const ids::CholArgs& a, int blocks, ck_stream_t s) {
    if (int e = set_smem(ids_panel_kernel, kTileSmem)) return e;
    ids_panel_kernel<<<blocks, kThreads, kTileSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int trail_launch(const ids::CholArgs& a, int64_t blocks, ck_stream_t s) {
    if (int e = set_smem(ids_trail_kernel, kTileSmem)) return e;
    ids_trail_kernel<<<(unsigned)blocks, kThreads, kTileSmem, s>>>(a);
    return (int)cudaGetLastError();
}

int solve_launch(const ids::SolveArgs& a, ck_stream_t s) {
    const size_t bytes = solve_smem(a);
    if (int e = set_smem(ids_solve_kernel, bytes)) return e;
    ids_solve_kernel<<<1, kThreads, bytes, s>>>(a);
    return (int)cudaGetLastError();
}

int line_launch(const ids::LineArgs& a, ck_stream_t s) {
    ids_line_kernel<<<1, kThreads, kLineSmem, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

int padded(int dim) { return (dim + 1 + kG - 1) / kG * kG; }

struct Layout {
    size_t beta, bbar, g, r, o, ob, idx, part, off, lanes, ps, pt, G, scal, total;
};

Layout layout(int64_t n, int dim) {
    const size_t Dp = (size_t)padded(dim), M = 2 * (size_t)n, H = (size_t)ids::chunks_of((int64_t)M);
    const size_t vec = align256(Dp * sizeof(double)), rows = align256(M * sizeof(double));
    Layout L;
    L.beta = 0;
    L.bbar = L.beta + vec;
    L.g = L.bbar + vec;
    L.r = L.g + vec;
    L.o = L.r + vec;
    L.ob = L.o + rows;
    L.idx = L.ob + rows;
    L.part = L.idx + align256(M * sizeof(int));
    L.off = L.part + align256(3 * H * sizeof(double));
    L.lanes = L.off + align256(H * sizeof(int));
    L.ps = L.lanes + align256(M * ids::kLanes * sizeof(double));
    L.pt = L.ps + align256(H * Dp * sizeof(double));
    L.G = L.pt + align256(H * Dp * sizeof(double));
    L.scal = L.G + align256(Dp * Dp * sizeof(double));
    L.total = L.scal + align256(ids::kSlots * sizeof(double));
    return L;
}

bool bad_shape(int64_t n, int dim) {
    return n < 1 || dim < 1 || dim > ids::kMaxDim || n * 2 * (int64_t)(dim + 1) >= ((int64_t)1 << 31);
}

// o = X~ b.
int margins(const ids::Data& X, const double* beta, double* lanes, double* o, ck_stream_t s) {
    CUDA_TRY(comod::ck_launch(ids::MarginPartK{X, beta, lanes}, X.rows() * ids::kLanes, s));
    CUDA_TRY(comod::ck_launch(ids::MarginK{lanes, beta, o, X.d}, X.rows(), s));
    return 0;
}

// b~ = G^-1 r: the Gram's lower tiles, the blocked Cholesky factorisation in place, the two substitutions.
int newton(const ids::Data& X, const int* idx, const double* scal, double* G, const double* r, double* bbar, int Dp,
           ck_stream_t s) {
    CUDA_TRY(gram_launch(ids::GramArgs{X, idx, scal, Dp, G}, s));
    const int nb = Dp / kG;
    for (int p = 0; p < nb; ++p) {
        const ids::CholArgs a{G, Dp, p};
        CUDA_TRY(diag_launch(a, s));
        const int m = nb - p - 1;
        if (m == 0) break;
        CUDA_TRY(panel_launch(a, m, s));
        CUDA_TRY(trail_launch(a, (int64_t)m * (m + 1) / 2, s));
    }
    CUDA_TRY(solve_launch(ids::SolveArgs{G, r, bbar, Dp}, s));
    return 0;
}

}  // namespace

extern "C" {

size_t ids_workspace_bytes(int64_t n, int dim) {
    if (bad_shape(n, dim)) return 0;
    return layout(n, dim).total;
}

int ids_scores(const void* real, const void* fake, int64_t n, int dim, int dtype, double* coef, double out[5],
               int iterations[2], void* workspace, size_t workspace_bytes, void* stream) {
    if (!real || !fake || !coef || !out || !iterations)
        return fail(MIGAN_ERR_INVALID, "ids_scores: null real / fake / coef / out / iterations");
    if (n < 1) return fail(MIGAN_ERR_INVALID, "ids_scores: n %lld < 1", (long long)n);
    if (dim < 1 || dim > ids::kMaxDim)
        return fail(MIGAN_ERR_INVALID, "ids_scores: dim %d outside 1..%d", dim, ids::kMaxDim);
    if (bad_shape(n, dim))
        return fail(MIGAN_ERR_INVALID, "ids_scores: n %lld x 2 x (dim + 1) reaches 2^31", (long long)n);
    if (dtype != IDS_FLOAT32 && dtype != IDS_FLOAT64)
        return fail(MIGAN_ERR_INVALID, "ids_scores: dtype %d is neither IDS_FLOAT32 nor IDS_FLOAT64", dtype);
    if (!workspace) return fail(MIGAN_ERR_INVALID, "ids_scores: null workspace");
    if (reinterpret_cast<uintptr_t>(workspace) % 256)
        return fail(MIGAN_ERR_INVALID, "ids_scores: workspace not 256-byte aligned");
    const Layout L = layout(n, dim);
    if (workspace_bytes < L.total)
        return fail(MIGAN_ERR_INVALID, "ids_scores: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
    char* ws = static_cast<char*>(workspace);
    double* beta = reinterpret_cast<double*>(ws + L.beta);
    double* bbar = reinterpret_cast<double*>(ws + L.bbar);
    double* g = reinterpret_cast<double*>(ws + L.g);
    double* r = reinterpret_cast<double*>(ws + L.r);
    double* o = reinterpret_cast<double*>(ws + L.o);
    double* ob = reinterpret_cast<double*>(ws + L.ob);
    int* idx = reinterpret_cast<int*>(ws + L.idx);
    double* part = reinterpret_cast<double*>(ws + L.part);
    int* off = reinterpret_cast<int*>(ws + L.off);
    double* lanes = reinterpret_cast<double*>(ws + L.lanes);
    double* ps = reinterpret_cast<double*>(ws + L.ps);
    double* pt = reinterpret_cast<double*>(ws + L.pt);
    double* G = reinterpret_cast<double*>(ws + L.G);
    double* scal = reinterpret_cast<double*>(ws + L.scal);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    const ids::Data X{real, fake, (int)n, dim, dtype == IDS_FLOAT64};
    const int Dp = padded(dim), D = dim + 1;
    const int64_t M = X.rows(), H = ids::chunks_of(M);

    CUDA_TRY(comod::ck_launch(ids::NonFiniteK{X, part}, H, s));
    CUDA_TRY(comod::ck_launch(ids::SumK{part, scal + ids::kNonFinite, H}, 1, s));
    double bad = 0.0;
    CUDA_TRY(to_host(&bad, scal + ids::kNonFinite, sizeof(bad), s));
    if (bad != 0.0) return fail(MIGAN_ERR_INVALID, "ids_scores: %.0f non-finite feature values", bad);

    // b_0 = 0, so o = 0; no active-set change recorded yet.
    CUDA_TRY(comod::ck_launch(ids::FillK{beta, 0.0}, Dp, s));
    CUDA_TRY(comod::ck_launch(ids::FillK{o, 0.0}, M, s));
    CUDA_TRY(comod::ck_launch(ids::FillK{scal, -1.0}, ids::kSlots, s));
    double g0 = 0.0, status[3] = {0.0, 0.0, -1.0};
    int k = 0, rule = 0;
    for (;; ++k) {
        // The active set at b_k and the gradient there.
        CUDA_TRY(comod::ck_launch(ids::ActiveCountK{X, o, part}, H, s));
        CUDA_TRY(comod::ck_launch(ids::ScanK{part, off, scal, H}, 1, s));
        CUDA_TRY(comod::ck_launch(ids::ScatterK{X, o, off, idx}, H, s));
        CUDA_TRY(comod::ck_launch(ids::GradPartK{X, o, idx, scal, Dp, ps, pt}, H * D, s));
        CUDA_TRY(comod::ck_launch(ids::GradK{ps, pt, beta, g, r, H, D, Dp}, Dp, s));
        CUDA_TRY(comod::ck_launch(ids::NormK{g, scal, D}, 1, s));
        CUDA_TRY(to_host(status, scal, sizeof(status), s));
        if (!isfinite(status[ids::kGnorm2])) return fail(MIGAN_ERR_INVALID, "ids_scores: the gradient is not finite");
        const double gn = sqrt(status[ids::kGnorm2]);
        if (k == 0) g0 = gn;
        if (k > 0 && status[ids::kMismatch] == 0.0) {
            rule = IDS_STOP_ACTIVE_SET;
        } else if (gn <= kGradTol * g0) {
            rule = IDS_STOP_GRADIENT;
        }
        if (rule) {
            out[4] = g0 > 0.0 ? gn / g0 : 0.0;
            break;
        }
        if (k == kMaxIter)
            return fail(MIGAN_ERR_INVALID,
                        "ids_scores: no convergence in %d Newton iterations (last active-set change %.0f rows, relative "
                        "gradient %.3g)", kMaxIter, status[ids::kMismatch], gn / g0);
        // b~, the rows that change sides there, the line search and the step.
        if (int rc = newton(X, idx, scal, G, r, bbar, Dp, s)) return rc;
        if (int rc = margins(X, bbar, lanes, ob, s)) return rc;
        CUDA_TRY(comod::ck_launch(ids::MismatchK{X, o, ob, part}, H, s));
        CUDA_TRY(comod::ck_launch(ids::SumK{part, scal + ids::kMismatch, H}, 1, s));
        CUDA_TRY(line_launch(ids::LineArgs{X, o, ob, beta, bbar, scal, Dp}, s));
        CUDA_TRY(comod::ck_launch(ids::StepK{beta, bbar, scal}, Dp, s));
        if (int rc = margins(X, beta, lanes, o, s)) return rc;
    }
    CUDA_TRY(comod::ck_launch(ids::ScorePartK{X, o, part}, H, s));
    CUDA_TRY(comod::ck_launch(ids::ScoreK{part, beta, scal, coef, H, dim}, 1, s));
    double res[ids::kSlots];
    CUDA_TRY(to_host(res, scal, sizeof(res), s));
    CUDA_TRY(to_host(out + 2, beta + dim, sizeof(double), s));
    out[0] = res[ids::kPairs] / (double)n;
    out[1] = res[ids::kWrong] / (2.0 * (double)n);
    out[3] = res[ids::kObjective];
    iterations[0] = k;
    iterations[1] = rule;
    return 0;
}

}  // extern "C"

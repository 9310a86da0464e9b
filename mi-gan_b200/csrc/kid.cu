// C ABI of the kernel Inception distance (include/inception_b200.h): kid_workspace_bytes and kid_subset_terms.
// Argument and index-table checks, workspace layout and the launches; the arithmetic is kid_kernels.cuh's.  The tile
// kernel is one body over portable.cuh's block layer, run with a block's threads at once on the device and on the host
// in the emulation build (MIGAN_EMULATE).
//
// Workspace (nb = m rounded up to 64, over 64; each region 256-byte aligned): the fake and the real index tables
// (S m ints each), the tile partials (S x 3 x nb^2 doubles).
#include <string.h>

#include <vector>

#include "../../include/inception_b200.h"
#include "abi_error.h"
#include "kid_kernels.cuh"

namespace {
using kid::kG;
using kid::kRedDoubles;
using kid::kThreads;
using kid::kTileDoubles;
using migan::fail;

static_assert(kid::kMaxDim == KID_MAX_DIM, "one cap");
static_assert(IDS_FLOAT32 == 0 && IDS_FLOAT64 == 1, "the dtype codes of ids_scores");
constexpr size_t kTileSmem = (2 * kTileDoubles + kRedDoubles) * sizeof(double);

template <class B>
CK_D void tile_block(const B& blk, const kid::TileArgs& a, int64_t b, double* smem) {
    double* Xs = smem;
    double* Ys = Xs + kTileDoubles;
    double* red = Ys + kTileDoubles;
    kid::Accs<B> c;
    frechet::panel_product(blk, c, a.fake.d, Xs, Ys, a, b);
    blk.each([&](int t) { a.reduce(b, t, c[t], red); });
    blk.sync();
    blk.each([&](int t) { a.combine(t, red); });
    blk.sync();
    blk.each([&](int t) { a.store(b, t, red); });
}

#ifdef MIGAN_EMULATE
int tile_launch(const kid::TileArgs& a, ck_stream_t) {
    return ck_blocks<kThreads>(a.blocks(), kTileSmem,
                               [&](auto& blk, int64_t b, void* smem) { tile_block(blk, a, b, (double*)smem); });
}
#else
__global__ void __launch_bounds__(kThreads) kid_tile_kernel(const __grid_constant__ kid::TileArgs a) {
    extern __shared__ __align__(16) double smem[];
    tile_block(DeviceBlock(), a, blockIdx.x, smem);
}

int tile_launch(const kid::TileArgs& a, ck_stream_t s) {
    if (int e = set_smem(kid_tile_kernel, kTileSmem)) return e;
    kid_tile_kernel<<<(unsigned)a.blocks(), kThreads, kTileSmem, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

struct Layout {
    size_t fake_idx, real_idx, partials, total;
};

Layout layout(int S, int m) {
    const size_t nb = (size_t)kid::tiles_of(m), table = align256((size_t)S * m * sizeof(int));
    Layout L;
    L.fake_idx = 0;
    L.real_idx = L.fake_idx + table;
    L.partials = L.real_idx + table;
    L.total = L.partials + align256((size_t)S * kid::kKinds * nb * nb * sizeof(double));
    return L;
}

// Grids and tables past 2^31 - 1 blocks or entries are refused rather than split.
bool bad_shape(int S, int m) {
    if (S < 1 || m < 2) return true;
    const int64_t nb = kid::tiles_of(m);
    return (int64_t)S * m >= ((int64_t)1 << 31) || (int64_t)S * (nb * (nb + 1) + nb * nb) >= ((int64_t)1 << 31);
}

// Every entry of idx[S][m] in 0..n-1 and the m entries of each subset distinct.
int check_table(const char* name, const int32_t* idx, int S, int m, int64_t n) {
    std::vector<int> seen((size_t)n, -1);
    for (int s = 0; s < S; ++s)
        for (int k = 0; k < m; ++k) {
            const int32_t v = idx[(int64_t)s * m + k];
            if (v < 0 || v >= n)
                return fail(MIGAN_ERR_INVALID, "kid_subset_terms: %s index %d of subset %d is %d, outside 0..%lld",
                            name, k, s, (int)v, (long long)(n - 1));
            if (seen[v] == s)
                return fail(MIGAN_ERR_INVALID, "kid_subset_terms: subset %d draws %s row %d twice", s, name, (int)v);
            seen[v] = s;
        }
    return MIGAN_OK;
}

}  // namespace

extern "C" {

size_t kid_workspace_bytes(int num_subsets, int m) {
    if (bad_shape(num_subsets, m)) return 0;
    return layout(num_subsets, m).total;
}

int kid_subset_terms(const void* real, int64_t n_real, const void* fake, int64_t n_fake, int dim, int dtype,
                     const int32_t* real_idx_host, const int32_t* fake_idx_host, int num_subsets, int m, double* terms,
                     void* workspace, size_t workspace_bytes, void* stream) {
    const int S = num_subsets;
    if (!real || !fake || !real_idx_host || !fake_idx_host || !terms || !workspace)
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: null real / fake / index table / terms / workspace");
    if (S < 1) return fail(MIGAN_ERR_INVALID, "kid_subset_terms: %d subsets (at least 1)", S);
    if (m < 2) return fail(MIGAN_ERR_INVALID, "kid_subset_terms: subsets of %d rows (at least 2)", m);
    if (m > n_real || m > n_fake)
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: subsets of %d rows from %lld real and %lld fake rows", m,
                    (long long)n_real, (long long)n_fake);
    if (n_real >= ((int64_t)1 << 31) || n_fake >= ((int64_t)1 << 31))
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: %lld real / %lld fake rows reach 2^31", (long long)n_real,
                    (long long)n_fake);
    if (dim < 1 || dim > kid::kMaxDim)
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: dim %d outside 1..%d", dim, kid::kMaxDim);
    if (dtype != IDS_FLOAT32 && dtype != IDS_FLOAT64)
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: dtype %d is neither IDS_FLOAT32 nor IDS_FLOAT64", dtype);
    if (bad_shape(S, m))
        return fail(MIGAN_ERR_INVALID, "kid_subset_terms: %d subsets of %d rows reach 2^31 tiles or table entries", S,
                    m);
    if (int rc = check_table("fake", fake_idx_host, S, m, n_fake)) return rc;
    if (int rc = check_table("real", real_idx_host, S, m, n_real)) return rc;
    if (reinterpret_cast<uintptr_t>(workspace) % 256)
        return fail(MIGAN_ERR_WORKSPACE, "kid_subset_terms: workspace not 256-byte aligned");
    const Layout L = layout(S, m);
    if (workspace_bytes < L.total)
        return fail(MIGAN_ERR_WORKSPACE, "kid_subset_terms: workspace of %zu bytes, %zu needed", workspace_bytes,
                    L.total);
    char* ws = static_cast<char*>(workspace);
    int* fake_idx = reinterpret_cast<int*>(ws + L.fake_idx);
    int* real_idx = reinterpret_cast<int*>(ws + L.real_idx);
    double* partials = reinterpret_cast<double*>(ws + L.partials);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    const size_t table = (size_t)S * m * sizeof(int);
    CUDA_TRY(to_device(fake_idx, fake_idx_host, table, s));
    CUDA_TRY(to_device(real_idx, real_idx_host, table, s));
    const int fp64 = dtype == IDS_FLOAT64;
    const kid::TileArgs a{kid::Rows{fake, dim, fp64}, kid::Rows{real, dim, fp64}, fake_idx, real_idx, m, S, partials};
    CUDA_TRY(tile_launch(a, s));
    CUDA_TRY(comod::ck_launch(kid::TermsK{partials, terms, a.nb()}, (int64_t)S * kid::kKinds, s));
    return 0;
}

}  // extern "C"

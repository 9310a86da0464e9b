// Arithmetic of the kernel Inception distance (kid.cu), written once for the device kernels and for the emulation
// build's host loops, the way ids_kernels.cuh is.  Everything is float64, there are no atomics, and every sum has an
// order that depends on the shapes alone, so a call returns the same bytes on every run and on every stream.
//
// KID (Binkowski et al. 2018) is the unbiased estimate of the squared MMD under the cubic polynomial kernel
//     k(u, v) = t t t,   t = (u.v) / d + 1,
// averaged over S subsets of m fake rows X and m real rows Y, drawn without replacement on the host.  Per subset the
// device computes three sums of kernel values:
//     Sxx = sum_{i != j} k(x_i, x_j),   Syy = sum_{i != j} k(y_i, y_j),   Sxy = sum_{i, j} k(x_i, y_j),
// and the host finishes e_s = ((Sxx + Syy) / (m - 1) - 2 Sxy / m) / m.
//
// Tile kernel: one block per 64 x 64 output tile of a subset's three Gram products, on the tiles on and below the
// diagonal of X X^T and Y Y^T and on every tile of X Y^T.  The block walks the features in 64-column panels: it stages
// the panels of its 64 tile rows and 64 tile columns, gathered through the subset's index tables and promoted to fp64
// (zero past m and past d), then multiplies them on fp64 mma.sync m8n8k4 (frechet::tile_mma, k in column order).  The
// epilogue applies t t t in registers, drops the diagonal i == j of the X X^T and Y Y^T tiles on it and everything past
// m (zero rows are not enough: k(0, v) = 1), and reduces the tile in a fixed order: each thread's 16 values in
// accumulator order, then 8 lanes of 32 threads, then the 8 lanes.  An off-diagonal tile of X X^T or Y Y^T stands for
// its mirror too and counts twice (x 2 is exact).  The partial goes to partials[s][kind][tile].
// Sum kernel: one item per (subset, kind) adds its partials in tile order into terms[s][kind].
#pragma once
#include "frechet_kernels.cuh"

namespace kid {

using frechet::Acc;
using frechet::Accs;
using frechet::acc_col;
using frechet::acc_row;
using frechet::kG;
using frechet::kLd;
using frechet::kThreads;
using frechet::kTileDoubles;
using frechet::Rows;
using metrics::ddiv;

constexpr int kMaxDim = 4096;
constexpr int kLanes = kThreads / 32;             // the reduction's second level: one lane per warp's worth of threads
constexpr int kRedDoubles = kThreads + kLanes;    // shared memory of the tile reduction
enum Kind { kXX = 0, kYY = 1, kXY = 2, kKinds = 3 };

CK_HD int tiles_of(int m) { return (m + kG - 1) / kG; }
CK_HD int64_t lower_tiles(int nb) { return (int64_t)nb * (nb + 1) / 2; }

// b = k (k + 1) / 2 + l, l <= k: the lower tile (k, l).  The float root is a guess; the loops make it exact.
CK_HD void lower_tile(int64_t b, int* k, int* l) {
    int64_t kk = (int64_t)((sqrt(8.0 * (double)b + 1.0) - 1.0) / 2.0);
    while (kk * (kk + 1) / 2 > b) --kk;
    while ((kk + 1) * (kk + 2) / 2 <= b) ++kk;
    *k = (int)kk;
    *l = (int)(b - kk * (kk + 1) / 2);
}

// The tile one block owns.
struct Tile {
    int s, kind, bi, bj;
    int64_t slot;     // its index among its kind's tiles of its subset
};

struct TileArgs {
    Rows fake, real; const int* fake_idx; const int* real_idx; int m, S; double* partials;

    CK_HD int nb() const { return tiles_of(m); }
    CK_HD int64_t per_subset() const { return 2 * lower_tiles(nb()) + (int64_t)nb() * nb(); }
    CK_HD int64_t blocks() const { return (int64_t)S * per_subset(); }

    // Blocks in subset order; within a subset the lower tiles of X X^T, those of Y Y^T, then X Y^T row by row.
    CK_HD Tile tile(int64_t b) const {
        const int64_t per = per_subset(), L = lower_tiles(nb());
        Tile T;
        T.s = (int)(b / per);
        int64_t r = b % per;
        if (r < 2 * L) {
            T.kind = r < L ? kXX : kYY;
            T.slot = r < L ? r : r - L;
            lower_tile(T.slot, &T.bi, &T.bj);
        } else {
            T.kind = kXY;
            T.slot = r - 2 * L;
            T.bi = (int)(T.slot / nb());
            T.bj = (int)(T.slot % nb());
        }
        return T;
    }
    // Xs[k][x] = the row side's feature k0 + k of tile row x, Ys[k][x] the column side's; 0 past m and past d.
    CK_HD void stage(int64_t b, int t, int k0, double* Xs, double* Ys) const {
        const Tile T = tile(b);
        const Rows& A = T.kind == kYY ? real : fake;
        const Rows& B = T.kind == kXX ? fake : real;
        const int* ia = (T.kind == kYY ? real_idx : fake_idx) + (int64_t)T.s * m;
        const int* ib = (T.kind == kXX ? fake_idx : real_idx) + (int64_t)T.s * m;
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, k = e % kG, c = k0 + k;
            const int ra = T.bi * kG + x, rb = T.bj * kG + x;
            Xs[k * kLd + x] = ra < m && c < A.d ? A.x(ia[ra], c) : 0.0;
            Ys[k * kLd + x] = rb < m && c < B.d ? B.x(ib[rb], c) : 0.0;
        }
    }
    // red[t] = thread t's kernel values in accumulator order, past m and the diagonal of X X^T, Y Y^T left out.
    CK_HD void reduce(int64_t b, int t, const Acc& c, double* red) const {
        const Tile T = tile(b);
        const int i = T.bi * kG + acc_row(t);
        const double d = (double)fake.d;
        double sum = 0.0;
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) {
                const int j = T.bj * kG + acc_col(t, nt, h);
                if (i >= m || j >= m || (T.kind != kXY && i == j)) continue;
                const double u = dadd_rn(ddiv(c.v[nt][h], d), 1.0);
                sum = dadd_rn(sum, dmul_rn(dmul_rn(u, u), u));
            }
        red[t] = sum;
    }
    // red[kThreads + w] = red[32 w .. 32 w + 31] in order, for w < kLanes.
    CK_HD void combine(int t, double* red) const {
        if (t >= kLanes) return;
        double sum = 0.0;
        for (int k = 0; k < 32; ++k) sum = dadd_rn(sum, red[32 * t + k]);
        red[kThreads + t] = sum;
    }
    // partials[s][kind][slot] = the lanes in order, twice for an off-diagonal tile of X X^T or Y Y^T.
    CK_HD void store(int64_t b, int t, const double* red) const {
        if (t != 0) return;
        const Tile T = tile(b);
        double sum = 0.0;
        for (int w = 0; w < kLanes; ++w) sum = dadd_rn(sum, red[kThreads + w]);
        if (T.kind != kXY && T.bi != T.bj) sum = dmul_rn(2.0, sum);
        partials[((int64_t)T.s * kKinds + T.kind) * nb() * nb() + T.slot] = sum;
    }
};

// terms[s][kind] = partials[s][kind][0 ..) in tile order.  items = S * kKinds.
struct TermsK {
    const double* partials; double* terms; int nb;
    CK_HD void operator()(int64_t e) const {
        const int64_t count = e % kKinds == kXY ? (int64_t)nb * nb : lower_tiles(nb);
        const double* p = partials + e * nb * nb;
        double sum = 0.0;
        for (int64_t k = 0; k < count; ++k) sum = dadd_rn(sum, p[k]);
        terms[e] = sum;
    }
};

}  // namespace kid

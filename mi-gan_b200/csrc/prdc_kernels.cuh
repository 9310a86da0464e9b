// Arithmetic of precision, recall, density and coverage (prdc.cu), written once for the device kernels and for the
// emulation build's host loops, the way kid_kernels.cuh is.  Distances are float64 and squared throughout; the
// selection keeps values, not indices, and the flags and counts are integers, so a call returns the same bytes on every
// run, on any stream and for any order of the rows.
//
// The manifold metrics (Kynkaanniemi et al. 2019, Naeem et al. 2020) of real rows Y [N] and fake rows X [M], with
// r_i the (k + 1)-th smallest of {|Y_i - Y_j|^2 : j} (row i itself included, its 0 first) and s_j the same within X:
//     precision = #{j : exists i, |X_j - Y_i|^2 <= r_i} / M       recall   = #{i : exists j, |Y_i - X_j|^2 <= s_j} / N
//     density   = sum_j #{i : |X_j - Y_i|^2 <= r_i} / (k M)       coverage = #{i : min_j |Y_i - X_j|^2 <= r_i} / N
// The device computes the four integer counts; the caller divides.
//
// Distance: |a - b|^2 = max(0, (|a|^2 + |b|^2) - 2 a.b), with a.b from 64 x 64 fp64 DMMA tiles (frechet::tile_mma, the
// features in 64-column panels in column order) and |a|^2 from the diagonal of the same tile product of a's own tile.
// For a = b the three terms are the same bits, so identical rows are at distance exactly 0, within a set and across the
// two sets; and a.b is the same bits as b.a, so every distance is a function of its two rows alone.
//
// One tile kernel runs three kinds of pass, a block per (row tile, column split): it walks the column tiles of its split
// and, per column tile, stages both 64-row panels (promoted to fp64, zero past n and past d), multiplies them, and hands
// the accumulators to the pass's epilogue:
//   kNorms   the diagonal tile of a set only: |a|^2 of each row.
//   kRadii   the set against itself: each thread keeps the k + 1 smallest distances of its row among its 16 columns
//            per tile, sorted, in shared memory; the block writes the lists, and RadiusK merges a row's 4 x splits lists
//            into r.
//   kCross   X (rows) against Y (columns): per fake row the count of reals with d <= r_i (a per-thread counter, summed
//            over the row's 4 threads into counts[split][j]); per real column whether some fake lies within r_i
//            (coverage) and whether it lies within some s_j (recall), ORed in shared memory per tile and then into the
//            per-real flags.
// TotalsPartK and TotalsK add the counts and flags into out[4] = {precision, recall, density, coverage} counts.
#pragma once
#include "frechet_kernels.cuh"

namespace prdc {

using frechet::Acc;
using frechet::acc_col;
using frechet::acc_row;
using frechet::kG;
using frechet::kLd;
using frechet::kThreads;
using frechet::kTileDoubles;
using frechet::Rows;

constexpr int kMaxDim = 4096;
constexpr int kMaxK = 32;        // the neighbourhood size: lists of at most 33 values per thread
constexpr int kSplits = 8;       // column splits of a pass: a block walks at most ceil(tiles / 8) column tiles
enum Mode { kNorms = 0, kRadii = 1, kCross = 2 };

CK_HD int tiles_of(int64_t n) { return (int)((n + kG - 1) / kG); }
CK_HD int splits_of(int col_tiles) { return col_tiles < kSplits ? col_tiles : kSplits; }

// max(0, (na + nb) - 2 g): 0 exactly when na = nb = g.
CK_HD double sq_dist(double na, double nb, double g) {
    const double v = dsub_rn(dadd_rn(na, nb), dmul_rn(2.0, g));
    return v > 0.0 ? v : 0.0;
}

// v into the ascending list L[0], L[stride], .., L[(n - 1) stride], dropping its largest value; equal values are
// interchangeable, so a value not below the largest leaves the list as it is.
CK_HD void insert(double* L, int n, int stride, double v) {
    if (!(v < L[(n - 1) * stride])) return;
    int p = n - 1;
    while (p > 0 && L[(p - 1) * stride] > v) {
        L[p * stride] = L[(p - 1) * stride];
        --p;
    }
    L[p * stride] = v;
}

// *p |= 1, from any thread of any block.
CK_HD void flag_set(int* p) {
#ifdef __CUDA_ARCH__
    atomicOr(p, 1);
#else
    __atomic_fetch_or(p, 1, __ATOMIC_RELAXED);
#endif
}

// The thread that holds accumulator row r, column quarter q.
CK_HD int row_thread(int r, int q) { return (r / 8) * 32 + (r % 8) * 4 + q; }

struct PassArgs {
    Rows A, B;                   // row side and column side (the same rows for kNorms and kRadii)
    int nA, nB, mode, K1;        // K1 = k + 1
    const double* normA; const double* normB;
    double* norms;               // kNorms: |a|^2 [nA]
    double* lists;               // kRadii: [row tile][split][K1][kThreads]
    const double* rA; const double* rB;    // kCross: s_j of the fake rows, r_i of the real columns
    int* counts;                 // kCross: [split][row tiles x kG]
    int* cov; int* rec;          // kCross: [nB]

    CK_HD int row_tiles() const { return tiles_of(nA); }
    CK_HD int col_tiles() const { return tiles_of(nB); }
    CK_HD int splits() const { return mode == kNorms ? 1 : splits_of(col_tiles()); }
    CK_HD int64_t blocks() const { return (int64_t)row_tiles() * splits(); }
    CK_HD int bi(int64_t b) const { return (int)(b / splits()); }
    CK_HD int split(int64_t b) const { return (int)(b % splits()); }
    // Column tiles [first, last) of block b: the diagonal tile for kNorms, else split s of splits() near-equal ranges.
    CK_HD int first(int64_t b) const {
        return mode == kNorms ? bi(b) : (int)((int64_t)split(b) * col_tiles() / splits());
    }
    CK_HD int last(int64_t b) const {
        return mode == kNorms ? bi(b) + 1 : (int)((int64_t)(split(b) + 1) * col_tiles() / splits());
    }
    // Doubles of shared memory past the two panels: the lists, or the counters and the tile's flags.
    CK_HD int extra_doubles() const {
        return mode == kRadii ? K1 * kThreads : mode == kCross ? (kThreads + 2 * kG) / 2 : 0;
    }

    // kRadii: thread t's list empty (+inf).  kCross: its counter and the tile flags zero.
    CK_HD void begin(int t, double* ex) const {
        if (mode == kRadii) {
            for (int s = 0; s < K1; ++s) ex[s * kThreads + t] = INFINITY;
        } else if (mode == kCross) {
            int* ix = reinterpret_cast<int*>(ex);
            ix[t] = 0;
            if (t < 2 * kG) ix[kThreads + t] = 0;
        }
    }
    // Xs[k][x] = feature k0 + k of row tile bi's row x, Ys[k][x] of column tile jt's; 0 past n and past d.
    CK_HD void stage(int64_t b, int jt, int t, int k0, double* Xs, double* Ys) const {
        const int r0 = bi(b) * kG, c0 = jt * kG;
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, k = e % kG, c = k0 + k;
            Xs[k * kLd + x] = r0 + x < nA && c < A.d ? A.x(r0 + x, c) : 0.0;
            Ys[k * kLd + x] = c0 + x < nB && c < B.d ? B.x(c0 + x, c) : 0.0;
        }
    }
    CK_HD void product(int t, Acc& c, const double* Xs, const double* Ys) const {
        frechet::tile_mma(c, t, Xs, 1, kLd, Ys);
    }
    CK_HD void epilogue(int64_t b, int jt, int t, const Acc& c, double* ex) const {
        const int i = bi(b) * kG + acc_row(t);
        if (i >= nA) return;
        if (mode == kNorms) {
            for (int nt = 0; nt < 8; ++nt)
                for (int h = 0; h < 2; ++h)
                    if (acc_col(t, nt, h) == acc_row(t)) norms[i] = c.v[nt][h];
        } else if (mode == kRadii) {
            const double ni = normA[i];
            for (int nt = 0; nt < 8; ++nt)
                for (int h = 0; h < 2; ++h) {
                    const int j = jt * kG + acc_col(t, nt, h);
                    if (j < nB) insert(ex + t, K1, kThreads, sq_dist(ni, normB[j], c.v[nt][h]));
                }
        } else {
            int* ix = reinterpret_cast<int*>(ex);
            const double ni = normA[i], si = rA[i];
            int n = 0;
            for (int nt = 0; nt < 8; ++nt)
                for (int h = 0; h < 2; ++h) {
                    const int col = acc_col(t, nt, h), j = jt * kG + col;
                    if (j >= nB) continue;
                    const double v = sq_dist(ni, normB[j], c.v[nt][h]);
                    if (v <= rB[j]) {
                        ++n;
                        flag_set(ix + kThreads + col);
                    }
                    if (v <= si) flag_set(ix + kThreads + kG + col);
                }
            ix[t] += n;
        }
    }
    // kCross, after the epilogue's barrier: thread t < kG moves column t's tile flags into the per-real flags.
    CK_HD void flush(int jt, int t, double* ex) const {
        if (mode != kCross || t >= kG) return;
        int* ix = reinterpret_cast<int*>(ex) + kThreads;
        const int j = jt * kG + t;
        if (j < nB && ix[t]) flag_set(cov + j);
        if (j < nB && ix[kG + t]) flag_set(rec + j);
        ix[t] = ix[kG + t] = 0;
    }
    // kRadii: thread t's list to lists[bi][split].  kCross: thread t < kG sums row t's four counters.
    CK_HD void end(int64_t b, int t, const double* ex) const {
        if (mode == kRadii) {
            double* L = lists + ((int64_t)bi(b) * splits() + split(b)) * K1 * kThreads;
            for (int s = 0; s < K1; ++s) L[s * kThreads + t] = ex[s * kThreads + t];
        } else if (mode == kCross && t < kG) {
            const int* ix = reinterpret_cast<const int*>(ex);
            int n = 0;
            for (int q = 0; q < 4; ++q) n += ix[row_thread(t, q)];
            counts[(int64_t)split(b) * row_tiles() * kG + (int64_t)bi(b) * kG + t] = n;
        }
    }
};

// r[i] = the K1-th smallest of row i's 4 x splits lists, merged into the first one in place.  items = n.
struct RadiusK {
    double* lists; double* r; int K1, splits;
    CK_HD void operator()(int64_t i) const {
        const int64_t rt = i / kG;
        const int row = (int)(i % kG);
        double* base = lists + rt * splits * K1 * kThreads + row_thread(row, 0);
        for (int m = 1; m < 4 * splits; ++m) {   // list m: split m / 4, quarter m % 4
            const double* L = base + (int64_t)(m / 4) * K1 * kThreads + m % 4;
            for (int p = 0; p < K1 && L[p * kThreads] < base[(K1 - 1) * kThreads]; ++p)
                insert(base, K1, kThreads, L[p * kThreads]);
        }
        r[i] = base[(K1 - 1) * kThreads];
    }
};

// The per-real flags zero.  items = n.
struct ZeroK {
    int* cov; int* rec;
    CK_HD void operator()(int64_t i) const { cov[i] = rec[i] = 0; }
};

// Item e < tiles_of(M): fake rows [64 e, 64 e + 64): part[e] = {#rows with a count, sum of counts}, each row's count
// summed over the splits.  Item tiles_of(M) + e: real rows [64 e, ..): part = {#recall flags, #coverage flags}.
struct TotalsPartK {
    const int* counts; const int* cov; const int* rec; int64_t* part; int M, N, splits;
    CK_HD void operator()(int64_t e) const {
        const int tm = tiles_of(M);
        int64_t a = 0, b = 0;
        if (e < tm) {
            for (int j = (int)e * kG; j < M && j < (int)(e + 1) * kG; ++j) {
                int64_t c = 0;
                for (int s = 0; s < splits; ++s) c += counts[(int64_t)s * tm * kG + j];
                a += c > 0;
                b += c;
            }
        } else {
            for (int i = (int)(e - tm) * kG; i < N && i < (int)(e - tm + 1) * kG; ++i) {
                a += rec[i] != 0;
                b += cov[i] != 0;
            }
        }
        part[2 * e] = a;
        part[2 * e + 1] = b;
    }
};

// out = {precision, recall, density, coverage} counts from the parts.  items = 1.
struct TotalsK {
    const int64_t* part; int64_t* out; int M, N;
    CK_HD void operator()(int64_t) const {
        const int tm = tiles_of(M), tn = tiles_of(N);
        int64_t precision = 0, recall = 0, density = 0, coverage = 0;
        for (int e = 0; e < tm; ++e) {
            precision += part[2 * e];
            density += part[2 * e + 1];
        }
        for (int e = tm; e < tm + tn; ++e) {
            recall += part[2 * e];
            coverage += part[2 * e + 1];
        }
        out[0] = precision;
        out[1] = recall;
        out[2] = density;
        out[3] = coverage;
    }
};

}  // namespace prdc

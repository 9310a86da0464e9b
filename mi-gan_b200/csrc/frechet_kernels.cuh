// Arithmetic of the Fréchet distance (frechet.cu), written once for the device kernels and for the emulation build, the
// way metrics_kernels.cuh is: a block kernel's body (portable.cuh's block layer) calls these phase functions for each
// thread between its barriers, and the same body runs in both builds.
// Everything is float64, there are no atomics, and every sum has a fixed order, so a call returns the same bytes on
// every run.
//
// tr sqrt(S1 S2) = sum_i sqrt(max(lambda_i(M), 0)) with M = D^1/2 V^T S2 V D^1/2 and S1 = V D V^T: two symmetric
// eigenproblems on matrices padded to N = a multiple of kG (zero rows and columns; padding adds zero eigenvalues).
//
// Eigensolver: parallel block Jacobi.  The N indices form nb = N / kB blocks of kB; a sweep is nb - 1 rounds of the
// round-robin (circle) pairing of the blocks, so every pair of blocks meets once per sweep.  One round is two launches:
//   pair kernel   one CTA per block pair (p, q): the kG x kG subproblem A[I, I] (I = block p, then block q) is
//                 reduced by cyclic scalar Jacobi in shared memory: kMaxInner sweeps in the circle order of its kG
//                 indices (one: more leave the outer sweep count as it is), stopping early when a sweep rotates
//                 nothing.  Rotations are at most 45 degrees
//                 and start from the identity, so the factor J stays close to the identity (no sorting, no swaps).
//                 The CTA writes J - I; the diagonalised subproblem itself is discarded.
//   update kernel A[I_k, I_l] <- J_k^T A[I_k, I_l] J_l for the tiles on and below the diagonal (mirrored, so A stays
//                 exactly symmetric), and V[:, I_l] <- V[:, I_l] J_l in the first solve: 64 x 64 x 64 products on fp64
//                 mma.sync m8n8k4 (the emulation runs the same products as loops, in the same k order).
// A rotation is skipped when |a_pq| <= 2^-53 sqrt(|a_pp|) sqrt(|a_qq|): then J is exactly the identity wherever nothing
// rotates, and the update leaves those entries exactly as they are.
#pragma once
#include "metrics_kernels.cuh"

namespace frechet {

using metrics::ddiv;

constexpr int kB = 32;              // block size of the eigensolver
constexpr int kG = 2 * kB;          // one pair of blocks: the subproblem and the tile size
constexpr int kLd = kG + 1;         // shared-memory row stride of a kG x kG tile (doubles)
constexpr int kThreads = 256;       // 8 warps; warp w owns rows 8w..8w+7 of a tile product
constexpr int kMaxInner = 1;        // inner sweeps of a pair kernel: more leave the outer sweeps as they are
constexpr int kMaxDim = 4096;
constexpr double kEps = 1.1102230246251565e-16;   // 2^-53
constexpr int kTileDoubles = kG * kLd;

CK_HD double dsqrt(double x) { return sqrt(x); }

// One side's feature rows, fp32 or fp64 as stored, promoted exactly to fp64.
struct Rows {
    const void* p; int d, fp64;

    CK_HD double x(int64_t row, int c) const {
        const int64_t e = row * d + c;
        return fp64 ? static_cast<const double*>(p)[e] : (double)static_cast<const float*>(p)[e];
    }
};
CK_HD double dabs(double x) { return fabs(x); }

// Round r (0 <= r < m - 1) of the circle pairing of m (even) players: pair k of m / 2, returned with a < b.
CK_HD void circle(int m, int r, int k, int* a, int* b) {
    int x, y;
    if (k == 0) {
        x = r;
        y = m - 1;
    } else {
        x = (r + k) % (m - 1);
        y = (r - k + m - 1) % (m - 1);
    }
    *a = x < y ? x : y;
    *b = x < y ? y : x;
}
// Global index of position x (0 <= x < kG) of the block pair (p, q).
CK_HD int pair_index(int p, int q, int x) { return x < kB ? p * kB + x : q * kB + (x - kB); }

// ---- item kernels ---------------------------------------------------------------------------------------------------
// mu = shift + sum / n and sigma = (sumsq - sum sum^T / n) / (n - 1), each operation rounded on its own in the order of
// FeatureStatistics.mean_cov() (np.outer, then / n, then the difference, then / (n - 1)).  items = dim * dim.
struct MeanCovK {
    const double* shift; const double* sum; const double* sumsq; double* mu; double* sigma; int dim; double n;
    CK_HD void operator()(int64_t i) const {
        const int a = (int)(i / dim), b = (int)(i % dim);
        sigma[i] = ddiv(dsub_rn(sumsq[i], ddiv(dmul_rn(sum[a], sum[b]), n)), dsub_rn(n, 1.0));
        if (a == 0) mu[b] = dadd_rn(shift[b], ddiv(sum[b], n));
    }
};

// A[N][N] = (S + S^T) / 2 padded with zeros; V = the identity when given.  items = N * N.
struct LoadK {
    const double* S; double* A; double* V; int n, N;
    CK_HD void operator()(int64_t i) const {
        const int r = (int)(i / N), c = (int)(i % N);
        double v = 0.0;
        if (r < n && c < n) v = dmul_rn(0.5, dadd_rn(S[(int64_t)r * n + c], S[(int64_t)c * n + r]));
        A[i] = v;
        if (V) V[i] = r == c ? 1.0 : 0.0;
    }
};

// The numerical-rank cutoff of the diagonalised S1: dim 2^-52 max_i |d_i|, as numpy's matrix_rank draws it.  The
// eigenvalues of S1 at or below it are indistinguishable from 0 in float64 (a rank-deficient covariance's null space
// comes out as +-round-off) and count as 0, so M is exactly 0 on that null space.  Otherwise the square roots of
// round-off-sized eigenvalues of M add a floor to the trace.  M's own eigenvalues are only clamped at 0: they can
// span more decades than the cutoff allows (d1 d2 from 1e-11 to 1e3 for spectra 1e-6..1e2 and 1e-5..1e1), and the
// Jacobi solver resolves them.
CK_HD double rank_cutoff(const double* A, int dim, int N) {
    double m = 0.0;
    for (int i = 0; i < N; ++i) m = fmax(m, dabs(A[(int64_t)i * N + i]));
    return dmul_rn(dmul_rn((double)dim, 2.0 * kEps), m);
}
// cut[0] = rank_cutoff(A).  items = 1.
struct CutoffK {
    const double* A; double* cut; int dim, N;
    CK_HD void operator()(int64_t) const { cut[0] = rank_cutoff(A, dim, N); }
};

// sd[i] = sqrt(A[i][i]) above the cutoff, else 0.  items = N.
struct SqrtDiagK {
    const double* A; const double* cut; double* sd; int N;
    CK_HD void operator()(int64_t i) const {
        const double d = A[i * N + i];
        sd[i] = d > cut[0] ? dsqrt(d) : 0.0;
    }
};

// M[i][j] = (W[i][j] + W[j][i]) / 2 * (sd[i] sd[j]): exactly symmetric.  items = N * N.
struct ScaleK {
    const double* W; const double* sd; double* M; int N;
    CK_HD void operator()(int64_t e) const {
        const int i = (int)(e / N), j = (int)(e % N);
        M[e] = dmul_rn(dmul_rn(0.5, dadd_rn(W[e], W[(int64_t)j * N + i])), dmul_rn(sd[i], sd[j]));
    }
};

// Column j's sum of squares off the diagonal and its diagonal square, rows in order.  items = N.
struct ColNormK {
    const double* A; double* part; int N;
    CK_HD void operator()(int64_t j) const {
        double off = 0.0;
        for (int i = 0; i < N; ++i)
            if (i != j) off = fma(A[(int64_t)i * N + j], A[(int64_t)i * N + j], off);
        const double d = A[j * N + j];
        part[2 * j] = off;
        part[2 * j + 1] = dmul_rn(d, d);
    }
};
// out[0] = off(A)^2, out[1] = ||A||_F^2, columns in order.  items = 1.
struct NormSumK {
    const double* part; double* out; int N;
    CK_HD void operator()(int64_t) const {
        double off = 0.0, diag = 0.0;
        for (int j = 0; j < N; ++j) {
            off = dadd_rn(off, part[2 * j]);
            diag = dadd_rn(diag, part[2 * j + 1]);
        }
        out[0] = off;
        out[1] = dadd_rn(off, diag);
    }
};

// out = {||mu1 - mu2||^2, tr S1, tr S2, sum_i sqrt(max(lambda_i, 0))}, each summed in index order.  items = 1.
struct ResultK {
    const double* mu1; const double* s1; const double* mu2; const double* s2; const double* A; double* out; int n, N;
    CK_HD void operator()(int64_t) const {
        double dm = 0.0, t1 = 0.0, t2 = 0.0, ts = 0.0;
        for (int i = 0; i < n; ++i) {
            const double d = dsub_rn(mu1[i], mu2[i]);
            dm = fma(d, d, dm);
            t1 = dadd_rn(t1, s1[(int64_t)i * n + i]);
            t2 = dadd_rn(t2, s2[(int64_t)i * n + i]);
        }
        for (int i = 0; i < N; ++i) {
            const double l = A[(int64_t)i * N + i];
            if (l > 0.0) ts = dadd_rn(ts, dsqrt(l));
        }
        out[0] = dm;
        out[1] = t1;
        out[2] = t2;
        out[3] = ts;
    }
};

// ---- the tile product: C[64][64] += X * Y on fp64 mma.sync m8n8k4 ----------------------------------------------------
// X(i, k) = X[i * xr + k * xc], Y(k, j) = Y[k * kLd + j] in shared memory.  Thread t (warp w = t / 32, lane g * 4 + q)
// owns C(8w + g, 8nt + 2q + h) for nt < 8, h < 2 in acc[nt][h]: the m8n8k4 accumulator layout.  The emulation computes
// the same outputs as loops with one fma per product in k order, which is the order a k-step of 4 is accumulated in.
struct Acc {
    double v[8][2];
};
CK_HD void acc_zero(Acc& c) {
    for (int nt = 0; nt < 8; ++nt) c.v[nt][0] = c.v[nt][1] = 0.0;
}
CK_HD int acc_row(int t) { return (t / 32) * 8 + (t % 32) / 4; }
CK_HD int acc_col(int t, int nt, int h) { return nt * 8 + (t % 4) * 2 + h; }
// acc = thread t's entries of the kG x kLd tile X.
CK_HD void acc_load(Acc& c, int t, const double* X) {
    for (int nt = 0; nt < 8; ++nt)
        for (int h = 0; h < 2; ++h) c.v[nt][h] = X[acc_row(t) * kLd + acc_col(t, nt, h)];
}

#ifdef __CUDA_ARCH__
__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
        : "+d"(c[0]), "+d"(c[1])
        : "d"(a), "d"(b));
}
__device__ __forceinline__ void tile_mma(Acc& c, int t, const double* X, int xr, int xc, const double* Y) {
    const int lane = t % 32, g = lane / 4, q = lane % 4, row = (t / 32) * 8 + g;
#pragma unroll 4
    for (int k0 = 0; k0 < kG; k0 += 4) {
        const double a = X[row * xr + (k0 + q) * xc];
        const double* y = Y + (k0 + q) * kLd + g;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) dmma(c.v[nt], a, y[nt * 8]);
    }
}
#else
inline void tile_mma(Acc& c, int t, const double* X, int xr, int xc, const double* Y) {
    const int row = acc_row(t);
    for (int nt = 0; nt < 8; ++nt)
        for (int h = 0; h < 2; ++h) {
            const int col = acc_col(t, nt, h);
            double s = c.v[nt][h];
            for (int k = 0; k < kG; ++k) s = fma(X[row * xr + k * xc], Y[k * kLd + col], s);
            c.v[nt][h] = s;
        }
}
#endif

// A block's accumulators: one Acc per thread.
template <class B>
using Accs = typename B::template Local<Acc>;

// c = the product of the panels over the K extent, kG columns at a time: a.stage(tile..., t, k0, Xs, Ys) writes thread
// t's share of the panels Xs[k][x], Ys[k][x] of columns k0 .. k0 + kG, and the tile product adds them in k order.
template <class B, class Args, class... Tile>
CK_D void panel_product(const B& blk, Accs<B>& c, int K, double* Xs, double* Ys, const Args& a, Tile... tile) {
    blk.each([&](int t) { acc_zero(c[t]); });
    for (int k0 = 0; k0 < K; k0 += kG) {
        blk.each([&](int t) { a.stage(tile..., t, k0, Xs, Ys); });
        blk.sync();
        blk.each([&](int t) { tile_mma(c[t], t, Xs, 1, kLd, Ys); });
        blk.sync();
    }
}

// ---- pair kernel ----------------------------------------------------------------------------------------------------
// Block pair k of round `round`.  Shared memory: S and K = J - I (kG x kLd each), then kB rotations (c, s, t, c - 1).
// The factor is kept as its difference from the identity, and so is every update made with it: a rotation by a small
// angle then changes K, and through it A and V, by amounts rounded relative to the change, not to the entries.
struct PairArgs {
    double* A; double* J; int N, nb, round;

    CK_HD void blocks(int k, int* p, int* q) const { circle(nb, round, k, p, q); }

    CK_HD void load(int k, int t, double* S, double* Jl) const {
        int p, q;
        blocks(k, &p, &q);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            S[x * kLd + y] = A[(int64_t)pair_index(p, q, x) * N + pair_index(p, q, y)];
            Jl[x * kLd + y] = 0.0;
        }
    }

    // Thread t < kB: the rotation of pair t of inner step `step`; returns 1 when it rotates.
    CK_HD int rot(int step, int t, const double* S, double* cs) const {
        int i, j;
        circle(kG, step, t, &i, &j);
        const double aii = S[i * kLd + i], ajj = S[j * kLd + j], aij = S[i * kLd + j];
        double c = 1.0, s = 0.0, tn = 0.0, cm1 = 0.0;
        const int go = dabs(aij) > dmul_rn(dmul_rn(kEps, dsqrt(dabs(aii))), dsqrt(dabs(ajj)));
        if (go) {
            // Golub & Van Loan's sym.schur2: tau = (a_jj - a_ii) / (2 a_ij), t = sign(tau) / (|tau| + sqrt(1 + tau^2))
            const double tau = ddiv(dsub_rn(ajj, aii), dmul_rn(2.0, aij));
            const double at = dabs(tau);
            tn = at > 1e150 ? ddiv(0.5, at) : ddiv(1.0, dadd_rn(at, dsqrt(fma(at, at, 1.0))));
            if (tau < 0.0) tn = -tn;
            const double r = dsqrt(fma(tn, tn, 1.0));
            c = ddiv(1.0, r);
            s = dmul_rn(tn, c);
            cm1 = -ddiv(dmul_rn(tn, tn), dmul_rn(r, dadd_rn(1.0, r)));   // c - 1 without the cancellation
        }
        cs[4 * t] = c;
        cs[4 * t + 1] = s;
        cs[4 * t + 2] = tn;
        cs[4 * t + 3] = cm1;
        return go;
    }

    // S <- R^T S R (each 2 x 2 sub-block of two rotation pairs at once, the lower ones mirrored), J <- J R as
    // K <- K + (I + K)(R - I).
    CK_HD void apply(int step, int t, double* S, double* Jl, const double* cs) const {
        for (int e = t; e < kB * kB; e += kThreads) {
            const int P = e / kB, Q = e % kB;
            if (Q > P) continue;
            int i, j, k, l;
            circle(kG, step, P, &i, &j);
            const double cp = cs[4 * P], sp = cs[4 * P + 1];
            if (P == Q) {
                const double tn = cs[4 * P + 2], aij = S[i * kLd + j];
                S[i * kLd + i] = fma(-tn, aij, S[i * kLd + i]);
                S[j * kLd + j] = fma(tn, aij, S[j * kLd + j]);
                if (tn != 0.0) S[i * kLd + j] = S[j * kLd + i] = 0.0;
                continue;
            }
            circle(kG, step, Q, &k, &l);
            const double cq = cs[4 * Q], sq = cs[4 * Q + 1];
            const double bik = S[i * kLd + k], bil = S[i * kLd + l], bjk = S[j * kLd + k], bjl = S[j * kLd + l];
            // rows: i' = c i - s j, j' = s i + c j
            const double tik = fma(cp, bik, -dmul_rn(sp, bjk)), til = fma(cp, bil, -dmul_rn(sp, bjl));
            const double tjk = fma(sp, bik, dmul_rn(cp, bjk)), tjl = fma(sp, bil, dmul_rn(cp, bjl));
            // columns: k' = c k - s l, l' = s k + c l
            const double nik = fma(cq, tik, -dmul_rn(sq, til)), nil = fma(sq, tik, dmul_rn(cq, til));
            const double njk = fma(cq, tjk, -dmul_rn(sq, tjl)), njl = fma(sq, tjk, dmul_rn(cq, tjl));
            S[i * kLd + k] = S[k * kLd + i] = nik;
            S[i * kLd + l] = S[l * kLd + i] = nil;
            S[j * kLd + k] = S[k * kLd + j] = njk;
            S[j * kLd + l] = S[l * kLd + j] = njl;
        }
        for (int e = t; e < kG * kB; e += kThreads) {
            const int r = e / kB, P = e % kB;
            int i, j;
            circle(kG, step, P, &i, &j);
            const double s = cs[4 * P + 1], cm1 = cs[4 * P + 3];
            const double ki = Jl[r * kLd + i], kj = Jl[r * kLd + j];
            const double ji = dadd_rn(r == i ? 1.0 : 0.0, ki), jj = dadd_rn(r == j ? 1.0 : 0.0, kj);
            Jl[r * kLd + i] = dadd_rn(ki, fma(cm1, ji, -dmul_rn(s, jj)));
            Jl[r * kLd + j] = dadd_rn(kj, fma(s, ji, dmul_rn(cm1, jj)));
        }
    }

    CK_HD void store(int k, int t, const double* S, const double* Jl) const {
        int p, q;
        blocks(k, &p, &q);
        double* Jk = J + (int64_t)k * kG * kG;
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            Jk[e] = Jl[x * kLd + y];
        }
    }
};

// ---- update kernel --------------------------------------------------------------------------------------------------
// Blocks [0, tilesA): tile (k, l), k >= l, of the pair groups: A[I_k, I_l] <- J_k^T A[I_k, I_l] J_l, written with its
// mirror (the diagonal tiles: their lower triangle, mirrored).  Blocks [tilesA, tilesA + (N / kG) * groups) when V is
// given: V[rows, I_l] <- V[rows, I_l] J_l.  With J = I + K both products are increments, X + X K_l and T + K_k^T T: the
// accumulators start from the tile.  Shared memory: three kG x kLd tiles X, P, R.
struct UpdateArgs {
    double* A; double* V; const double* J; int N, nb, round, tilesA;

    CK_HD int groups() const { return nb / 2; }
    CK_HD int64_t blocks() const { return tilesA + (V ? (int64_t)(N / kG) * groups() : 0); }
    CK_HD void tile_of(int64_t b, int* k, int* l) const {   // b = k (k + 1) / 2 + l, l <= k
        int kk = 0;
        while ((int64_t)(kk + 2) * (kk + 1) / 2 <= b) ++kk;
        *k = kk;
        *l = (int)(b - (int64_t)kk * (kk + 1) / 2);
    }

    // Phase 1: X = the A (or V) tile, P = K_l, R = K_k (A tiles only).
    CK_HD void load(int64_t b, int t, double* X, double* P, double* R) const {
        int k, l, pk = 0, qk = 0, pl, ql;
        int64_t r0 = 0;
        if (b < tilesA) {
            tile_of(b, &k, &l);
            circle(nb, round, k, &pk, &qk);
        } else {
            const int64_t v = b - tilesA;
            l = (int)(v % groups());
            k = -1;
            r0 = v / groups() * kG;
        }
        circle(nb, round, l, &pl, &ql);
        const double* Jl = J + (int64_t)l * kG * kG;
        const double* Jk = J + (int64_t)(k < 0 ? 0 : k) * kG * kG;
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            const int64_t col = pair_index(pl, ql, y);
            X[x * kLd + y] = k < 0 ? V[(r0 + x) * N + col] : A[(int64_t)pair_index(pk, qk, x) * N + col];
            P[x * kLd + y] = Jl[e];
            if (k >= 0) R[x * kLd + y] = Jk[e];
        }
    }

    // Phase 2: acc = X + X K_l.
    CK_HD void right(int t, Acc& c, const double* X, const double* P) const {
        acc_load(c, t, X);
        tile_mma(c, t, X, kLd, 1, P);
    }
    // V tiles: write acc back.  A tiles: store acc (= X J_l) over X.
    CK_HD void after_right(int64_t b, int t, const Acc& c, double* X) const {
        const int row = acc_row(t);
        if (b >= tilesA) {
            const int64_t v = b - tilesA;
            const int l = (int)(v % groups());
            const int64_t r0 = v / groups() * kG;
            int pl, ql;
            circle(nb, round, l, &pl, &ql);
            for (int nt = 0; nt < 8; ++nt)
                for (int h = 0; h < 2; ++h) V[(r0 + row) * N + pair_index(pl, ql, acc_col(t, nt, h))] = c.v[nt][h];
            return;
        }
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) X[row * kLd + acc_col(t, nt, h)] = c.v[nt][h];
    }
    // Phase 3 (A tiles): acc = T + K_k^T T with T = X J_l, written to A[I_k, I_l] and A[I_l, I_k].
    CK_HD void left(int64_t b, int t, Acc& c, const double* X, const double* R) const {
        acc_load(c, t, X);
        tile_mma(c, t, R, 1, kLd, X);
        int k, l, pk, qk, pl, ql;
        tile_of(b, &k, &l);
        circle(nb, round, k, &pk, &qk);
        circle(nb, round, l, &pl, &ql);
        const int64_t gr = pair_index(pk, qk, acc_row(t));
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) {
                const int col = acc_col(t, nt, h);
                if (k == l && col > acc_row(t)) continue;   // the diagonal tile: its lower triangle, mirrored
                const int64_t gc = pair_index(pl, ql, col);
                A[gr * N + gc] = A[gc * N + gr] = c.v[nt][h];
            }
    }
};

// ---- dense product for M: C[N][N] = X^T Y (X, Y row-major N x N) -----------------------------------------------------
// Block (bi, bj) of (N / kG)^2 owns C's 64 x 64 tile and walks k in chunks of kG: stage both chunks, then the tile
// product.  Shared memory: two kG x kLd tiles.
struct GemmArgs {
    const double* X; const double* Y; double* C; int N;

    CK_HD void stage(int64_t b, int t, int k0, double* Xs, double* Ys) const {
        const int tn = N / kG, bi = (int)(b / tn), bj = (int)(b % tn);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int kk = e / kG, x = e % kG;
            Xs[kk * kLd + x] = X[(int64_t)(k0 + kk) * N + bi * kG + x];
            Ys[kk * kLd + x] = Y[(int64_t)(k0 + kk) * N + bj * kG + x];
        }
    }
    CK_HD void store(int64_t b, int t, const Acc& c) const {
        const int tn = N / kG, bi = (int)(b / tn), bj = (int)(b % tn);
        const int64_t r = (int64_t)bi * kG + acc_row(t);
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) C[r * N + bj * kG + acc_col(t, nt, h)] = c.v[nt][h];
    }
};

}  // namespace frechet

// Arithmetic of the Inception discriminative scores (ids.cu), written once for the device kernels and for the emulation
// build's host loops, the way frechet_kernels.cuh is.  Everything is float64, there are no atomics, and every sum has a
// fixed order, so a call returns the same bytes on every run and on every stream.
//
// The scores come from the linear SVM sklearn.svm.LinearSVC(dual=False) fits: rows x~_i = [x_i, 1] (D = d + 1), labels
// y_i = +1 for the real rows 0..n-1 and -1 for the fake rows n..2n-1, and
//     f(b) = 1/2 |b|^2 + C sum_i max(0, 1 - y_i b.x~_i)^2,   C = 1,
// minimised by the finite Newton method (Mangasarian 2002; Keerthi & DeCoste 2005).  One iteration at b_k:
//   margins      o = X~ b_k (row i: 32 lane partials over its columns, then the lanes in order)
//   active set   I = {i : y_i o_i < 1} as an index list, compacted by a chunked prefix scan
//   gradient     g = b_k - 2C X~_I^T (y - o)_I and r = 2C X~_I^T y_I (per column: chunks of rows, then the chunks)
//   Newton       G = I + 2C X~_I^T X~_I from its lower 64 x 64 tiles on fp64 mma.sync m8n8k4 (frechet::tile_mma, the
//                active rows read through the list, k in row order), D padded to Dp = a multiple of 64 with the
//                identity on the padded diagonal; blocked Cholesky G = L L^T (64-wide panels: diagonal block, panel
//                triangular solve, trailing update on the same DMMA tile); b~ = L^-T L^-1 r
//   stop         the active set at b~ is I: b~ is the minimiser.  Or |g| <= 1e-12 |g(0)|.
//   line search  exact, along d = b~ - b_k over t >= 0: phi'(t) is piecewise linear and non-decreasing; bisect until
//                no row changes sides inside the bracket, then solve that segment in closed form.
#pragma once
#include "frechet_kernels.cuh"

namespace ids {

using frechet::Acc;
using frechet::Accs;
using frechet::acc_col;
using frechet::acc_row;
using frechet::kG;
using frechet::kLd;
using frechet::kThreads;
using frechet::kTileDoubles;
using metrics::ddiv;

constexpr int kMaxDim = 4096;
constexpr int kChunk = 256;          // rows per chunk of the row reductions and of the gradient's column sums
constexpr int kLanes = 32;           // partial sums per row of a margin
constexpr double kTwoC = 2.0;        // 2C, C = 1
constexpr int kMaxBracket = 64;      // doublings of the line search's upper end
constexpr int kMaxBisect = 256;      // bisection steps of the line search (fp64 runs out of midpoints first)

// Slots of the status block (doubles) the host reads back.
enum Slot { kCount = 0, kGnorm2, kMismatch, kStep, kNonFinite, kPairs, kWrong, kHinge, kObjective, kSlots = 16 };

// The rows: real then fake, fp32 or fp64 as stored, promoted exactly to fp64.
struct Data {
    const void* real; const void* fake; int n, d, fp64;

    CK_HD int64_t rows() const { return 2 * (int64_t)n; }
    CK_HD double y(int64_t i) const { return i < n ? 1.0 : -1.0; }
    CK_HD double x(int64_t i, int c) const {
        const bool re = i < n;
        const int64_t e = (re ? i : i - n) * d + c;
        const void* p = re ? real : fake;
        return fp64 ? static_cast<const double*>(p)[e] : (double)static_cast<const float*>(p)[e];
    }
    // x~(i, c): the feature, 1 in column d, 0 in the padding.
    CK_HD double xt(int64_t i, int c) const { return c < d ? x(i, c) : (c == d ? 1.0 : 0.0); }
};

CK_HD int64_t chunks_of(int64_t rows) { return (rows + kChunk - 1) / kChunk; }
CK_HD bool active(double y, double o) { return dmul_rn(y, o) < 1.0; }

// b = k (k + 1) / 2 + l, l <= k: the lower tile (k, l).
CK_HD void lower_tile(int64_t b, int* k, int* l) {
    int kk = 0;
    while ((int64_t)(kk + 2) * (kk + 1) / 2 <= b) ++kk;
    *k = kk;
    *l = (int)(b - (int64_t)kk * (kk + 1) / 2);
}

// ---- item kernels ---------------------------------------------------------------------------------------------------
// v[i] = value.  items = len.
struct FillK {
    double* v; double value;
    CK_HD void operator()(int64_t i) const { v[i] = value; }
};

// part[c] = the non-finite features of chunk c's rows.  items = chunks.
struct NonFiniteK {
    Data X; double* part;
    CK_HD void operator()(int64_t c) const {
        double bad = 0.0;
        const int64_t end = X.rows() < (c + 1) * kChunk ? X.rows() : (c + 1) * kChunk;
        for (int64_t i = c * kChunk; i < end; ++i)
            for (int k = 0; k < X.d; ++k) {
                const double v = X.x(i, k);
                if (!(v - v == 0.0)) bad = dadd_rn(bad, 1.0);
            }
        part[c] = bad;
    }
};

// out[0] = sum of part[0..len) in order.  items = 1.
struct SumK {
    const double* part; double* out; int64_t len;
    CK_HD void operator()(int64_t) const {
        double s = 0.0;
        for (int64_t c = 0; c < len; ++c) s = dadd_rn(s, part[c]);
        out[0] = s;
    }
};

// part[c] = active rows of chunk c at margins o.  items = chunks.
struct ActiveCountK {
    Data X; const double* o; double* part;
    CK_HD void operator()(int64_t c) const {
        double k = 0.0;
        const int64_t end = X.rows() < (c + 1) * kChunk ? X.rows() : (c + 1) * kChunk;
        for (int64_t i = c * kChunk; i < end; ++i)
            if (active(X.y(i), o[i])) k = dadd_rn(k, 1.0);
        part[c] = k;
    }
};

// off[c] = the active rows before chunk c; scal[kCount] = all of them.  items = 1.
struct ScanK {
    const double* part; int* off; double* scal; int64_t chunks;
    CK_HD void operator()(int64_t) const {
        int s = 0;
        for (int64_t c = 0; c < chunks; ++c) {
            off[c] = s;
            s += (int)part[c];
        }
        scal[kCount] = (double)s;
    }
};

// idx[off[c] ...] = chunk c's active rows in order.  items = chunks.
struct ScatterK {
    Data X; const double* o; const int* off; int* idx;
    CK_HD void operator()(int64_t c) const {
        int k = off[c];
        const int64_t end = X.rows() < (c + 1) * kChunk ? X.rows() : (c + 1) * kChunk;
        for (int64_t i = c * kChunk; i < end; ++i)
            if (active(X.y(i), o[i])) idx[k++] = (int)i;
    }
};

// Column sums over chunk h of the active list: ps[h][c] = sum x~(i, c) (y_i - o_i), pt[h][c] = sum x~(i, c) y_i, rows in
// list order (0 past the list's end, count = scal[kCount]).  items = chunks(rows) * (d + 1), item = h * (d + 1) + c.
struct GradPartK {
    Data X; const double* o; const int* idx; const double* scal; int Dp; double* ps; double* pt;
    CK_HD void operator()(int64_t e) const {
        const int D = X.d + 1;
        const int64_t h = e / D, count = (int64_t)scal[kCount];
        const int c = (int)(e % D);
        const int64_t end = count < (h + 1) * kChunk ? count : (h + 1) * kChunk;
        double s = 0.0, t = 0.0;
        for (int64_t k = h * kChunk; k < end; ++k) {
            const int64_t i = idx[k];
            const double x = X.xt(i, c), y = X.y(i);
            s = fma(x, dsub_rn(y, o[i]), s);
            t = fma(x, y, t);
        }
        ps[h * Dp + c] = s;
        pt[h * Dp + c] = t;
    }
};

// g = b - 2C sum_h ps[h], r = 2C sum_h pt[h], chunks in order; 0 in the padding.  items = Dp.
struct GradK {
    const double* ps; const double* pt; const double* beta; double* g; double* r; int64_t chunks; int D, Dp;
    CK_HD void operator()(int64_t c) const {
        double s = 0.0, t = 0.0;
        if (c < D)
            for (int64_t h = 0; h < chunks; ++h) {
                s = dadd_rn(s, ps[h * Dp + c]);
                t = dadd_rn(t, pt[h * Dp + c]);
            }
        g[c] = c < D ? dsub_rn(beta[c], dmul_rn(kTwoC, s)) : 0.0;
        r[c] = c < D ? dmul_rn(kTwoC, t) : 0.0;
    }
};

// scal[kGnorm2] = |g|^2 in column order.  items = 1.
struct NormK {
    const double* g; double* scal; int D;
    CK_HD void operator()(int64_t) const {
        double s = 0.0;
        for (int c = 0; c < D; ++c) s = fma(g[c], g[c], s);
        scal[kGnorm2] = s;
    }
};

// part[i][lane] = sum over columns lane, lane + 32, ... < d of x(i, c) b[c].  items = rows * kLanes.
struct MarginPartK {
    Data X; const double* beta; double* part;
    CK_HD void operator()(int64_t e) const {
        const int64_t i = e / kLanes;
        const int lane = (int)(e % kLanes);
        double s = 0.0;
        for (int c = lane; c < X.d; c += kLanes) s = fma(X.x(i, c), beta[c], s);
        part[e] = s;
    }
};

// o[i] = the lanes of row i in order, plus the intercept b[d].  items = rows.
struct MarginK {
    const double* part; const double* beta; double* o; int d;
    CK_HD void operator()(int64_t i) const {
        double s = 0.0;
        for (int l = 0; l < kLanes; ++l) s = dadd_rn(s, part[i * kLanes + l]);
        o[i] = dadd_rn(s, beta[d]);
    }
};

// part[c] = the rows of chunk c on different sides of the margin at o and at ob.  items = chunks.
struct MismatchK {
    Data X; const double* o; const double* ob; double* part;
    CK_HD void operator()(int64_t c) const {
        double k = 0.0;
        const int64_t end = X.rows() < (c + 1) * kChunk ? X.rows() : (c + 1) * kChunk;
        for (int64_t i = c * kChunk; i < end; ++i)
            if (active(X.y(i), o[i]) != active(X.y(i), ob[i])) k = dadd_rn(k, 1.0);
        part[c] = k;
    }
};

// b <- b~ when no row changed sides (the next iteration stops there), else b + t (b~ - b).  items = Dp.
struct StepK {
    double* beta; const double* bbar; const double* scal;
    CK_HD void operator()(int64_t c) const {
        beta[c] = scal[kMismatch] == 0.0 ? bbar[c] : fma(scal[kStep], dsub_rn(bbar[c], beta[c]), beta[c]);
    }
};

// Per chunk of rows: part[3c] = sum of squared hinges, part[3c + 1] = misclassified rows (real o <= 0, fake o > 0),
// part[3c + 2] = pairs among the chunk's real rows whose fake decision value is above the real one.  items = chunks.
struct ScorePartK {
    Data X; const double* o; double* part;
    CK_HD void operator()(int64_t c) const {
        double h = 0.0, wrong = 0.0, pairs = 0.0;
        const int64_t end = X.rows() < (c + 1) * kChunk ? X.rows() : (c + 1) * kChunk;
        for (int64_t i = c * kChunk; i < end; ++i) {
            const double y = X.y(i), m = dsub_rn(1.0, dmul_rn(y, o[i]));
            if (m > 0.0) h = fma(m, m, h);
            if (i < X.n ? o[i] <= 0.0 : o[i] > 0.0) wrong = dadd_rn(wrong, 1.0);
            if (i < X.n && o[i + X.n] > o[i]) pairs = dadd_rn(pairs, 1.0);
        }
        part[3 * c] = h;
        part[3 * c + 1] = wrong;
        part[3 * c + 2] = pairs;
    }
};

// The chunks in order: scal[kPairs], scal[kWrong], scal[kHinge], scal[kObjective] = 1/2 |b|^2 + C hinges; coef = b[0..d).
// items = 1.
struct ScoreK {
    const double* part; const double* beta; double* scal; double* coef; int64_t chunks; int d;
    CK_HD void operator()(int64_t) const {
        double h = 0.0, wrong = 0.0, pairs = 0.0, bb = 0.0;
        for (int64_t c = 0; c < chunks; ++c) {
            h = dadd_rn(h, part[3 * c]);
            wrong = dadd_rn(wrong, part[3 * c + 1]);
            pairs = dadd_rn(pairs, part[3 * c + 2]);
        }
        for (int c = 0; c <= d; ++c) bb = fma(beta[c], beta[c], bb);
        for (int c = 0; c < d; ++c) coef[c] = beta[c];
        scal[kPairs] = pairs;
        scal[kWrong] = wrong;
        scal[kHinge] = h;
        scal[kObjective] = dadd_rn(dmul_rn(0.5, bb), h);   // C = 1
    }
};

// ---- Gram kernel: G = I + 2C X~_I^T X~_I, its lower tiles ------------------------------------------------------------
// Block b owns the lower tile (bi, bj) and walks the active list in chunks of kG rows: stage both 64-column panels of
// those rows (zero past the list's end, count = scal[kCount]), then the tile product.  Shared memory: two kG x kLd
// tiles.
struct GramArgs {
    Data X; const int* idx; const double* scal; int Dp; double* G;

    CK_HD int count() const { return (int)scal[kCount]; }

    CK_HD int64_t tiles() const {
        const int64_t nb = Dp / kG;
        return nb * (nb + 1) / 2;
    }
    CK_HD void stage(int64_t b, int t, int k0, double* Xs, double* Ys) const {
        int bi, bj;
        lower_tile(b, &bi, &bj);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int kk = e / kG, x = e % kG;
            double u = 0.0, v = 0.0;
            if (k0 + kk < count()) {
                const int64_t i = idx[k0 + kk];
                u = X.xt(i, bi * kG + x);
                v = X.xt(i, bj * kG + x);
            }
            Xs[kk * kLd + x] = u;
            Ys[kk * kLd + x] = v;
        }
    }
    CK_HD void store(int64_t b, int t, const Acc& c) const {
        int bi, bj;
        lower_tile(b, &bi, &bj);
        const int row = bi * kG + acc_row(t);
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) {
                const int col = bj * kG + acc_col(t, nt, h);
                if (col > row) continue;
                G[(int64_t)row * Dp + col] = dadd_rn(row == col ? 1.0 : 0.0, dmul_rn(kTwoC, c.v[nt][h]));
            }
    }
};

// ---- blocked Cholesky of the lower triangle, panel p -----------------------------------------------------------------
struct CholArgs {
    double* G; int Dp, p;

    CK_HD double* tile(int i, int j) const { return G + (int64_t)i * kG * Dp + (int64_t)j * kG; }

    // Diagonal block: right-looking unblocked Cholesky of the lower triangle of G[p, p] in shared memory S.
    CK_HD void diag_load(int t, double* S) const {
        const double* T = tile(p, p);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            S[x * kLd + y] = y <= x ? T[(int64_t)x * Dp + y] : 0.0;
        }
    }
    // Step j, phase 1: column j below the diagonal divided by sqrt(S[j][j]) (S[j][j] itself is left for phase 2).
    CK_HD void diag_scale(int j, int t, double* S) const {
        const double piv = frechet::dsqrt(S[j * kLd + j]);
        for (int i = j + 1 + t; i < kG; i += kThreads) S[i * kLd + j] = ddiv(S[i * kLd + j], piv);
    }
    // Step j, phase 2: S[j][j] = its square root; S[i][k] -= S[i][j] S[k][j] for j < k <= i.
    CK_HD void diag_update(int j, int t, double* S) const {
        if (t == 0) S[j * kLd + j] = frechet::dsqrt(S[j * kLd + j]);
        const int m = kG - j - 1;
        for (int e = t; e < m * m; e += kThreads) {
            const int i = j + 1 + e / m, k = j + 1 + e % m;
            if (k > i) continue;
            S[i * kLd + k] = fma(-S[i * kLd + j], S[k * kLd + j], S[i * kLd + k]);
        }
    }
    CK_HD void diag_store(int t, const double* S) const {
        double* T = tile(p, p);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            if (y <= x) T[(int64_t)x * Dp + y] = S[x * kLd + y];
        }
    }

    // Panel: block b solves L[p + 1 + b, p] = G[p + 1 + b, p] L[p, p]^-T, one row per thread, by forward substitution.
    CK_HD void panel_load(int b, int t, double* L, double* B) const {
        const double* Tl = tile(p, p);
        const double* Tb = tile(p + 1 + b, p);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            L[x * kLd + y] = y <= x ? Tl[(int64_t)x * Dp + y] : 0.0;
            B[x * kLd + y] = Tb[(int64_t)x * Dp + y];
        }
    }
    CK_HD void panel_solve(int t, const double* L, double* B) const {
        if (t >= kG) return;
        double* row = B + t * kLd;
        for (int j = 0; j < kG; ++j) {
            double x = row[j];
            for (int k = 0; k < j; ++k) x = fma(-row[k], L[j * kLd + k], x);
            row[j] = ddiv(x, L[j * kLd + j]);
        }
    }
    CK_HD void panel_store(int b, int t, const double* B) const {
        double* Tb = tile(p + 1 + b, p);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            Tb[(int64_t)x * Dp + y] = B[x * kLd + y];
        }
    }

    // Trailing update: block b = the lower tile (k, l) of the m = nb - p - 1 trailing tile rows, i = p + 1 + k,
    // j = p + 1 + l: G[i, j] -= L[i, p] L[j, p]^T on the DMMA tile, accumulators starting from G[i, j].
    // Shared memory: Xs = -L[i, p] (rows x k), Ys = L[j, p]^T (k x columns).
    CK_HD void trail_tiles(int64_t b, int* i, int* j) const {
        int k, l;
        lower_tile(b, &k, &l);
        *i = p + 1 + k;
        *j = p + 1 + l;
    }
    CK_HD void trail_stage(int64_t b, int t, double* Xs, double* Ys) const {
        int i, j;
        trail_tiles(b, &i, &j);
        const double* Li = tile(i, p);
        const double* Lj = tile(j, p);
        for (int e = t; e < kG * kG; e += kThreads) {
            const int x = e / kG, y = e % kG;
            Xs[x * kLd + y] = -Li[(int64_t)x * Dp + y];
            Ys[y * kLd + x] = Lj[(int64_t)x * Dp + y];
        }
    }
    CK_HD void trail_product(int64_t b, int t, Acc& c, const double* Xs, const double* Ys) const {
        int i, j;
        trail_tiles(b, &i, &j);
        const double* T = tile(i, j);
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) c.v[nt][h] = T[(int64_t)acc_row(t) * Dp + acc_col(t, nt, h)];
        frechet::tile_mma(c, t, Xs, kLd, 1, Ys);
    }
    CK_HD void trail_store(int64_t b, int t, const Acc& c) const {
        int i, j;
        trail_tiles(b, &i, &j);
        double* T = tile(i, j);
        const int row = acc_row(t);
        for (int nt = 0; nt < 8; ++nt)
            for (int h = 0; h < 2; ++h) {
                const int col = acc_col(t, nt, h);
                if (i == j && col > row) continue;
                T[(int64_t)row * Dp + col] = c.v[nt][h];
            }
    }
};

// ---- substitution: b~ = L^-T L^-1 r in one block -----------------------------------------------------------------
// Column-oriented: step j of the forward pass divides z[j] by L[j][j] (every thread, into w[j] by thread 0) and takes
// L[i][j] w[j] off z[i] for i > j; the backward pass does the same with L^T on w.  One barrier per step; z, w in shared
// memory.
struct SolveArgs {
    const double* L; const double* r; double* bbar; int Dp;

    CK_HD void load(int t, double* z) const {
        for (int i = t; i < Dp; i += kThreads) z[i] = r[i];
    }
    CK_HD void forward(int j, int t, double* z, double* w) const {
        const double zj = ddiv(z[j], L[(int64_t)j * Dp + j]);
        if (t == 0) w[j] = zj;
        for (int i = j + 1 + t; i < Dp; i += kThreads) z[i] = fma(-L[(int64_t)i * Dp + j], zj, z[i]);
    }
    CK_HD void backward(int j, int t, double* w) const {
        const double bj = ddiv(w[j], L[(int64_t)j * Dp + j]);
        if (t == 0) bbar[j] = bj;
        for (int i = t; i < j; i += kThreads) w[i] = fma(-L[(int64_t)j * Dp + i], bj, w[i]);
    }
};

// ---- exact line search along d = b~ - b in one block -----------------------------------------------------------------
// With a_i = 1 - y_i o_i and e_i = y_i (ob_i - o_i), row i is active at t when a_i - t e_i > 0, and
//     phi'(t) = b.d + t d.d - 2C sum_{active at t} e_i (a_i - t e_i) = P + t Q,
//     P = b.d - 2C sum a_i e_i,  Q = d.d + 2C sum e_i^2   (sums over the rows active at t).
// Every thread adds its rows (stride kThreads) into three partials; the partials are then summed in thread order.
struct LineArgs {
    Data X; const double* o; const double* ob; const double* beta; const double* bbar; double* scal; int Dp;

    CK_HD void dir_part(int t, double* part) const {
        double bd = 0.0, dd = 0.0;
        for (int c = t; c < Dp; c += kThreads) {
            const double dc = dsub_rn(bbar[c], beta[c]);
            bd = fma(beta[c], dc, bd);
            dd = fma(dc, dc, dd);
        }
        part[3 * t] = bd;
        part[3 * t + 1] = dd;
        part[3 * t + 2] = 0.0;
    }
    // Partials at `mid` of sum a e and sum e^2, and the rows on different sides at `lo` and `hi`.
    CK_HD void row_part(int t, double lo, double hi, double mid, double* part) const {
        double ae = 0.0, ee = 0.0, moved = 0.0;
        for (int64_t i = t; i < X.rows(); i += kThreads) {
            const double y = X.y(i);
            const double a = dsub_rn(1.0, dmul_rn(y, o[i])), e = dmul_rn(y, dsub_rn(ob[i], o[i]));
            if (dsub_rn(a, dmul_rn(mid, e)) > 0.0) {
                ae = fma(a, e, ae);
                ee = fma(e, e, ee);
            }
            if ((dsub_rn(a, dmul_rn(lo, e)) > 0.0) != (dsub_rn(a, dmul_rn(hi, e)) > 0.0)) moved = dadd_rn(moved, 1.0);
        }
        part[3 * t] = ae;
        part[3 * t + 1] = ee;
        part[3 * t + 2] = moved;
    }
};

CK_HD void sum_parts(const double* part, double s[3]) {
    s[0] = s[1] = s[2] = 0.0;
    for (int t = 0; t < kThreads; ++t) {
        s[0] = dadd_rn(s[0], part[3 * t]);
        s[1] = dadd_rn(s[1], part[3 * t + 1]);
        s[2] = dadd_rn(s[2], part[3 * t + 2]);
    }
}

// The line search's state machine; every thread of the block runs its own copy on the same sums.  Bracketing
// evaluates phi' at hi = 1, 2, 4, ... until it is >= 0; bisection then halves [lo, hi] until no row changes sides
// inside it, where phi' is P + t Q on the whole bracket and its root is -P / Q.
struct LineSearch {
    double bd, dd, lo, hi, t;
    int bisect, steps;

    CK_HD void start(const double dir[3]) {
        bd = dir[0];
        dd = dir[1];
        lo = 0.0;
        hi = 1.0;
        t = 1.0;
        bisect = 0;
        steps = 0;
    }
    CK_HD double mid() const { return bisect ? dmul_rn(0.5, dadd_rn(lo, hi)) : hi; }
    CK_HD double eval_lo() const { return bisect ? lo : hi; }
    // Takes the sums at (eval_lo(), hi, mid()); returns 1 when t is final.
    CK_HD int next(const double s[3]) {
        const double P = dsub_rn(bd, dmul_rn(kTwoC, s[0])), Q = dadd_rn(dd, dmul_rn(kTwoC, s[1]));
        if (!bisect) {
            if (fma(hi, Q, P) < 0.0 && steps < kMaxBracket) {
                lo = hi;
                hi = dmul_rn(2.0, hi);
                ++steps;
                return 0;
            }
            bisect = 1;
            steps = 0;
            return 0;
        }
        const double m = mid();
        if (s[2] == 0.0) {   // one segment: phi' = P + t Q on [lo, hi]
            t = Q > 0.0 ? -ddiv(P, Q) : lo;
            t = t < lo ? lo : (t > hi ? hi : t);
            return 1;
        }
        if (!(m > lo && m < hi) || steps >= kMaxBisect) {
            t = m;
            return 1;
        }
        if (fma(m, Q, P) < 0.0)
            lo = m;
        else
            hi = m;
        ++steps;
        return 0;
    }
};

}  // namespace ids

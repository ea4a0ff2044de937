// logistic.cuh — Spark 2.4's LogisticRegression over the feature matrix in HBM (lo_lr_stats, lo_lr_loss_grad;
// DESIGN.md §3.6.3).  Included by loexec.cu after naive_bayes.cuh, whose read-once loads it uses; the partials it writes
// are reduced by k_nb_reduce, and transform / evaluate run in k_nb_predict (its binomial epilogue is lr_sigmoid).
//   * k_lr_stats<T, PASS>: per-column sums of x (PASS kLrSum, with each column's min and max, the label histogram and
//     the refused cells) or of (x_j - mean_j)^2 (PASS kLrM2).
//   * k_lr_loss_grad<T, MULTI>: LogisticAggregator's loss and gradient sums at one point, one read of every row.
// Both add every sum in a fixed order, in per-thread runs of at most kLrCtaRows rows, with no floating-point atomics.
#pragma once

namespace lo {

constexpr int kLrThreads = 256;
constexpr int kLrCtaRows = 2048;            // rows of one CTA: no sequential run in a thread is longer
constexpr int kLrTileMax = 128;             // rows staged in shared memory at once
constexpr int kLrStatCols = 512;            // columns of one CTA of the stats passes (blockIdx.y picks the chunk)
constexpr int kLrHist = 1024;               // label bins (LO_NB_MAX_CLASSES); bin kLrHist counts the labels beyond
constexpr int kLrUnroll = 4;                // staging loads a thread keeps in flight
constexpr int kLrSmemMax = 227 * 1024;
constexpr int kLrMarginBlock = 4;           // classes whose margins one thread forms over one staged row
constexpr int kLrBlockC = 2;                // loss / grad: classes x columns of the sums one thread owns
constexpr int kLrBlockJ = 4;

enum { kLrSum = 0, kLrM2 = 1 };

// The launch shape lo_lr_stats / lo_lr_loss_grad choose from (k, classes, dtype) alone, so that the order of every sum,
// hence its bits, depends on the data and the shard layout only.
struct LrShape {
    int R;      // rows per tile, a power of two <= kLrTileMax (dividing kLrCtaRows)
    int G;      // row groups: thread (g, s) adds rows g, g + G, ... of each tile into sum s
    int S;      // sums of a CTA (stats: its chunk's columns; loss / grad: 1 + C' * (k + 1))
    int kc;     // columns staged per row (stats: kLrStatCols or k; loss / grad: k)
    int ks;     // staged row stride in doubles (kc or kc + 1: odd, so the threads' rows fall on different banks)
    int vw;     // values per load: 16 / sizeof(T) when every row is 16-byte aligned, else 1
    int nbj;    // loss / grad: column blocks of kLrBlockJ over k + 1 columns (column k: the intercept's 1.0)
    int nb;     // loss / grad: blocks of kLrBlockC x kLrBlockJ sums, plus one for the loss
    int cs;     // loss / grad: the coefficients staged in shared memory (else read from global memory)
};

// A double's order as a u64 (-0 below +0), so that integer atomicMin / atomicMax find a column's min and max
__device__ __forceinline__ unsigned long long lr_ordered(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return b >> 63 ? ~b : b | (1ull << 63);
}

// Spark's MLUtils.log1pExp
__device__ __forceinline__ double lr_log1p_exp(double v) { return v > 0.0 ? v + log1p(exp(-v)) : log1p(exp(v)); }

// Stage rows [t0, t0 + nr) x columns [j0, j0 + kw) into xs (f64, row stride ks): unit u = (row u / Q, 16-byte column
// group u % Q), kLrUnroll units' loads in flight before the first is stored.  SUM: the lowest non-finite cell's key.
template <typename T, int VW, bool CHECK>
__device__ __forceinline__ void lr_stage(const T *__restrict__ x, long long ld, int k, long long t0, int nr, int j0, int kw,
                                         int ks, double *xs, uint64_t pol, unsigned long long &bad) {
    const int Q = (kw + VW - 1) / VW, units = nr * Q;
    for (int u0 = threadIdx.x; u0 < units; u0 += kLrThreads * kLrUnroll) {
        double v[kLrUnroll][VW];
#pragma unroll
        for (int i = 0; i < kLrUnroll; ++i) {
            const int u = u0 + i * kLrThreads;
            if (u < units) {
                const int r = u / Q, q = u - r * Q;
                nb_load<T, VW>(x + (t0 + r) * ld + j0 + q * VW, pol, v[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < kLrUnroll; ++i) {
            const int u = u0 + i * kLrThreads;
            if (u >= units) continue;
            const int r = u / Q, q = u - r * Q;
#pragma unroll
            for (int w = 0; w < VW; ++w) {
                const int j = q * VW + w;
                if (j >= kw) continue;
                xs[r * ks + j] = v[i][w];
                if (CHECK && !isfinite(v[i][w])) bad = min(bad, cell_key(t0 + r, k, j0 + j));
            }
        }
    }
}

// One pass.  CTA (b, chunk) takes rows [row0 + b * kLrCtaRows, + kLrCtaRows) of [row0, row1) in tiles of R rows and, for
// the stats, columns [chunk * kc, + kc).  Per tile the rows are staged as f64.  Stats: thread (g, s) adds the tile's rows
// g, g + G, ... of term s (kLrSum x_j, kLrM2 (x_j - mean_j)^2) into its own acc[g][s] in shared memory.  Loss / grad:
// the staged row carries a 1.0 in column k; thread (row, block of kLrMarginBlock classes) forms the margins sum_j
// coef[c][j] x_j + icpt[c] (coefficients from shared memory when sh.cs), thread (row) turns its C' margins into
// LogisticAggregator's multipliers and loss, then thread (g, block) adds rows g, g + G, ... of the outer product
// multiplier_c x_j over its kLrBlockC x kLrBlockJ block of (class, column) sums, in registers over the tile, into its
// own acc[g][.] (one more block adds the loss).  Sum slots: 0 the loss, 1 + c k + j the multiplier_c x_j, 1 + C' k + c
// the multiplier_c (column k).  Every sum has one owner thread and a fixed row order.  At the end acc[0..G)[s] is added
// in g order into
// partial[b * pstride + chunk * kc + s].  kLrSum also keeps every (g, s)'s min and max of the column (in shared memory
// beside acc) and merges them per column into ext[j] (lr_ordered min) and ext[k + j] (max) by integer atomics, which
// are exact in any order, so a constant column is known as one whatever the sum's rounding; it also counts the labels (integer-valued, >= 0; bin kLrHist: >= kLrHist)
// into hist_out by integer atomics and gives the lowest refused cell's key to *err: a feature that is not finite, or a
// label (column k) that is NaN, infinite, negative or fractional.
template <typename T, int MODE>   // MODE: kLrSum, kLrM2, 2 + binomial / multinomial
__device__ __forceinline__ void lr_pass(const T *__restrict__ x, long long ld, int k, const T *__restrict__ y,
                                        long long row0, long long row1, const double *__restrict__ coef,
                                        const double *__restrict__ icpt, int nc, const double *__restrict__ mean,
                                        LrShape sh, double *__restrict__ partial, long long pstride,
                                        unsigned long long *__restrict__ hist_out, unsigned long long *__restrict__ ext,
                                        unsigned long long *__restrict__ err) {
    constexpr bool MODEL = MODE >= 2, MULTI = MODE == 3;
    extern __shared__ double lr_smem[];
    const int R = sh.R, G = sh.G, ks = sh.ks;
    const int j0 = blockIdx.y * sh.kc, kw = MODEL ? k : min(sh.kc, k - j0);
    const int S = MODEL ? sh.S : kw;
    const bool labels = MODEL || (MODE == kLrSum && blockIdx.y == 0);
    double *xs = lr_smem;                                          // [R][ks]
    double *ys = xs + (size_t)R * ks;                              // [R]
    double *mult = ys + R;                                         // [R][nc]: margins, then multipliers
    double *lossr = mult + (MODEL ? (size_t)R * nc : 0);           // [R]
    double *acc = lossr + (MODEL ? R : 0);                         // [G][sh.S]
    double *coef_s = acc + (size_t)G * sh.S;                       // [nc][k] (MODEL, sh.cs)
    double *lo = acc + (size_t)G * sh.S, *hi = lo + (size_t)G * sh.S;                // [G][sh.S] each (kLrSum)
    unsigned *hist = reinterpret_cast<unsigned *>(hi + (size_t)G * sh.S);       // [kLrHist + 1] (kLrSum)
    for (int i = threadIdx.x; i < G * sh.S; i += kLrThreads) acc[i] = 0.0;
    if (MODE == kLrSum) {
        for (int i = threadIdx.x; i < G * sh.S; i += kLrThreads) {
            lo[i] = INFINITY;
            hi[i] = -INFINITY;
        }
        for (int i = threadIdx.x; i <= kLrHist; i += kLrThreads) hist[i] = 0;
    }
    if (MODEL && sh.cs)
        for (int i = threadIdx.x; i < nc * k; i += kLrThreads) coef_s[i] = coef[i];
    const double *cf = MODEL && sh.cs ? coef_s : coef;
    const long long r0 = row0 + (long long)blockIdx.x * kLrCtaRows, r1 = min(row1, r0 + kLrCtaRows);
    const uint64_t pol = l2_evict_first_policy();
    unsigned long long bad = ~0ull;
    for (long long t0 = r0; t0 < r1; t0 += R) {
        const int nr = (int)min((long long)R, r1 - t0);
        __syncthreads();                                           // the previous tile's readers done (and the tables)
        if (sh.vw > 1) lr_stage<T, 16 / (int)sizeof(T), MODE == kLrSum>(x, ld, k, t0, nr, j0, kw, ks, xs, pol, bad);
        else           lr_stage<T, 1, MODE == kLrSum>(x, ld, k, t0, nr, j0, kw, ks, xs, pol, bad);
        if (labels)
            for (int r = threadIdx.x; r < nr; r += kLrThreads) {
                const double v = (double)y[t0 + r];
                ys[r] = v;
                if (MODEL) xs[r * ks + k] = 1.0;
                if (MODE == kLrSum) {
                    if (!(v >= 0.0 && isfinite(v) && floor(v) == v)) bad = min(bad, cell_key(t0 + r, k, k));
                    else atomicAdd(&hist[v < (double)kLrHist ? (int)v : kLrHist], 1u);
                }
            }
        __syncthreads();
        if (MODEL) {
            const int ncb = (nc + kLrMarginBlock - 1) / kLrMarginBlock;
            for (int p = threadIdx.x; p < nr * ncb; p += kLrThreads) {
                const int cb = p / nr, r = p - cb * nr, c0 = cb * kLrMarginBlock;
                const double *xr = xs + r * ks;
                const double *w[kLrMarginBlock];
                double m[kLrMarginBlock];
#pragma unroll
                for (int i = 0; i < kLrMarginBlock; ++i) {
                    w[i] = cf + (size_t)min(c0 + i, nc - 1) * k;
                    m[i] = 0.0;
                }
                for (int j = 0; j < k; ++j) {
                    const double xv = xr[j];
#pragma unroll
                    for (int i = 0; i < kLrMarginBlock; ++i) m[i] = fma(w[i][j], xv, m[i]);
                }
#pragma unroll
                for (int i = 0; i < kLrMarginBlock; ++i)
                    if (c0 + i < nc) mult[r * nc + c0 + i] = m[i] + __ldg(icpt + c0 + i);
            }
            __syncthreads();
            for (int r = threadIdx.x; r < nr; r += kLrThreads) {
                double *mr = mult + r * nc;
                const double label = ys[r];
                if (!MULTI) {                                      // binaryUpdateInPlace
                    const double margin = -mr[0];
                    mr[0] = 1.0 / (1.0 + exp(margin)) - label;
                    lossr[r] = label > 0.0 ? lr_log1p_exp(margin) : lr_log1p_exp(margin) - margin;
                } else {                                           // multinomialUpdateInPlace
                    double top = -INFINITY, of_label = 0.0, sum = 0.0;
                    for (int c = 0; c < nc; ++c) {
                        if ((double)c == label) of_label = mr[c];
                        if (mr[c] > top) top = mr[c];
                    }
                    for (int c = 0; c < nc; ++c) {
                        const double e = exp(top > 0.0 ? mr[c] - top : mr[c]);
                        mr[c] = e;
                        sum += e;
                    }
                    for (int c = 0; c < nc; ++c) mr[c] = mr[c] / sum - ((double)c == label ? 1.0 : 0.0);
                    lossr[r] = top > 0.0 ? log(sum) - of_label + top : log(sum) - of_label;
                }
            }
            __syncthreads();
            for (int u = threadIdx.x; u < G * sh.nb; u += kLrThreads) {     // the same (g, block) on every tile
                const int g = u / sh.nb, blk = u - g * sh.nb;
                double *ag = acc + (size_t)g * sh.S;
                if (blk == sh.nb - 1) {
                    double a = ag[0];
                    for (int r = g; r < nr; r += G) a += lossr[r];
                    ag[0] = a;
                    continue;
                }
                const int cb = blk / sh.nbj, c0 = cb * kLrBlockC, jc0 = (blk - cb * sh.nbj) * kLrBlockJ;
                int slot[kLrBlockC][kLrBlockJ], ci[kLrBlockC], ji[kLrBlockJ];
                double a[kLrBlockC][kLrBlockJ];
#pragma unroll
                for (int i = 0; i < kLrBlockC; ++i) ci[i] = min(c0 + i, nc - 1);
#pragma unroll
                for (int jj = 0; jj < kLrBlockJ; ++jj) ji[jj] = min(jc0 + jj, k);
#pragma unroll
                for (int i = 0; i < kLrBlockC; ++i)
#pragma unroll
                    for (int jj = 0; jj < kLrBlockJ; ++jj) {
                        const bool live = c0 + i < nc && jc0 + jj <= k;
                        slot[i][jj] = !live ? -1 : jc0 + jj < k ? 1 + (c0 + i) * k + jc0 + jj : 1 + nc * k + c0 + i;
                        a[i][jj] = live ? ag[slot[i][jj]] : 0.0;
                    }
                for (int r = g; r < nr; r += G) {
                    double mv[kLrBlockC], xv[kLrBlockJ];
#pragma unroll
                    for (int i = 0; i < kLrBlockC; ++i) mv[i] = mult[r * nc + ci[i]];
#pragma unroll
                    for (int jj = 0; jj < kLrBlockJ; ++jj) xv[jj] = xs[r * ks + ji[jj]];
#pragma unroll
                    for (int i = 0; i < kLrBlockC; ++i)
#pragma unroll
                        for (int jj = 0; jj < kLrBlockJ; ++jj) a[i][jj] = fma(mv[i], xv[jj], a[i][jj]);
                }
#pragma unroll
                for (int i = 0; i < kLrBlockC; ++i)
#pragma unroll
                    for (int jj = 0; jj < kLrBlockJ; ++jj)
                        if (slot[i][jj] >= 0) ag[slot[i][jj]] = a[i][jj];
            }
            continue;
        }
        for (int u = threadIdx.x; u < G * S; u += kLrThreads) {    // the same (g, s) for this thread on every tile
            const int g = u / S, s = u - g * S;
            double a = acc[g * sh.S + s];
            if (MODE == kLrSum) {
                double l = lo[g * sh.S + s], h = hi[g * sh.S + s];
                for (int r = g; r < nr; r += G) {
                    const double v = xs[r * ks + s];
                    a += v;
                    l = fmin(l, v);
                    h = fmax(h, v);
                }
                lo[g * sh.S + s] = l;
                hi[g * sh.S + s] = h;
            } else {
                const double mu = __ldg(mean + j0 + s);
                for (int r = g; r < nr; r += G) {
                    const double d = xs[r * ks + s] - mu;
                    a = fma(d, d, a);
                }
            }
            acc[g * sh.S + s] = a;
        }
    }
    if (MODE == kLrSum) report_cell(bad, err);
    __syncthreads();
    double *out = partial + (size_t)blockIdx.x * pstride + j0;
    for (int s = threadIdx.x; s < S; s += kLrThreads) {
        double v = acc[s];
        for (int g = 1; g < G; ++g) v += acc[g * sh.S + s];
        out[s] = v;
        if (MODE == kLrSum) {
            double l = lo[s], h = hi[s];
            for (int g = 1; g < G; ++g) {
                l = fmin(l, lo[g * sh.S + s]);
                h = fmax(h, hi[g * sh.S + s]);
            }
            atomicMin(&ext[j0 + s], lr_ordered(l));
            atomicMax(&ext[k + j0 + s], lr_ordered(h));
        }
    }
    if (MODE == kLrSum && blockIdx.y == 0)
        for (int i = threadIdx.x; i <= kLrHist; i += kLrThreads)
            if (hist[i]) atomicAdd(&hist_out[i], (unsigned long long)hist[i]);
}

template <typename T, int PASS>
__global__ void __launch_bounds__(kLrThreads) k_lr_stats(const T *__restrict__ x, long long ld, int k, const T *__restrict__ y,
                                                         long long row0, long long row1, const double *__restrict__ mean,
                                                         LrShape sh, double *__restrict__ partial,
                                                         unsigned long long *__restrict__ hist,
                                                         unsigned long long *__restrict__ ext,
                                                         unsigned long long *__restrict__ err) {
    lr_pass<T, PASS>(x, ld, k, y, row0, row1, nullptr, nullptr, 0, mean, sh, partial, k, hist, ext, err);
}

template <typename T, bool MULTI>
__global__ void __launch_bounds__(kLrThreads) k_lr_loss_grad(const T *__restrict__ x, long long ld, int k,
                                                             const T *__restrict__ y, long long row0, long long row1,
                                                             const double *__restrict__ coef, const double *__restrict__ icpt,
                                                             int nc, LrShape sh, double *__restrict__ partial) {
    lr_pass<T, MULTI ? 3 : 2>(x, ld, k, y, row0, row1, coef, icpt, nc, nullptr, sh, partial, sh.S, nullptr, nullptr, nullptr);
}

}  // namespace lo

// naive_bayes.cuh — Spark 2.4's multinomial NaiveBayes over the feature matrix in HBM (lo_nb_fit, lo_nb_predict;
// DESIGN.md §3.6.2).  Included by loexec.cu after kernels.cuh, whose streaming loads and refused-cell keys it uses.
//   * k_nb_sums + k_nb_reduce (fit): per-class row counts and f64 column sums of a row-major f32 / f64 matrix, reduced
//     in a fixed order and in bounded runs (no floating-point atomics), and the lowest row holding a negative or NaN
//     feature.
//   * k_nb_predict<T, EVAL> (transform / evaluate): per row raw_c = (sum_j theta_cj * x_j) + pi_c with every product
//     and add rounded on its own (F2J dgemv, no FMA), Spark's raw2probabilityInPlace and Vector.argmax; EVAL counts
//     (label slot, prediction) pairs instead of writing rows.
#pragma once

namespace lo {

constexpr int kNbMaxClasses = 1024;          // LO_NB_MAX_CLASSES
constexpr int kNbMaxTheta = 16384;           // LO_NB_MAX_THETA: C * k f64 = 128 KiB of shared memory
constexpr int kNbThreads = 256;              // k_nb_sums, k_nb_reduce
constexpr int kNbRun = 256;                  // rows a k_nb_sums thread adds in sequence into one sum
constexpr int kNbFan = 32;                   // partials one k_nb_reduce thread adds in sequence
constexpr long long kNbPartialBytes = 256ll << 20;   // k_nb_sums' partials per window of rows (lo_nb_fit)
constexpr int kNbSumsSmem = 100 * 1024;      // k_nb_sums' row-group copies beyond the first: two CTAs per SM
constexpr int kNbUnroll = 4;                 // rows whose loads a k_nb_sums thread keeps in flight
constexpr int kNbTile = 128;                 // rows per tile (and threads) of k_nb_predict
constexpr int kNbChunk = 32;                 // columns of a tile staged at once
constexpr int kNbBlock = 8;                  // classes per register block of the dot products
constexpr int kNbSmemMax = 227 * 1024;       // sm_90's opt-in shared memory per CTA

// The class of label value v in the ascending table cls[0 .. C): v itself when the classes are exactly 0 .. C-1
// (direct), else a binary search; -1 when v is none of them (NaN included).  -0.0 finds the class 0.0.
__device__ __forceinline__ int nb_class(double v, const double *cls, int C, bool direct) {
    if (direct) {
        if (!(v >= 0.0 && v < (double)C)) return -1;
        const int i = (int)v;
        return (double)i == v ? i : -1;
    }
    int lo = 0, hi = C;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cls[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo < C && cls[lo] == v ? lo : -1;
}

// The confusion counts of an evaluate pass (the EVAL form of k_nb_predict, k_dt_predict and k_gb_predict): CO
// predictions per label, NT threads per CTA.  The kernel places evl ([neval] f64) and hist ([neval][CO] u32) in its
// shared memory.  stage() copies eval_labels to evl and, with smem, zeroes hist; the kernel syncs before the first
// count.  count() adds a row's (label slot, prediction) to hist (smem) or straight to confusion, or keeps the lowest key
// cell_key(row, k, k) of a label that is not in eval_labels.  finish() reports that key to *err and flushes hist into
// confusion with integer atomics.
template <int NT>
struct Confusion {
    double *evl;
    unsigned *hist;
    unsigned long long *confusion;
    int neval, CO, direct, smem;
    unsigned long long bad = ~0ull;

    __device__ __forceinline__ void stage(const double *eval_labels) {
        for (int i = threadIdx.x; i < neval; i += NT) evl[i] = eval_labels[i];
        if (smem)
            for (int i = threadIdx.x; i < neval * CO; i += NT) hist[i] = 0;
    }
    __device__ __forceinline__ void count(double label, int p, long long row, int k) {
        const int a = nb_class(label, evl, neval, direct);
        if (a < 0) bad = min(bad, cell_key(row, k, k));
        else if (smem) atomicAdd(&hist[a * CO + p], 1u);
        else atomicAdd(&confusion[(size_t)a * CO + p], 1ull);
    }
    __device__ __forceinline__ void finish(unsigned long long *err) {
        report_cell(bad, err);
        if (smem) {
            __syncthreads();
            for (int i = threadIdx.x; i < neval * CO; i += NT)
                if (hist[i]) atomicAdd(&confusion[i], (unsigned long long)hist[i]);
        }
    }
};

// an LO_F32 label vector widened to f64 for the group-by of lo_nb_labels (exact)
__global__ void __launch_bounds__(256) k_nb_widen(const float *__restrict__ in, long long n, double *__restrict__ out) {
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) out[i] = (double)in[i];
}

template <typename T> __device__ __forceinline__ double nb_ld(const T *p, uint64_t pol);
template <> __device__ __forceinline__ double nb_ld<float>(const float *p, uint64_t pol) {
    return (double)__uint_as_float(ldg_u32_stream(p, pol));
}
template <> __device__ __forceinline__ double nb_ld<double>(const double *p, uint64_t pol) {
    return __longlong_as_double((long long)ldg_u64_stream(p, pol));
}

// VW values of one row from p: one 16-byte read-once load (VW = 16 / sizeof(T)) or one scalar load (VW = 1)
template <typename T, int VW>
__device__ __forceinline__ void nb_load(const T *p, uint64_t pol, double (&v)[VW]) {
    if constexpr (VW == 1) {
        v[0] = nb_ld(p, pol);
    } else {
        unsigned long long a, b;
        ldg_v2u64_stream(p, pol, a, b);
        if constexpr (sizeof(T) == 8) {
            v[0] = __longlong_as_double((long long)a);
            v[1] = __longlong_as_double((long long)b);
        } else {
            v[0] = (double)__uint_as_float((unsigned)a);
            v[1] = (double)__uint_as_float((unsigned)(a >> 32));
            v[2] = (double)__uint_as_float((unsigned)b);
            v[3] = (double)__uint_as_float((unsigned)(b >> 32));
        }
    }
}

// Fit, pass 1.  CTA b takes rows [row0 + b * G * kNbRun, + G * kNbRun) of [row0, row1).  Thread t owns units u = t,
// t + 256, ...: unit u is row group g = u / Q (rows g, g + G, ... of the CTA: kNbRun rows) and column group q = u % Q
// (columns q * VW .. + VW, one 16-byte load per row with VW = 16 / sizeof(T), else VW = 1).  Each row group adds its
// rows, in row order, into its own copy acc[g] of the C x k sums in shared memory, so no two threads ever add to one sum
// and no sum takes more than kNbRun adds here.  Column j of class c sits at c * kp + nb_col(j) of a copy: the one-double
// skew per 16 columns puts a warp's column groups on different banks, and the copy stride (= 2 mod 16 doubles) its row
// groups.  At the end the copies are added into partial[b][c * k + j] in runs of 16 (g order), the class counts go to
// counts[] by integer atomics, and the lowest key cell_key(row, k, j) of a feature that is not >= 0 (negative or NaN)
// or of a label that is no class (j = k) to *err.
__host__ __device__ __forceinline__ int nb_col(int j) { return j + (j >> 4); }

template <typename T, int VW>
__global__ void __launch_bounds__(kNbThreads) k_nb_sums(const T *__restrict__ x, long long ld, int k, const T *__restrict__ y,
                                                        long long row0, long long row1, const double *__restrict__ classes,
                                                        int C, int direct, int G, int Q, int kp, int stride,
                                                        double *__restrict__ partial, unsigned long long *__restrict__ counts,
                                                        unsigned long long *__restrict__ err) {
    extern __shared__ double nb_smem[];
    double *acc = nb_smem;
    double *cls = acc + (size_t)G * stride;
    unsigned *cnt = reinterpret_cast<unsigned *>(cls + C);
    for (int i = threadIdx.x; i < G * stride; i += kNbThreads) acc[i] = 0.0;
    for (int i = threadIdx.x; i < C; i += kNbThreads) { cls[i] = classes[i]; cnt[i] = 0; }
    __syncthreads();
    const long long r0 = row0 + (long long)blockIdx.x * G * kNbRun, r1 = min(row1, r0 + (long long)G * kNbRun);
    const uint64_t pol = l2_evict_first_policy();
    unsigned long long bad = ~0ull;
    for (int u = threadIdx.x; u < G * Q; u += kNbThreads) {
        const int g = u / Q, q = u - g * Q;
        double *mine = acc + (size_t)g * stride + nb_col(q * VW);
        for (long long r = r0 + g; r < r1; r += (long long)G * kNbUnroll) {
            double v[kNbUnroll][VW], lab[kNbUnroll];
#pragma unroll
            for (int i = 0; i < kNbUnroll; ++i) {           // every load of the batch in flight before the first is used
                const long long rr = r + (long long)i * G;
                if (rr < r1) {
                    nb_load<T, VW>(x + rr * ld + q * VW, pol, v[i]);
                    lab[i] = (double)y[rr];
                }
            }
#pragma unroll
            for (int i = 0; i < kNbUnroll; ++i) {
                const long long rr = r + (long long)i * G;
                if (rr >= r1) continue;
                const int c = nb_class(lab[i], cls, C, direct);
                if (c < 0) {
                    bad = min(bad, cell_key(rr, k, k));
                    continue;
                }
                if (q == 0) atomicAdd(&cnt[c], 1u);
                double *row = mine + c * kp;
#pragma unroll
                for (int w = 0; w < VW; ++w) {
                    const int j = q * VW + w;
                    if (j >= k) continue;
                    if (!(v[i][w] >= 0.0)) bad = min(bad, cell_key(rr, k, j));
                    row[w] += v[i][w];
                }
            }
        }
    }
    report_cell(bad, err);
    __syncthreads();
    double *out = partial + (size_t)blockIdx.x * C * k;
    for (int s = threadIdx.x; s < C * k; s += kNbThreads) {
        const int c = s / k, at = c * kp + nb_col(s - c * k);
        double sum = 0.0;
        for (int g0 = 0; g0 < G; g0 += 16) {
            double run = acc[(size_t)g0 * stride + at];
            for (int g = g0 + 1; g < min(G, g0 + 16); ++g) run += acc[(size_t)g * stride + at];
            sum = g0 == 0 ? run : sum + run;
        }
        out[s] = sum;
    }
    for (int c = threadIdx.x; c < C; c += kNbThreads)
        if (cnt[c]) atomicAdd(&counts[c], (unsigned long long)cnt[c]);
}

// Fit, pass 2, one level of a fixed-order tree: out[b][s] = in[32 b][s] + in[32 b + 1][s] + ... (at most kNbFan rows
// of m, in order).  lo_nb_fit repeats it until one row is left, so a sum takes at most kNbFan adds per level.
__global__ void __launch_bounds__(kNbThreads) k_nb_reduce(const double *__restrict__ in, long long m, int slots,
                                                          double *__restrict__ out) {
    const int s = blockIdx.x * kNbThreads + threadIdx.x;
    const long long b = blockIdx.y, end = min(m, (b + 1) * kNbFan);
    if (s >= slots) return;
    double sum = in[b * kNbFan * slots + s];
    for (long long i = b * kNbFan + 1; i < end; ++i) sum += in[i * slots + s];
    out[b * slots + s] = sum;
}

// NB classes' raw values of one row over one staged chunk: raw[b * kNbTile] (b < NB) plus theta_cj * x_j for the
// chunk's kc columns in ascending j, each product and each add rounded on its own.  th = thetaT + j0 * C + c0.
template <int NB>
__device__ __forceinline__ void nb_dot(const double *xrow, const double *th, int C, int kc, bool first, double *raw) {
    double a[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) a[b] = first ? 0.0 : raw[b * kNbTile];
    for (int j = 0; j < kc; ++j) {
        const double xv = xrow[j];
#pragma unroll
        for (int b = 0; b < NB; ++b) a[b] = __dadd_rn(a[b], __dmul_rn(th[j * C + b], xv));
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) raw[b * kNbTile] = a[b];
}

// Spark's raw2probabilityInPlace and Vector.argmax on one row's C raw values (raw[c * kNbTile]): m = the left fold
// max(m, r) as (m >= r ? m : r), e_c = exp(raw_c - m) summed in c order, p_c = e_c / sum, and the first c whose p_c
// is strictly greater than every earlier one.  raw[] receives the probabilities.  Out of line: the library's exp and
// its correctly rounded division are built on FMA, and the raw rule must not be (the SASS check on k_nb_predict).
__device__ __noinline__ int nb_softmax(double *raw, int C) {
    double m = raw[0];
    for (int c = 1; c < C; ++c) m = m >= raw[c * kNbTile] ? m : raw[c * kNbTile];
    double sum = 0.0;
    for (int c = 0; c < C; ++c) {
        const double e = exp(raw[c * kNbTile] - m);
        raw[c * kNbTile] = e;
        sum += e;
    }
    int best = 0;
    double top = 0.0;
    for (int c = 0; c < C; ++c) {
        const double p = raw[c * kNbTile] / sum;
        raw[c * kNbTile] = p;
        if (c == 0 || p > top) { best = c; top = p; }
    }
    return best;
}

// BinaryLogisticRegressionModel's raw2probabilityInPlace: p1 = 1 / (1 + exp(-m)) of the margin m (the binomial epilogue
// of k_nb_predict).  Out of line for the same reason as nb_softmax.
__device__ __noinline__ double lr_sigmoid(double m) { return 1.0 / (1.0 + exp(-m)); }

// LogisticRegressionModel's multinomial raw2probabilityInPlace and probability2prediction on one row's C raw values
// (raw[c * kNbTile]): m = the first greatest raw value (Vector.argmax); m == +inf gives probability 1 at its index and 0
// elsewhere; else e_c = exp(raw_c - m) when m > 0, exp(raw_c) otherwise, summed in c order, p_c = e_c * (1 / sum)
// (BLAS.scal), and the prediction is Vector.argmax(p).  raw[] receives the probabilities.  Out of line like nb_softmax.
__device__ __noinline__ int lr_softmax(double *raw, int C) {
    int at = 0;
    double m = raw[0];
    for (int c = 1; c < C; ++c)
        if (raw[c * kNbTile] > m) { m = raw[c * kNbTile]; at = c; }
    if (m == INFINITY) {
        for (int c = 0; c < C; ++c) raw[c * kNbTile] = c == at ? 1.0 : 0.0;
        return at;
    }
    double sum = 0.0;
    for (int c = 0; c < C; ++c) {
        const double e = exp(m > 0.0 ? raw[c * kNbTile] - m : raw[c * kNbTile]);
        raw[c * kNbTile] = e;
        sum += e;
    }
    const double inv = 1.0 / sum;
    int best = 0;
    double top = 0.0;
    for (int c = 0; c < C; ++c) {
        const double p = raw[c * kNbTile] * inv;
        raw[c * kNbTile] = p;
        if (c == 0 || p > top) { best = c; top = p; }
    }
    return best;
}

// Transform / evaluate.  A CTA of kNbTile threads holds thetaT (k x C, j-major) and pi in shared memory and takes tiles
// of kNbTile rows, one row per thread: chunks of kNbChunk columns are staged as f64 (row stride kNbChunk + 1, so the
// threads' rows fall on different banks), the raw values of classes c0 .. c0 + kNbBlock are carried in registers over a
// chunk and parked in raws (shared memory when it fits, else this CTA's slice of global scratch; [c * kNbTile + t]).
// !EVAL: raw (optional), probability and prediction of every row, with streaming stores.  EVAL: nothing per row; each
// row's (label, prediction) counts in a Confusion whose evl and hist follow the tables.  mode picks the epilogue
// (lo_lr_predict): kNbSoftmax NaiveBayes' nb_softmax; kLrBinomial (C = 1, theta the coefficients, pi the intercept) the
// one raw value m gives two outputs, raw [-m, m], probability [1 - p1, p1] with p1 = lr_sigmoid(m), and prediction p1 >
// threshold, with 2 confusion columns; kLrMultinomial lr_softmax.  A flag rather than a template parameter: the branch is uniform over the launch,
// and the tiling, staging and dot loop stay one copy per (T, EVAL).
enum { kNbSoftmax = 0, kLrBinomial = 1, kLrMultinomial = 2 };
template <typename T, bool EVAL>
__global__ void __launch_bounds__(kNbTile) k_nb_predict(const T *__restrict__ x, long long ld, int k, long long n,
                                                        const double *__restrict__ theta_t, const double *__restrict__ pi,
                                                        int C, double *__restrict__ prob, double *__restrict__ raw_out,
                                                        double *__restrict__ pred, const T *__restrict__ y,
                                                        const double *__restrict__ eval_labels, int neval, int direct,
                                                        unsigned long long *__restrict__ confusion,
                                                        double *__restrict__ raws_global, int hist_in_smem,
                                                        unsigned long long *__restrict__ err, int mode,
                                                        double threshold) {
    extern __shared__ double nb_smem[];
    const bool binomial = mode == kLrBinomial;
    const int CO = binomial ? 2 : C;                        // outputs per row
    double *th = nb_smem;                                   // [k][C]
    double *pis = th + (size_t)k * C;                       // [C]
    double *xt = pis + C;                                   // [kNbTile][kNbChunk + 1]
    double *evl = xt + kNbTile * (kNbChunk + 1);            // [neval] (EVAL)
    double *raws = raws_global ? raws_global + (size_t)blockIdx.x * C * kNbTile : evl + (EVAL ? neval : 0);
    unsigned *hist = reinterpret_cast<unsigned *>(evl + (EVAL ? neval : 0) + (raws_global ? 0 : (size_t)C * kNbTile));
    Confusion<kNbTile> cm{evl, hist, confusion, neval, CO, direct, hist_in_smem};
    for (int i = threadIdx.x; i < k * C; i += kNbTile) th[i] = theta_t[i];
    for (int i = threadIdx.x; i < C; i += kNbTile) pis[i] = pi[i];
    if (EVAL) cm.stage(eval_labels);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const uint64_t pol = l2_evict_first_policy();
    const long long ntiles = (n + kNbTile - 1) / kNbTile;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long row0 = tile * kNbTile;
        const int nr = (int)min((long long)kNbTile, n - row0);
        const bool live = t < nr;
        for (int j0 = 0; j0 < k; j0 += kNbChunk) {
            const int kc = min(kNbChunk, k - j0);
            __syncthreads();                                // the previous chunk (and the tables, at first) done
            for (int r = warp; r < nr; r += kNbTile / 32)
                if (lane < kc) xt[r * (kNbChunk + 1) + lane] = nb_ld(x + (row0 + r) * ld + j0 + lane, pol);
            __syncthreads();
            if (!live) continue;
            const double *xrow = xt + t * (kNbChunk + 1);
            for (int c0 = 0; c0 < C; c0 += kNbBlock) {
                const double *thc = th + (size_t)j0 * C + c0;
                double *rc = raws + (size_t)c0 * kNbTile + t;
                switch (min(kNbBlock, C - c0)) {
                    case 8: nb_dot<8>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 7: nb_dot<7>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 6: nb_dot<6>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 5: nb_dot<5>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 4: nb_dot<4>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 3: nb_dot<3>(xrow, thc, C, kc, j0 == 0, rc); break;
                    case 2: nb_dot<2>(xrow, thc, C, kc, j0 == 0, rc); break;
                    default: nb_dot<1>(xrow, thc, C, kc, j0 == 0, rc); break;
                }
            }
        }
        if (!live) continue;
        const long long row = row0 + t;
        double *rr = raws + t;
        for (int c = 0; c < C; ++c) {
            const double r = __dadd_rn(rr[c * kNbTile], pis[c]);
            rr[c * kNbTile] = r;
            if (!EVAL && raw_out && !binomial) __stcs(raw_out + row * C + c, r);
        }
        int p;
        if (binomial) {
            const double m = rr[0], p1 = lr_sigmoid(m);
            p = p1 > threshold ? 1 : 0;
            if (!EVAL) {
                if (raw_out) {
                    __stcs(raw_out + row * 2, -m);
                    __stcs(raw_out + row * 2 + 1, m);
                }
                __stcs(prob + row * 2, 1.0 - p1);
                __stcs(prob + row * 2 + 1, p1);
            }
        } else {
            p = mode == kLrMultinomial ? lr_softmax(rr, C) : nb_softmax(rr, C);
            if (!EVAL)
                for (int c = 0; c < C; ++c) __stcs(prob + row * C + c, rr[c * kNbTile]);
        }
        if (!EVAL) __stcs(pred + row, (double)p);
        else cm.count((double)y[row], p, row, k);
    }
    if (EVAL) cm.finish(err);
}

}  // namespace lo

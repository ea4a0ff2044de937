// tree.cuh — Spark 2.4's DecisionTreeClassifier and GBTClassifier over the feature matrix in HBM (lo_dt_sort,
// lo_dt_rank, lo_dt_bin, lo_dt_level, lo_dt_predict; lo_gb_level, lo_gb_update, lo_gb_predict; DESIGN.md §3.6.4-5).  Included by loexec.cu after naive_bayes.cuh, whose loads and class
// lookup it uses.
//   * k_dt_keys + CUB's radix sort + k_dt_distinct (split candidates): every column as sorted order-preserving codes
//     (-0.0 as 0.0), its count of distinct values and, when few, those values with their first positions.
//   * k_dt_rank: #(x < v) and #(x <= v) of probe codes v in the sorted columns, the step of the host's bisection.
//   * k_dt_bin: every value's bin, Java's Arrays.binarySearch of its column's thresholds as findBin reads it (without
//     equal thresholds, the count of thresholds < x), as a byte in an n x kp code matrix.
//   * k_dt_level: one tree level — routes every row by its node's split and counts (node, feature, bin, class); codes
//     >= nbins and labels outside [0, C) are refused, never counted.  k_gb_level: the same pass counting GBT's exact
//     fixed-point residual sums.
//   * k_dt_predict<T, EVAL>: walks the tree per row; raw = the leaf's class counts, probability = raw / sum.
//   * k_gb_update<T>: GBT's margins F and residuals r after each tree; k_gb_predict<T, EVAL>: the forest's margin.
//   * k_rf_level<T>: one level of a batch of RandomForest trees, each row counted with its bagging weight over its
//     node's feature subset; k_rf_predict<T, EVAL>: the forest's votes (lo_rf_level, lo_rf_predict, §3.6.6).
#pragma once

namespace lo {

constexpr int kDtMaxBins = 256;              // LO_DT_MAX_BINS: a bin index is a byte
constexpr int kDtMaxClasses = 100;           // LO_DT_MAX_CLASSES
constexpr int kDtThreads = 256;
constexpr int kDtVec = 16;                   // codes per 16-byte load, and the code matrix's row pitch granule
constexpr int kDtHistSmem = 112 * 1024;      // k_dt_level's histogram per CTA: two CTAs per SM
constexpr int kDtBinSmem = 96 * 1024;        // k_dt_bin's thresholds per CTA
constexpr int kDtTreeSmem = 96 * 1024;       // k_dt_predict's tree (and evaluation tables) in shared memory up to this
constexpr long long kDtPassHist = 1ll << 30; // LO_DT_PASS_HIST: bytes of one level pass's u64 histogram

// the order-preserving code of a finite value, -0.0 taken as 0.0: unsigned order of codes = order of values
__device__ __forceinline__ unsigned dt_code(float v) {
    const unsigned b = __float_as_uint(v == 0.0f ? 0.0f : v);
    return b >> 31 ? ~b : b | 0x80000000u;
}
__device__ __forceinline__ unsigned long long dt_code(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v);
    return b >> 63 ? ~b : b | (1ull << 63);
}
template <typename T> struct DtKey { using type = unsigned; };
template <> struct DtKey<double> { using type = unsigned long long; };

// keys[c * n + r] = dt_code(x[r][j0 + c]) for the kc columns from j0: one thread per cell, the row's cells adjacent
template <typename T>
__global__ void __launch_bounds__(kDtThreads) k_dt_keys(const T *__restrict__ x, long long ld, int j0, int kc, long long n,
                                                        typename DtKey<T>::type *__restrict__ keys) {
    const long long cells = n * kc;
    for (long long i = blockIdx.x * (long long)kDtThreads + threadIdx.x; i < cells; i += (long long)gridDim.x * kDtThreads) {
        const long long r = i / kc;
        const int c = (int)(i - r * kc);
        keys[(long long)c * n + r] = dt_code(x[r * ld + j0 + c]);
    }
}

// The distinct values of every sorted column (blockIdx.y): count[c] += the run starts (i == 0 or keys[i] != keys[i-1]);
// the first `cap` starts claimed (in no particular order) write their code and position to first_key / first_pos
// [c * cap + slot].  One atomic per CTA and pass.
template <typename K>
__global__ void __launch_bounds__(kDtThreads) k_dt_distinct(const K *__restrict__ keys, long long n, int cap,
                                                            unsigned long long *__restrict__ count,
                                                            unsigned long long *__restrict__ first_key,
                                                            long long *__restrict__ first_pos) {
    __shared__ unsigned wcnt[kDtThreads / 32];
    __shared__ unsigned long long base;
    const int c = blockIdx.y, t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const K *col = keys + (long long)c * n;
    for (long long i0 = blockIdx.x * (long long)kDtThreads; i0 < n; i0 += (long long)gridDim.x * kDtThreads) {
        const long long i = i0 + t;
        const bool start = i < n && (i == 0 || col[i] != col[i - 1]);
        const unsigned mask = __ballot_sync(0xffffffffu, start);
        if (lane == 0) wcnt[warp] = __popc(mask);
        __syncthreads();
        if (t == 0) {
            unsigned total = 0;
            for (int w = 0; w < kDtThreads / 32; ++w) { const unsigned m = wcnt[w]; wcnt[w] = total; total += m; }
            base = total ? atomicAdd(&count[c], (unsigned long long)total) : 0;
        }
        __syncthreads();
        if (start) {
            const unsigned long long slot = base + wcnt[warp] + __popc(mask & ((1u << lane) - 1));
            if (slot < (unsigned long long)cap) {
                first_key[(long long)c * cap + slot] = (unsigned long long)col[i];
                first_pos[(long long)c * cap + slot] = i;
            }
        }
        __syncthreads();
    }
}

// lt[i] = #(keys of column cols[i] < probe[i]), le[i] = #(<= probe[i]): two binary searches per probe
template <typename K>
__global__ void __launch_bounds__(kDtThreads) k_dt_rank(const K *__restrict__ keys, long long n, int m,
                                                        const int *__restrict__ cols,
                                                        const unsigned long long *__restrict__ probe,
                                                        long long *__restrict__ lt, long long *__restrict__ le) {
    const int i = blockIdx.x * kDtThreads + threadIdx.x;
    if (i >= m) return;
    const K *col = keys + (long long)cols[i] * n;
    const K v = (K)probe[i];
    long long a = 0, b = n;
    while (a < b) {
        const long long mid = (a + b) >> 1;
        if (col[mid] < v) a = mid + 1; else b = mid;
    }
    lt[i] = a;
    b = n;
    while (a < b) {
        const long long mid = (a + b) >> 1;
        if (col[mid] <= v) a = mid + 1; else b = mid;
    }
    le[i] = a;
}

// java.util.Arrays.binarySearch(t[0 .. m), x) as Spark's findBin reads it: the index the search lands on for a hit,
// else the insertion point -(ret) - 1.  Step for step Java's loop — mid = (low + high) >>> 1, `<` and `>` first, then
// the signed order of doubleToLongBits for values that compare equal — so that with equal adjacent thresholds (two
// midpoints that round to one double) the same one of them is hit.  Without duplicates both cases are the count of
// thresholds < x.
__device__ __forceinline__ int dt_bin(const double *t, int m, double x) {
    int low = 0, high = m - 1;
    const long long kb = __double_as_longlong(x);
    while (low <= high) {
        const int mid = (int)((unsigned)(low + high) >> 1);
        const double v = t[mid];
        if (v < x) {
            low = mid + 1;
        } else if (v > x) {
            high = mid - 1;
        } else {
            const long long vb = __double_as_longlong(v);
            if (vb == kb) return mid;
            if (vb < kb) low = mid + 1; else high = mid - 1;
        }
    }
    return low;
}

// Bin codes of columns [j0, j0 + kc) (j0 = blockIdx.y * kc, kc a multiple of 16): the chunk's thresholds (thr[j *
// tstride ..], nthr[j] of them) sit in shared memory; unit u = (row, column group of VW) reads VW values with one
// 16-byte read-once load (VW = 16 / sizeof(T); VW = 1: one scalar load) and writes their VW codes to codes[r * kp + j].
template <typename T, int VW>
__global__ void __launch_bounds__(kDtThreads) k_dt_bin(const T *__restrict__ x, long long ld, int k, long long n,
                                                       const double *__restrict__ thr, const int *__restrict__ nthr,
                                                       int tstride, int kc, unsigned char *__restrict__ codes, long long kp) {
    extern __shared__ double dt_smem[];
    int *ns = reinterpret_cast<int *>(dt_smem + (size_t)kc * tstride);
    const int j0 = blockIdx.y * kc, kw = min(kc, k - j0);
    for (int i = threadIdx.x; i < kw * tstride; i += kDtThreads) dt_smem[i] = thr[(size_t)j0 * tstride + i];
    for (int i = threadIdx.x; i < kw; i += kDtThreads) ns[i] = nthr[j0 + i];
    __syncthreads();
    const uint64_t pol = l2_evict_first_policy();
    const int Q = (kw + VW - 1) / VW;
    const long long units = n * Q;
    for (long long u = blockIdx.x * (long long)kDtThreads + threadIdx.x; u < units; u += (long long)gridDim.x * kDtThreads) {
        const long long r = u / Q;
        const int q = (int)(u - r * Q), c0 = q * VW;
        double v[VW];
        if (VW > 1 && c0 + VW <= kw) {
            nb_load<T, VW>(x + r * ld + j0 + c0, pol, v);
        } else {
#pragma unroll
            for (int w = 0; w < VW; ++w) v[w] = c0 + w < kw ? nb_ld(x + r * ld + j0 + c0 + w, pol) : 0.0;
        }
        unsigned char *out = codes + r * kp + j0 + c0;
#pragma unroll
        for (int w = 0; w < VW; ++w)
            if (c0 + w < kw) out[w] = (unsigned char)dt_bin(dt_smem + (size_t)(c0 + w) * tstride, ns[c0 + w], v[w]);
    }
}

// A row's slot at this level from its slot s at the previous one (k_dt_level, k_gb_level, k_rf_level): route, s sent by
// its split (sfeat[s] < 0: s is a leaf, so is the row: -1) to left[s] when the row's code of feature sfeat[s] is <=
// sbin[s], else right[s] (-1: a leaf child); !route, s itself.
__device__ __forceinline__ int dt_route(int s, int route, const unsigned char *row, const int *__restrict__ sfeat,
                                        const int *__restrict__ sbin, const int *__restrict__ left,
                                        const int *__restrict__ right) {
    if (route && s >= 0) {
        const int f = sfeat[s];
        s = f < 0 ? -1 : (int)row[f] <= sbin[s] ? left[s] : right[s];
    }
    return s;
}

// The leaf a row xr reaches from `node` (k_dt_predict, k_gb_update, k_gb_predict, k_rf_predict): an internal node (fe
// >= 0) sends it left when its value of feature fe[node] widened to f64 is <= th[node].
template <typename T>
__device__ __forceinline__ int dt_walk(const T *xr, int node, const int *fe, const double *th, const int *le,
                                       const int *ri) {
    int f;
    while ((f = fe[node]) >= 0) node = (double)xr[f] <= th[node] ? le[node] : ri[node];
    return node;
}

// A CTA's u32 counters hist[gn][fc][cell] into out[gn][kf][cell] (u64, integer atomics) from feature j0 of the kf
// (k_dt_level, k_rf_level): the fw features of its chunk, zero counters skipped.
__device__ __forceinline__ void dt_flush(const unsigned *hist, int cells, int fc, int cell, int fw, int kf, int j0,
                                         unsigned long long *__restrict__ out) {
    for (int i = threadIdx.x; i < cells; i += kDtThreads) {
        const unsigned v = hist[i];
        if (!v) continue;
        const int g = i / (fc * cell), rest = i - g * fc * cell, f = rest / cell;
        if (f >= fw) continue;
        atomicAdd(&out[((size_t)g * kf + j0 + f) * cell + (rest - f * cell)], (unsigned long long)v);
    }
}

// One pass of a tree level over every row.  A row's slot at this level: src == NULL, the root (0); else dt_route of
// src[r].  CTAs of blockIdx.y == 0 write the slot to dst (when given).  A row whose slot lies in the pass's node group [g0, g0 + gn)
// adds one to hist[slot - g0][f][code][class] for each feature f of the CTA's chunk [blockIdx.y * fc, + fc): u32
// counters in shared memory, flushed once per CTA into out ([gn][k][nbins][C], u64) with integer atomics.  VEC: the
// chunk's codes of a row in 16-byte loads (fc and the code pitch kp multiples of 16).  A code >= nbins or a label that
// is not a class in [0, C) is never counted: the lowest such cell's key (cell_key; col k: the label) goes to *err.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kDtThreads) k_dt_level(const unsigned char *__restrict__ codes, long long kp, int k,
                                                         const T *__restrict__ y, long long n, int nbins, int C,
                                                         const int *__restrict__ src, int route, int *__restrict__ dst,
                                                         const int *__restrict__ sfeat, const int *__restrict__ sbin,
                                                         const int *__restrict__ left, const int *__restrict__ right,
                                                         int g0, int gn, int fc, unsigned long long *__restrict__ out,
                                                         unsigned long long *__restrict__ err) {
    extern __shared__ unsigned dt_hist[];
    const int cell = nbins * C, j0 = blockIdx.y * fc, fw = min(fc, k - j0);
    const int cells = gn * fc * cell;
    for (int i = threadIdx.x; i < cells; i += kDtThreads) dt_hist[i] = 0;
    __syncthreads();
    const uint64_t pol = l2_evict_first_policy();
    const bool write = dst != nullptr && blockIdx.y == 0;
    unsigned long long bad = ~0ull;
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const unsigned char *row = codes + r * kp;
        const int s = src ? dt_route(src[r], route, row, sfeat, sbin, left, right) : 0;
        if (write) dst[r] = s;
        if (s < g0 || s >= g0 + gn) continue;
        const double lab = (double)y[r];
        const int cls = (int)lab;
        if (!(lab >= 0.0 && lab < (double)C) || (double)cls != lab) {   // not a class: refused, never counted
            bad = min(bad, cell_key(r, k, k));
            continue;
        }
        unsigned *h = dt_hist + (size_t)(s - g0) * fc * cell + cls;
        if constexpr (VEC) {
            for (int q = 0; q < fw; q += kDtVec) {
                unsigned long long a, b;
                ldg_v2u64_stream(row + j0 + q, pol, a, b);
#pragma unroll
                for (int w = 0; w < kDtVec; ++w) {
                    if (q + w >= fw) break;
                    const unsigned code = (unsigned)((w < 8 ? a >> (8 * w) : b >> (8 * (w - 8))) & 0xff);
                    if (code >= (unsigned)nbins) bad = min(bad, cell_key(r, k, j0 + q + w));
                    else atomicAdd(&h[(size_t)(q + w) * cell + code * C], 1u);
                }
            }
        } else {
            for (int w = 0; w < fw; ++w) {
                const unsigned code = row[j0 + w];
                if (code >= (unsigned)nbins) bad = min(bad, cell_key(r, k, j0 + w));
                else atomicAdd(&h[(size_t)w * cell + code * C], 1u);
            }
        }
    }
    report_cell(bad, err);
    __syncthreads();
    dt_flush(dt_hist, cells, fc, cell, fw, k, j0, out);
}

// GBT's regression sums per (node, feature, bin) (DESIGN.md §3.6.5): kGbWords u64 words, the count, Σ(q1 + 2^60) and
// Σq2 as 128-bit (lo, hi) pairs, with q1 = rint(r 2^58), q2 = rint(fl(r r) 2^58) of the row's residual r.  A 64-bit add
// carries into the hi word only when the lo word wraps, so every sum is exact in any order of the atomics.
constexpr int kGbWords = 5;                          // LO_GB_WORDS: count, Σ(q1 + 2^60) lo / hi, Σq2 lo / hi

// a residual's addends: |r| <= 4 (every residual of a fit) keeps q1 + 2^60 in [0, 2^61] and q2 in [0, 2^62]; NaN or
// anything larger is refused (false)
__device__ __forceinline__ bool gb_addends(double r, unsigned long long &q1, unsigned long long &q2) {
    if (!(fabs(r) <= 4.0)) return false;
    q1 = (unsigned long long)(__double2ll_rn(r * 0x1p58) + (1ll << 60));
    q2 = (unsigned long long)__double2ll_rn(__dmul_rn(r, r) * 0x1p58);
    return true;
}
__device__ __forceinline__ void add128(unsigned long long *lo, unsigned long long v) {
    const unsigned long long old = atomicAdd(lo, v);
    if (old + v < old) atomicAdd(lo + 1, 1ull);
}
// one row into a bin's words h (shared memory)
__device__ __forceinline__ void gb_add(unsigned long long *h, unsigned long long q1, unsigned long long q2) {
    atomicAdd(h, 1ull);
    add128(h + 1, q1);
    add128(h + 3, q2);
}
// a bin's words h (shared memory) into out (global memory), each 128-bit pair with the lo word's carry
__device__ __forceinline__ void gb_flush(unsigned long long *out, const unsigned long long *h) {
    atomicAdd(out, h[0]);
    for (int p = 1; p < kGbWords; p += 2) {
        const unsigned long long old = atomicAdd(out + p, h[p]);
        atomicAdd(out + p + 1, h[p + 1] + (old + h[p] < old ? 1ull : 0ull));
    }
}

// k_dt_level's pass counting GBT's sums: the same routing, refusals, launch shape and 16-byte code loads (DecisionTree
// keeps its own kernel, which stays as it was).  A row whose slot lies in the pass's node group adds its count and
// sums to hist[slot - g0][f][code][kGbWords] for each feature f of the CTA's chunk: u64 words in shared memory,
// flushed once per CTA into out ([gn][k][nbins][kGbWords]).  A code >= nbins or a refused residual (gb_addends) is
// never counted: the lowest such cell's key (cell_key; col k: the residual) goes to *err.  VEC does not unroll the 16
// codes of a 16-byte load: unrolled, the carry branches keep convergence state on the stack.
template <bool VEC>
__global__ void __launch_bounds__(kDtThreads) k_gb_level(const unsigned char *__restrict__ codes, long long kp, int k,
                                                         const double *__restrict__ res, long long n, int nbins,
                                                         const int *__restrict__ src, int route, int *__restrict__ dst,
                                                         const int *__restrict__ sfeat, const int *__restrict__ sbin,
                                                         const int *__restrict__ left, const int *__restrict__ right,
                                                         int g0, int gn, int fc, unsigned long long *__restrict__ out,
                                                         unsigned long long *__restrict__ err) {
    extern __shared__ unsigned long long gb_hist[];
    const int cell = nbins * kGbWords, j0 = blockIdx.y * fc, fw = min(fc, k - j0);
    const int cells = gn * fc * cell;
    for (int i = threadIdx.x; i < cells; i += kDtThreads) gb_hist[i] = 0;
    __syncthreads();
    const uint64_t pol = l2_evict_first_policy();
    const bool write = dst != nullptr && blockIdx.y == 0;
    unsigned long long bad = ~0ull;
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const unsigned char *row = codes + r * kp;
        const int s = src ? dt_route(src[r], route, row, sfeat, sbin, left, right) : 0;
        if (write) dst[r] = s;
        if (s < g0 || s >= g0 + gn) continue;
        unsigned long long q1, q2;
        if (!gb_addends(res[r], q1, q2)) {                 // refused: never counted
            bad = min(bad, cell_key(r, k, k));
            continue;
        }
        unsigned long long *h = gb_hist + (size_t)(s - g0) * fc * cell;
        if constexpr (VEC) {
            for (int q = 0; q < fw; q += kDtVec) {
                unsigned long long a, b;
                ldg_v2u64_stream(row + j0 + q, pol, a, b);
#pragma unroll 1
                for (int w = 0; w < kDtVec; ++w) {
                    if (q + w >= fw) break;
                    const unsigned code = (unsigned)((w < 8 ? a >> (8 * w) : b >> (8 * (w - 8))) & 0xff);
                    if (code >= (unsigned)nbins) bad = min(bad, cell_key(r, k, j0 + q + w));
                    else gb_add(&h[(size_t)(q + w) * cell + code * kGbWords], q1, q2);
                }
            }
        } else {
            for (int w = 0; w < fw; ++w) {
                const unsigned code = row[j0 + w];
                if (code >= (unsigned)nbins) bad = min(bad, cell_key(r, k, j0 + w));
                else gb_add(&h[(size_t)w * cell + code * kGbWords], q1, q2);
            }
        }
    }
    report_cell(bad, err);
    __syncthreads();
    for (int i = threadIdx.x * kGbWords; i < cells; i += kDtThreads * kGbWords) {
        if (!gb_hist[i]) continue;
        const int g = i / (fc * cell), rest = i - g * fc * cell, f = rest / cell;
        if (f >= fw) continue;
        gb_flush(&out[((size_t)g * k + j0 + f) * cell + (rest - f * cell)], gb_hist + i);
    }
}

// Transform / evaluate.  One row per thread: from node 0, an internal node (feat >= 0) sends the row left when its value
// widened to f64 is <= the node's threshold.  The leaf's class counts (counts[node * C ..]) are the raw values, the
// probabilities raw_c / sum (IEEE division, sum in c order) and the prediction their first argmax.  The tree's
// structure sits in shared memory when `tree_smem` (else it is read from global memory).  !EVAL: raw (optional),
// probability and prediction of every row with streaming stores.  EVAL: nothing per row; (label, prediction) counts in
// a Confusion (naive_bayes.cuh) whose evl and hist follow the tree.
template <typename T, bool EVAL>
__global__ void __launch_bounds__(kDtThreads) k_dt_predict(const T *__restrict__ x, long long ld, int k, long long n,
                                                           int M, const int *__restrict__ feat,
                                                           const double *__restrict__ thr, const int *__restrict__ left,
                                                           const int *__restrict__ right, const double *__restrict__ counts,
                                                           int C, int tree_smem, double *__restrict__ prob,
                                                           double *__restrict__ raw_out, double *__restrict__ pred,
                                                           const T *__restrict__ y, const double *__restrict__ eval_labels,
                                                           int neval, int direct, unsigned long long *__restrict__ confusion,
                                                           int hist_in_smem, unsigned long long *__restrict__ err) {
    extern __shared__ double dt_smem[];
    const double *th = thr;
    const int *fe = feat, *le = left, *ri = right;
    double *evl = dt_smem;
    if (tree_smem) {
        double *ts = dt_smem;
        int *fs = reinterpret_cast<int *>(ts + M);
        for (int i = threadIdx.x; i < M; i += kDtThreads) {
            ts[i] = thr[i];
            fs[i] = feat[i];
            fs[M + i] = left[i];
            fs[2 * M + i] = right[i];
        }
        th = ts;
        fe = fs;
        le = fs + M;
        ri = fs + 2 * M;
        evl = ts + M + (3 * M + 1) / 2;
    }
    Confusion<kDtThreads> cm{evl, reinterpret_cast<unsigned *>(evl + neval), confusion, neval, C, direct, hist_in_smem};
    if (EVAL) cm.stage(eval_labels);
    __syncthreads();
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const double *cnt = counts + (size_t)dt_walk(x + r * ld, 0, fe, th, le, ri) * C;
        double sum = 0.0;
        for (int c = 0; c < C; ++c) sum += cnt[c];
        int best = 0;
        double top = 0.0;
        for (int c = 0; c < C; ++c) {
            const double p = __ddiv_rn(cnt[c], sum);
            if (!EVAL) {
                __stcs(prob + r * C + c, p);
                if (raw_out) __stcs(raw_out + r * C + c, cnt[c]);
            }
            if (c == 0 || p > top) { best = c; top = p; }
        }
        if (!EVAL) __stcs(pred + r, (double)best);
        else cm.count((double)y[r], best, r, k);
    }
    if (EVAL) cm.finish(err);
}

// GBT's pass after each tree (DESIGN.md §3.6.5), one row per thread.  M == 0 initialises: F = 0, r = y' = 2y - 1.
// Else the row walks the tree (as k_dt_predict, on its raw values), F += value[leaf] * weight and r = -LogLoss.gradient
// = 4y' / (1 + exp(2y' F)), each operation rounded on its own (no fused multiply-add).  A label other than 0 or 1 is
// refused (cell_key(row, k, k) to *err) and its row left as it was.
template <typename T>
__global__ void __launch_bounds__(kDtThreads) k_gb_update(const T *__restrict__ x, long long ld, int k, long long n,
                                                          const T *__restrict__ y, int M, const int *__restrict__ feat,
                                                          const double *__restrict__ thr, const int *__restrict__ left,
                                                          const int *__restrict__ right, const double *__restrict__ value,
                                                          double weight, double *__restrict__ F, double *__restrict__ res,
                                                          unsigned long long *__restrict__ err) {
    unsigned long long bad = ~0ull;
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const double lab = (double)y[r];
        if (!(lab == 0.0 || lab == 1.0)) {
            bad = min(bad, cell_key(r, k, k));
            continue;
        }
        const double yp = lab == 1.0 ? 1.0 : -1.0;
        if (M == 0) {
            F[r] = 0.0;
            res[r] = yp;
            continue;
        }
        const int node = dt_walk(x + r * ld, 0, feat, thr, left, right);
        const double m = __dadd_rn(F[r], __dmul_rn(value[node], weight));
        F[r] = m;
        res[r] = __ddiv_rn(4.0 * yp, __dadd_rn(1.0, exp(__dmul_rn(2.0 * yp, m))));
    }
    report_cell(bad, err);
}

// GBT transform / evaluate, one row per thread: the margin m = sum over trees t (in order, from 0.0) of value[leaf_t] *
// weight[t], tree t's nodes from start[t] (children as indices into the whole forest).  raw = [-m, m], probability[0]
// = 1 / (1 + exp(2m)), probability[1] = 1 - probability[0], prediction = m > 0.  The forest sits in shared memory when
// `forest_smem` (else it is read from global memory).  EVAL: nothing per row; (label, prediction) counts in a
// Confusion, as in k_dt_predict.
template <typename T, bool EVAL>
__global__ void __launch_bounds__(kDtThreads) k_gb_predict(const T *__restrict__ x, long long ld, int k, long long n,
                                                           int ntrees, int M, const int *__restrict__ start,
                                                           const double *__restrict__ weight, const int *__restrict__ feat,
                                                           const double *__restrict__ thr, const int *__restrict__ left,
                                                           const int *__restrict__ right, const double *__restrict__ value,
                                                           int forest_smem, double *__restrict__ prob,
                                                           double *__restrict__ raw_out, double *__restrict__ pred,
                                                           const T *__restrict__ y, const double *__restrict__ eval_labels,
                                                           int neval, int direct, unsigned long long *__restrict__ confusion,
                                                           int hist_in_smem, unsigned long long *__restrict__ err) {
    extern __shared__ double dt_smem[];
    const double *th = thr, *va = value, *wt = weight;
    const int *fe = feat, *le = left, *ri = right, *st = start;
    double *evl = dt_smem;
    unsigned *hist_at = reinterpret_cast<unsigned *>(dt_smem + neval);
    if (forest_smem) {
        double *ts = dt_smem, *vs = ts + M, *ws = vs + M;
        evl = ws + ntrees;
        int *fs = reinterpret_cast<int *>(evl + neval), *ls = fs + M, *rs = ls + M, *ss = rs + M;
        for (int i = threadIdx.x; i < M; i += kDtThreads) {
            ts[i] = thr[i];
            vs[i] = value[i];
            fs[i] = feat[i];
            ls[i] = left[i];
            rs[i] = right[i];
        }
        for (int i = threadIdx.x; i < ntrees; i += kDtThreads) {
            ws[i] = weight[i];
            ss[i] = start[i];
        }
        th = ts, va = vs, wt = ws, fe = fs, le = ls, ri = rs, st = ss;
        hist_at = reinterpret_cast<unsigned *>(ss + ntrees);
    }
    Confusion<kDtThreads> cm{evl, hist_at, confusion, neval, 2, direct, hist_in_smem};
    if (EVAL) cm.stage(eval_labels);
    __syncthreads();
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        double m = 0.0;
        for (int t = 0; t < ntrees; ++t) m = __dadd_rn(m, __dmul_rn(va[dt_walk(x + r * ld, st[t], fe, th, le, ri)], wt[t]));
        const int best = m > 0.0 ? 1 : 0;
        if (!EVAL) {
            const double p0 = __ddiv_rn(1.0, __dadd_rn(1.0, exp(__dmul_rn(2.0, m))));
            __stcs(prob + 2 * r, p0);
            __stcs(prob + 2 * r + 1, __dsub_rn(1.0, p0));
            if (raw_out) {
                __stcs(raw_out + 2 * r, -m);
                __stcs(raw_out + 2 * r + 1, m);
            }
            __stcs(pred + r, (double)best);
        } else {
            cm.count((double)y[r], best, r, k);
        }
    }
    if (EVAL) cm.finish(err);
}

// ---- RandomForestClassifier (DESIGN.md §3.6.6) ----------------------------------------------------------------------
constexpr int kRfMaxDraws = 32;              // LO_RF_MAX_DRAWS: entries of a bagging threshold table
constexpr int kRfVotes = 8;                  // k_rf_predict's per-row votes held in registers per walk of the forest

// splitmix64's step: the golden-ratio increment, then its finaliser
__device__ __forceinline__ unsigned long long rf_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// A row's bagging weight in a tree: u = rf_mix(rf_mix(key ^ tree) ^ row) with key = rf_mix(seed), weight = #{j : u >=
// draw[j]} over the ascending table (so the count of its leading entries <= u)
__device__ __forceinline__ unsigned rf_weight(unsigned long long key, long long tree, long long row,
                                              const unsigned long long *draw, int ndraw) {
    const unsigned long long u = rf_mix(rf_mix(key ^ (unsigned long long)tree) ^ (unsigned long long)row);
    int w = 0;
    while (w < ndraw && u >= draw[w]) ++w;
    return (unsigned)w;
}

// One level of a batch of ntrees trees (global indices tree0 ..) over every row: k_dt_level's pass with each row's
// bagging weight and per-node feature subsets.  Row r's slot in tree t lives at src[t * n + r] (src NULL: the root, slot
// t), numbered across the batch in tree order, and is routed by its parent's split as in k_dt_level; CTAs of
// blockIdx.y == 0 write it to dst.  A (row, tree) whose slot lies in [g0, g0 + gn) and whose weight w (rf_weight of the
// global row row0 + r) is not 0 adds w to hist[slot - g0][q][code][class] for each q of the CTA's chunk [blockIdx.y * fc,
// + fc) of the node's m features feats[slot * m ..]: u32 counters in shared memory after the draw table, flushed once per
// CTA into out ([gn][m][nbins][C], u64).  A code >= nbins or a label that is not a class is never counted: the lowest
// such cell's key goes to *err.
template <typename T>
__global__ void __launch_bounds__(kDtThreads) k_rf_level(const unsigned char *__restrict__ codes, long long kp, int k,
                                                         const T *__restrict__ y, long long n, long long row0, int nbins,
                                                         int C, unsigned long long seed, int tree0, int ntrees,
                                                         const unsigned long long *__restrict__ draw, int ndraw,
                                                         const int *__restrict__ feats, int m, const int *__restrict__ src,
                                                         int route, int *__restrict__ dst, const int *__restrict__ sfeat,
                                                         const int *__restrict__ sbin, const int *__restrict__ left,
                                                         const int *__restrict__ right, int g0, int gn, int fc,
                                                         unsigned long long *__restrict__ out,
                                                         unsigned long long *__restrict__ err) {
    extern __shared__ unsigned long long rf_smem[];
    unsigned long long *dr = rf_smem;
    unsigned *hist = reinterpret_cast<unsigned *>(rf_smem + ndraw);
    const int cell = nbins * C, q0 = blockIdx.y * fc, fw = min(fc, m - q0);
    const int cells = gn * fc * cell;
    for (int i = threadIdx.x; i < ndraw; i += kDtThreads) dr[i] = draw[i];
    for (int i = threadIdx.x; i < cells; i += kDtThreads) hist[i] = 0;
    __syncthreads();
    const unsigned long long key = rf_mix(seed);
    const bool write = dst != nullptr && blockIdx.y == 0;
    unsigned long long bad = ~0ull;
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const unsigned char *row = codes + r * kp;
        const double lab = (double)y[r];
        const int cls = (int)lab;
        const bool is_class = lab >= 0.0 && lab < (double)C && (double)cls == lab;
        for (int t = 0; t < ntrees; ++t) {
            const int s = src ? dt_route(src[t * n + r], route, row, sfeat, sbin, left, right) : t;
            if (write) dst[t * n + r] = s;
            if (s < g0 || s >= g0 + gn) continue;
            const unsigned w = rf_weight(key, (long long)tree0 + t, row0 + r, dr, ndraw);
            if (!w) continue;
            if (!is_class) {                                    // not a class: refused, never counted
                bad = min(bad, cell_key(r, k, k));
                continue;
            }
            unsigned *h = hist + (size_t)(s - g0) * fc * cell + cls;
            const int *fl = feats + (size_t)s * m + q0;
            for (int q = 0; q < fw; ++q) {
                const int f = __ldg(fl + q);
                const unsigned code = row[f];
                if (code >= (unsigned)nbins) bad = min(bad, cell_key(r, k, f));
                else atomicAdd(&h[(size_t)q * cell + code * C], w);
            }
        }
    }
    report_cell(bad, err);
    __syncthreads();
    dt_flush(hist, cells, fc, cell, fw, m, q0, out);
}

// RandomForest transform / evaluate, one row per thread: raw_c = the sum over trees t (in order, from 0.0) of
// votes[leaf_t * C + c], the leaf's class counts over their total as the host computed them (0 for a leaf of no
// counts); probability = raw / sum (IEEE division, sum in c order), prediction = the first argmax of raw.  Tree t's
// nodes start at start[t] (children as indices into the whole forest).  The votes are kept in registers kRfVotes
// classes at a time, the forest walked once per such group; with C above kRfVotes the raw values wait in the row's
// probability slice until the sum is known.  The forest (structure and votes) sits in shared memory when `forest_smem`
// (else it is read from global memory).  EVAL: nothing per row; (label, prediction) counts in a Confusion, as in
// k_dt_predict.
template <typename T, bool EVAL>
__global__ void __launch_bounds__(kDtThreads) k_rf_predict(const T *__restrict__ x, long long ld, int k, long long n,
                                                           int ntrees, int M, const int *__restrict__ start,
                                                           const int *__restrict__ feat, const double *__restrict__ thr,
                                                           const int *__restrict__ left, const int *__restrict__ right,
                                                           const double *__restrict__ votes, int C, int forest_smem,
                                                           double *__restrict__ prob, double *__restrict__ raw_out,
                                                           double *__restrict__ pred, const T *__restrict__ y,
                                                           const double *__restrict__ eval_labels, int neval, int direct,
                                                           unsigned long long *__restrict__ confusion, int hist_in_smem,
                                                           unsigned long long *__restrict__ err) {
    extern __shared__ double dt_smem[];
    const double *th = thr, *vo = votes;
    const int *fe = feat, *le = left, *ri = right, *st = start;
    double *evl = dt_smem;
    unsigned *hist_at = reinterpret_cast<unsigned *>(dt_smem + neval);
    if (forest_smem) {
        double *ts = dt_smem, *vs = ts + M;
        evl = vs + (size_t)M * C;
        int *fs = reinterpret_cast<int *>(evl + neval), *ls = fs + M, *rs = ls + M, *ss = rs + M;
        for (int i = threadIdx.x; i < M; i += kDtThreads) {
            ts[i] = thr[i];
            fs[i] = feat[i];
            ls[i] = left[i];
            rs[i] = right[i];
        }
        for (int i = threadIdx.x; i < M * C; i += kDtThreads) vs[i] = votes[i];
        for (int i = threadIdx.x; i < ntrees; i += kDtThreads) ss[i] = start[i];
        th = ts, vo = vs, fe = fs, le = ls, ri = rs, st = ss;
        hist_at = reinterpret_cast<unsigned *>(ss + ntrees);
    }
    Confusion<kDtThreads> cm{evl, hist_at, confusion, neval, C, direct, hist_in_smem};
    if (EVAL) cm.stage(eval_labels);
    __syncthreads();
    for (long long r = blockIdx.x * (long long)kDtThreads + threadIdx.x; r < n; r += (long long)gridDim.x * kDtThreads) {
        const T *xr = x + r * ld;
        double sum = 0.0, top = 0.0;
        int best = 0;
        for (int c0 = 0; c0 < C; c0 += kRfVotes) {
            double v[kRfVotes];
#pragma unroll
            for (int i = 0; i < kRfVotes; ++i) v[i] = 0.0;
            for (int t = 0; t < ntrees; ++t) {
                const double *lv = vo + (size_t)dt_walk(xr, st[t], fe, th, le, ri) * C + c0;
#pragma unroll
                for (int i = 0; i < kRfVotes; ++i)
                    if (c0 + i < C) v[i] = __dadd_rn(v[i], lv[i]);
            }
#pragma unroll
            for (int i = 0; i < kRfVotes; ++i) {
                const int c = c0 + i;
                if (c < C) {
                    sum = __dadd_rn(sum, v[i]);
                    if (c == 0 || v[i] > top) { best = c; top = v[i]; }
                    if (!EVAL && raw_out) __stcs(raw_out + r * C + c, v[i]);
                    if (!EVAL && C > kRfVotes) prob[r * C + c] = v[i];
                }
            }
            if (!EVAL && C <= kRfVotes) {
#pragma unroll
                for (int i = 0; i < kRfVotes; ++i)
                    if (i < C) __stcs(prob + r * C + i, __ddiv_rn(v[i], sum));
            }
        }
        if (!EVAL) {
            if (C > kRfVotes)
                for (int c = 0; c < C; ++c) prob[r * C + c] = __ddiv_rn(prob[r * C + c], sum);
            __stcs(pred + r, (double)best);
        } else {
            cm.count((double)y[r], best, r, k);
        }
    }
    if (EVAL) cm.finish(err);
}

}  // namespace lo

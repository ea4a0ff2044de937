// loexec.cu — host side of libloexec.so: the C ABI declared in include/loexec.h.
//
// Nothing here computes on the CPU: every entry point either moves bytes or launches the
// sm_90a kernels in kernels.cuh.  There is no fallback path; without a Hopper device
// lo_init() fails and nothing else is callable.
#include "loexec.h"
#include "kernels.cuh"
#include "naive_bayes.cuh"
#include "logistic.cuh"
#include "tree.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <array>
#include <atomic>
#include <condition_variable>
#include <cctype>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    // a failed runtime call also stays this thread's "last error" until read; read it here, or the next call's
    // cudaGetLastError() after a launch would report it as its own (sticky errors of a broken context are unaffected)
    (void)cudaGetLastError();
    return code;
}

#define LO_CUDA(call)                                                                        \
    do {                                                                                     \
        cudaError_t e_ = (call);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            int code_ = (e_ == cudaErrorMemoryAllocation) ? LO_ERR_NOMEM : LO_ERR_CUDA;      \
            return fail(code_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),       \
                        __FILE__, __LINE__);                                                 \
        }                                                                                    \
    } while (0)

#define LO_TRY(call)                 \
    do {                             \
        int rc_ = (call);            \
        if (rc_ != LO_OK) return rc_; \
    } while (0)

size_t dtype_size(int dtype) {
    switch (dtype) {
        case LO_F64: return 8;
        case LO_F32: return 4;
        case LO_U8:  return 1;
        case LO_U32: return 4;
        case LO_I32: return 4;
        default:     return 0;
    }
}

}  // namespace

struct lo_table {
    int       dtype;
    int64_t   nrows;
    int32_t   ncols;
    int64_t   pitch;   // bytes between column slabs
    char     *base;
    bool      owned;
    int       device;
};

constexpr int kSlots = 3;      // staging slots of the *_host pipeline: H2D of chunk c+1/c+2 overlaps kernel c and D2H c-1
constexpr int kMaxStageSets = 4;

struct StageSet {
    cudaStream_t compute = nullptr, h2d = nullptr, d2h = nullptr;
    char        *in[kSlots]  = {nullptr, nullptr, nullptr};
    char        *out[kSlots] = {nullptr, nullptr, nullptr};
    size_t       in_bytes = 0, out_bytes = 0;
    unsigned long long *counts = nullptr;
    size_t       counts_n = 0;
    cudaEvent_t  ev_h2d[kSlots] = {}, ev_k[kSlots] = {}, ev_d2h[kSlots] = {};
};

// One device bin-edge table of the EDGES tile kernels: k x (nbins + 1) floats, E[0] = lo, E[1 .. nbins-1],
// E[nbins] = nextup(hi) per column.  Uploaded on the context's edge stream; every launch that reads it waits for `ready`
// and records an event in `uses`, so a retired table is freed in stream order after its last reader.
struct EdgeTable {
    int32_t            nbins = 0;
    std::vector<float> lo, hi;
    float             *dev = nullptr;
    size_t             bytes = 0;
    cudaEvent_t        ready = nullptr;
    std::vector<cudaEvent_t> uses;      // launches that read the table and may still be running
    uint64_t           last_use = 0;
};
constexpr int kEdgeTables = 8;          // tables cached per context (least recently used one retired first)

struct lo_ctx {
    int          device;
    int          sm_count;
    size_t       hbm_bytes;
    cudaStream_t stream;       // default stream for NULL `stream` arguments
    std::atomic<int64_t> launches{0};
    // *_host pipelines: each call borrows a StageSet (its own three streams, staging slots, events, count scratch)
    // from this pool, so concurrent calls on one context — the REST services run a thread per job — overlap instead
    // of queueing; at most kMaxStageSets exist, further callers wait for one to come back
    std::mutex   pool_mu;
    std::condition_variable pool_cv;
    std::vector<StageSet *> free_sets;
    int          nsets = 0;
    // bin-edge tables of the EDGES tile kernels, one per (nbins, lo[], hi[]) of a launch, at most kEdgeTables; edge_mu
    // is held from the lookup until the launch that reads the table has recorded its event
    std::mutex   edge_mu;
    cudaStream_t edge_stream = nullptr;
    std::vector<std::unique_ptr<EdgeTable>> edge_tables;
    uint64_t     edge_tick = 0;
    std::atomic<int64_t> divide_launches{0};   // tile-kernel launches that binned with the IEEE divide (w outside the window)
};

namespace {

cudaStream_t pick(lo_ctx *ctx, void *stream) { return stream ? (cudaStream_t)stream : ctx->stream; }

int check_ctx(const lo_ctx *ctx) {
    if (!ctx) return fail(LO_ERR_INVALID, "ctx is NULL");
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) return fail(LO_ERR_CUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
    return LO_OK;
}

// after n kernel launches on this thread: the launch error, or count them on the context
cudaError_t launched(lo_ctx *ctx, int n) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) ctx->launches.fetch_add(n, std::memory_order_relaxed);
    return e;
}

bool aligned32(const lo_table *t) {
    return ((uintptr_t)t->base % 32 == 0) && (t->pitch % 32 == 0);
}

int check_cols(const lo_table *in, const int32_t *col_idx, int32_t k) {
    if (k <= 0) return fail(LO_ERR_INVALID, "k must be > 0 (got %d)", k);
    if (!col_idx) return fail(LO_ERR_INVALID, "col_idx is NULL");
    for (int j = 0; j < k; ++j)
        if (col_idx[j] < 0 || col_idx[j] >= in->ncols)
            return fail(LO_ERR_INVALID, "col_idx[%d] = %d outside [0, %d)", j, col_idx[j], in->ncols);
    return LO_OK;
}

int check_spec(const lo_hist_spec *spec, int32_t k, float *w_out /* k */) {
    if (spec->nbins < 1 || spec->nbins > LO_MAX_BINS)
        return fail(LO_ERR_INVALID, "nbins = %d outside [1, %d]", spec->nbins, LO_MAX_BINS);
    if (spec->flags != 0) return fail(LO_ERR_INVALID, "unknown lo_hist_spec.flags 0x%x", spec->flags);
    if (!spec->lo || !spec->hi) return fail(LO_ERR_INVALID, "lo_hist_spec.lo / .hi is NULL");
    for (int j = 0; j < k; ++j) {
        const float lo = spec->lo[j], hi = spec->hi[j];
        // w = (hi - lo) / nbins in fp32 round-to-nearest, exactly as the oracle computes it
        volatile float span = hi - lo;
        volatile float w    = span / (float)spec->nbins;
        if (!(std::isfinite(lo) && std::isfinite(hi)) || !(hi > lo) || !std::isfinite(w) || !(w > 0.0f))
            return fail(LO_ERR_INVALID, "histogram range of column %d is not usable: lo=%g hi=%g nbins=%d",
                        j, (double)lo, (double)hi, spec->nbins);
        w_out[j] = w;
    }
    return LO_OK;
}

template <typename K>
int allow_smem(K kernel, int bytes) {
    LO_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    return LO_OK;
}

template <int OUT>
int allow_smem_hist() {
    LO_TRY(allow_smem(lo::k_project_cast_hist<OUT, true, true, true>, lo::kEdgeSmemBytes));
    LO_TRY(allow_smem(lo::k_project_cast_hist<OUT, true, true, false>, lo::kHistSmemBytes));
    LO_TRY(allow_smem(lo::k_project_cast_hist<OUT, true, false, true>, lo::kEdgeSmemBytes));
    LO_TRY(allow_smem(lo::k_project_cast_hist<OUT, true, false, false>, lo::kHistSmemBytes));
    return LO_OK;
}

// The branch-free divide of the FASTDIV kernels equals the IEEE quotient only under the
// conditions of Markstein's theorem (kernels.cuh, bin_index_f32): the divisor's significand must
// not be all ones, and w, 1/w and every quotient (<= nbins) must stay far from the exponent limits.
bool fastdiv_ok(float w) {
    uint32_t bits;
    memcpy(&bits, &w, 4);
    if ((bits & 0x007FFFFFu) == 0x007FFFFFu) return false;
    return w >= 0x1p-100f && w <= 0x1p100f;
}

// The edge-table kernels need r = RN(1/w) and r * 2^-9 normal (kernels.cuh, edge_counter_offset).
bool edges_ok(float w) { return w >= 0x1p-100f && w <= 0x1p100f; }

// host twin of bin_index_f32<false> for f in [lo, hi]: fp32 RN subtract, fp32 RN divide, truncate, close the last bin
int bin_ieee_host(float f, float lo, float w, int last) {
    volatile float d = f - lo;
    volatile float q = d / w;
    const int i = (int)q;
    return i < last ? i : last;
}

// fp32 <-> integer keys in value order (-0 and +0 share key 0)
int32_t f32_key(float f) {
    int32_t b;
    memcpy(&b, &f, 4);
    return b >= 0 ? b : -(b & 0x7FFFFFFF);
}
float key_f32(int32_t k) {
    const uint32_t b = k >= 0 ? (uint32_t)k : (0x80000000u | (uint32_t)(-(int64_t)k));
    float f;
    memcpy(&f, &b, 4);
    return f;
}

// E[0] = lo; E[i] = the smallest fp32 f in [lo, hi] with bin(f) >= i (nextup(hi) when no such f exists: bins i.. are
// empty); E[nbins] = nextup(hi).  w as check_spec computes it.  Search over the ordered keys: start at lo + i*w, gallop
// outwards until the edge is bracketed (a few ulps as a rule), then bisect; every answer is checked by the bracket
// itself, the estimate only decides how fast it is found.
void hist_edges(float lo, float hi, float w, int32_t nbins, float *E) {
    const int last = nbins - 1;
    const int64_t khi = f32_key(hi);
    const float above = std::nextafter(hi, INFINITY);
    auto at_or_above = [&](int64_t k, int32_t i) { return bin_ieee_host(key_f32((int32_t)k), lo, w, last) >= i; };
    E[0] = lo;
    int64_t floor_k = f32_key(lo);                         // every key below it bins below i (edges ascend)
    for (int32_t i = 1; i < nbins; ++i) {
        if (!at_or_above(khi, i)) { E[i] = above; continue; }
        const int64_t g = std::min(khi, std::max(floor_k, (int64_t)f32_key((float)((double)lo + (double)i * w))));
        int64_t a, b;                                      // invariant: key a bins below i (or a < floor_k), b at/above
        if (at_or_above(g, i)) {
            b = g;
            for (int64_t step = 1;; step *= 2) {
                a = b - step;
                if (a < floor_k) { a = floor_k - 1; break; }
                if (!at_or_above(a, i)) break;
                b = a;
            }
        } else {
            a = g;
            for (int64_t step = 1;; step *= 2) {
                b = a + step;
                if (b >= khi) { b = khi; break; }
                if (at_or_above(b, i)) break;
                a = b;
            }
        }
        while (b - a > 1) {
            const int64_t m = a + (b - a) / 2;
            if (at_or_above(m, i)) b = m; else a = m;
        }
        E[i] = key_f32((int32_t)b);
        floor_k = b;
    }
    E[nbins] = above;
}

// Free a table in stream order: the edge stream waits for every launch that read it (and, by stream order, for its
// upload), then frees it.  No host wait.
void edge_retire(lo_ctx *ctx, EdgeTable *t) {
    for (cudaEvent_t e : t->uses) {
        cudaStreamWaitEvent(ctx->edge_stream, e, 0);
        cudaEventDestroy(e);
    }
    t->uses.clear();
    if (t->ready) cudaEventDestroy(t->ready);
    if (t->dev) cudaFreeAsync(t->dev, ctx->edge_stream);
    t->ready = nullptr;
    t->dev = nullptr;
}

// The edge table of P's columns for a launch on stream s (ctx->edge_mu held by the caller until edge_used): cached, or
// built now in place of the least recently used one.  *out = nullptr when a width is outside the window (IEEE kernels).
int edge_acquire(lo_ctx *ctx, const lo::ColsF64 &P, cudaStream_t s, EdgeTable **out) {
    *out = nullptr;
    for (int j = 0; j < P.k; ++j)
        if (!edges_ok(P.w[j])) return LO_OK;
    EdgeTable *t = nullptr;
    for (const auto &c : ctx->edge_tables)
        if (c->nbins == P.nbins && (int)c->lo.size() == P.k && std::equal(c->lo.begin(), c->lo.end(), P.lo) &&
            std::equal(c->hi.begin(), c->hi.end(), P.hi)) {
            t = c.get();
            break;
        }
    if (!t) {
        if ((int)ctx->edge_tables.size() >= kEdgeTables) {
            auto lru = std::min_element(ctx->edge_tables.begin(), ctx->edge_tables.end(),
                                        [](const auto &x, const auto &y) { return x->last_use < y->last_use; });
            edge_retire(ctx, lru->get());
            ctx->edge_tables.erase(lru);
        }
        auto nt = std::make_unique<EdgeTable>();
        nt->nbins = P.nbins;
        nt->lo.assign(P.lo, P.lo + P.k);
        nt->hi.assign(P.hi, P.hi + P.k);
        const size_t n = (size_t)P.k * (P.nbins + 1);
        nt->bytes = n * 4;
        std::vector<float> h(n);
        for (int j = 0; j < P.k; ++j) hist_edges(P.lo[j], P.hi[j], P.w[j], P.nbins, h.data() + (size_t)j * (P.nbins + 1));
        // pageable source: the copy has taken the host bytes when it returns; `ready` marks its arrival on the device
        cudaError_t e = cudaMallocAsync((void **)&nt->dev, nt->bytes, ctx->edge_stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(nt->dev, h.data(), nt->bytes, cudaMemcpyHostToDevice, ctx->edge_stream);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&nt->ready, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(nt->ready, ctx->edge_stream);
        if (e != cudaSuccess) {
            edge_retire(ctx, nt.get());
            return fail(e == cudaErrorMemoryAllocation ? LO_ERR_NOMEM : LO_ERR_CUDA, "edge table upload: %s",
                        cudaGetErrorString(e));
        }
        t = nt.get();
        ctx->edge_tables.push_back(std::move(nt));
    }
    LO_CUDA(cudaStreamWaitEvent(s, t->ready, 0));
    t->last_use = ++ctx->edge_tick;
    *out = t;
    return LO_OK;
}

// after a launch on s that reads t: remember it (and forget the readers that have finished)
int edge_used(EdgeTable *t, cudaStream_t s) {
    t->uses.erase(std::remove_if(t->uses.begin(), t->uses.end(), [](cudaEvent_t e) {
                      if (cudaEventQuery(e) != cudaSuccess) return false;
                      cudaEventDestroy(e);
                      return true;
                  }), t->uses.end());
    (void)cudaGetLastError();       // cudaEventQuery's cudaErrorNotReady is not an error of this call
    cudaEvent_t e = nullptr;
    LO_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    const cudaError_t r = cudaEventRecord(e, s);
    if (r != cudaSuccess) {
        cudaEventDestroy(e);
        return fail(LO_ERR_CUDA, "edge table use: %s", cudaGetErrorString(r));
    }
    t->uses.push_back(e);
    return LO_OK;
}

int configure_kernels() {
    LO_TRY(allow_smem_hist<0>());
    LO_TRY(allow_smem_hist<1>());
    LO_TRY(allow_smem_hist<2>());
    LO_CUDA(cudaFuncSetAttribute(lo::k_hist_u8_cols_lanes<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kU8LSmemBytes));
    LO_CUDA(cudaFuncSetAttribute(lo::k_hist_u8_cols_lanes<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kU8LSmemBytes));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    LO_CUDA(cudaFuncSetAttribute(lo::k_project_cast_hist_bins<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kWBSmemWordsMax * 4));
    return LO_OK;
}

const lo::GroupStep kNoGroup = {};     // mode 0

// <<<>>> with one optional launch attribute: programmatic stream serialization lets THIS launch's CTAs start as soon
// as every CTA of the previous launch in the stream has called griddepcontrol.launch_dependents (or exited) instead
// of after its last CTA has drained (overlapped group steps, LO_GROUP_INDEPENDENT)
template <typename... KArgs, typename... Args>
cudaError_t launch_kernel(void (*kernel)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t s, bool overlap,
                          Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = overlap ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// one launch of the fused kernel over <= kMaxColsF64 projected columns
template <int OUT, bool HIST>
int launch_f64(lo_ctx *ctx, const lo_table *in, const lo_table *out, int32_t out_col0,
               const lo::ColsF64 &P, unsigned long long *counts, bool aligned, const lo::GroupStep &G, cudaStream_t s) {
    std::unique_lock<std::mutex> edge_lock(ctx->edge_mu, std::defer_lock);
    EdgeTable *et = nullptr;
    if (HIST) {
        edge_lock.lock();
        LO_TRY(edge_acquire(ctx, P, s, &et));
        if (!et) {
            edge_lock.unlock();
            ctx->divide_launches.fetch_add(1, std::memory_order_relaxed);
        }
    }
    const float *edges = et ? et->dev : nullptr;
    const size_t smem = !HIST ? 0 : edges ? lo::kEdgeSmemBytes : lo::kHistSmemBytes;
    char *out_base = out ? out->base + (int64_t)out_col0 * out->pitch : nullptr;
    const long long out_pitch = out ? out->pitch : 0;
    // one tile (kTileRows rows of one projected column) per CTA.  A tapered tail — the last wave cut into short
    // tiles — was built and was not faster, and a runtime tile shape slows the uniform case, so tiles are compile-time
    // uniform.
    const unsigned tiles_per_col = (unsigned)((in->nrows + lo::kTileRows - 1) / lo::kTileRows);
    const unsigned long long blocks = (unsigned long long)tiles_per_col * (unsigned)P.k;
    if (blocks > 0x7fffffffull) return fail(LO_ERR_INVALID, "table too large for one launch (%llu tiles)", blocks);
    const char *ib = in->base;
    const long long ip = in->pitch, nr = in->nrows;
#define LO_LAUNCH(AL, ED)                                                                                        \
    LO_CUDA(launch_kernel(lo::k_project_cast_hist<OUT, HIST, AL, ED>, (unsigned)blocks, lo::kThreads, smem, s,    \
                          G.overlap != 0, ib, ip, out_base, out_pitch, nr, tiles_per_col, counts, edges, P, G))
    if (aligned) { if (edges) LO_LAUNCH(true, true); else LO_LAUNCH(true, false); }
    else         { if (edges) LO_LAUNCH(false, true); else LO_LAUNCH(false, false); }
#undef LO_LAUNCH
    LO_CUDA(launched(ctx, 1));
    if (et) LO_TRY(edge_used(et, s));
    return LO_OK;
}

// histograms wider than the byte-counter tile kernel holds (LO_TILE_BINS < nbins <= LO_MAX_BINS): k_project_cast_hist_bins
template <int OUT>
int launch_f64_bins(lo_ctx *ctx, const lo_table *in, const lo_table *out, int32_t out_col0,
                    const lo::ColsF64 &P, unsigned long long *counts, bool aligned, const lo::GroupStep &G, cudaStream_t s) {
    char *out_base = out ? out->base + (int64_t)out_col0 * out->pitch : nullptr;
    const long long out_pitch = out ? out->pitch : 0;
    bool fast = true;
    for (int j = 0; j < P.k; ++j) fast = fast && fastdiv_ok(P.w[j]);
    int slots_log2 = -1;                                  // counters in shared memory while one slot per bin fits 224 KiB
    if (P.nbins <= lo::kWBSmemWords) {
        slots_log2 = 0;
        while (slots_log2 < 5 && (P.nbins << (slots_log2 + 1)) <= lo::kWBSmemWords) ++slots_log2;
    } else if (P.nbins <= lo::kWBSmemWordsMax) {
        slots_log2 = 0;
    }
    const size_t smem = slots_log2 >= 0 ? (size_t)(P.nbins << slots_log2) * 4 : 16;
    // chunk of a column per CTA: ~4 waves of CTAs (2 resident per SM), whole loop rounds, 32-bit counters cannot wrap
    const int64_t slots = (int64_t)ctx->sm_count * 2;
    int64_t want = (in->nrows * (int64_t)P.k) / (4 * slots);
    want = std::max<int64_t>(lo::kWBRoundRows, std::min<int64_t>(want, (int64_t)1 << 24));
    const int64_t chunk_rows = (want / lo::kWBRoundRows) * lo::kWBRoundRows;
    const unsigned chunks_per_col = (unsigned)((in->nrows + chunk_rows - 1) / chunk_rows);
    const unsigned long long blocks = (unsigned long long)chunks_per_col * (unsigned)P.k;
    if (blocks > 0x7fffffffull) return fail(LO_ERR_INVALID, "table too large for one launch (%llu chunks)", blocks);
    const char *ib = in->base;
    const long long ip = in->pitch, nr = in->nrows;
    if (fast) LO_CUDA(launch_kernel(lo::k_project_cast_hist_bins<OUT, true>, (unsigned)blocks, (unsigned)lo::kWBThreads, smem, s, G.overlap != 0,
                                    ib, ip, out_base, out_pitch, nr, chunks_per_col, (long long)chunk_rows, slots_log2, (int)aligned, counts, P, G));
    else      LO_CUDA(launch_kernel(lo::k_project_cast_hist_bins<OUT, false>, (unsigned)blocks, (unsigned)lo::kWBThreads, smem, s, G.overlap != 0,
                                    ib, ip, out_base, out_pitch, nr, chunks_per_col, (long long)chunk_rows, slots_log2, (int)aligned, counts, P, G));
    LO_CUDA(launched(ctx, 1));
    return LO_OK;
}

// the argument checks of project_cast_hist_impl, which enqueue nothing; w receives the bin widths when there is a spec
int check_project_cast_hist(const lo_table *in, const int32_t *col_idx, int32_t k, const lo_table *out,
                            const lo_hist_spec *spec, const uint64_t *counts_dev, bool group, std::vector<float> &w) {
    if (!in) return fail(LO_ERR_INVALID, "input table is NULL");
    if (in->dtype != LO_F64) return fail(LO_ERR_INVALID, "input table must be LO_F64 (got dtype %d)", in->dtype);
    LO_TRY(check_cols(in, col_idx, k));
    if (out) {
        if (out->dtype != LO_F32 && out->dtype != LO_F64)
            return fail(LO_ERR_INVALID, "output table must be LO_F32 or LO_F64 (got dtype %d)", out->dtype);
        if (out->nrows != in->nrows) return fail(LO_ERR_INVALID, "output rows %lld != input rows %lld",
                                                  (long long)out->nrows, (long long)in->nrows);
        if (out->ncols < k) return fail(LO_ERR_INVALID, "output has %d columns, need %d", out->ncols, k);
        if (out->device != in->device) return fail(LO_ERR_INVALID, "tables live on different devices");
    }
    if (!out && !spec) return fail(LO_ERR_INVALID, "nothing to do: no output table and no histogram spec");
    if (spec) {
        if (!counts_dev) return fail(LO_ERR_INVALID, "counts_dev is NULL");
        w.resize(k);
        LO_TRY(check_spec(spec, k, w.data()));
    }
    if (group && (!spec || k > lo::kMaxColsF64))
        return fail(LO_ERR_INVALID, "a group step needs a histogram spec and k <= %d (got %d)", lo::kMaxColsF64, k);
    return LO_OK;
}

int project_cast_hist_impl(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                           lo_table *out, const lo_hist_spec *spec, uint64_t *counts_dev, cudaStream_t s,
                           const lo::GroupStep *group = nullptr) {
    std::vector<float> w;
    LO_TRY(check_project_cast_hist(in, col_idx, k, out, spec, counts_dev, group != nullptr, w));
    if (in->nrows == 0 && !group) return LO_OK;
    const int out_mode = !out ? 0 : out->dtype == LO_F32 ? 1 : 2;
    const bool aligned = aligned32(in) && (!out || aligned32(out));
    const lo::GroupStep &G = group ? *group : kNoGroup;

    for (int32_t c0 = 0; c0 < k; c0 += lo::kMaxColsF64) {
        lo::ColsF64 P;
        P.k     = std::min<int32_t>(lo::kMaxColsF64, k - c0);
        P.nbins = spec ? spec->nbins : 0;
        for (int j = 0; j < P.k; ++j) {
            P.col[j] = col_idx[c0 + j];
            P.lo[j]  = spec ? spec->lo[c0 + j] : 0.f;
            P.hi[j]  = spec ? spec->hi[c0 + j] : 0.f;
            P.w[j]   = spec ? w[c0 + j] : 1.f;
        }
        unsigned long long *cnt = spec ? (unsigned long long *)counts_dev + (int64_t)c0 * spec->nbins : nullptr;
        int rc;
        if (spec && spec->nbins > LO_TILE_BINS) {
            if (out_mode == 0)      rc = launch_f64_bins<0>(ctx, in, out, c0, P, cnt, aligned, G, s);
            else if (out_mode == 1) rc = launch_f64_bins<1>(ctx, in, out, c0, P, cnt, aligned, G, s);
            else                    rc = launch_f64_bins<2>(ctx, in, out, c0, P, cnt, aligned, G, s);
        } else if (spec) {
            if (out_mode == 0)      rc = launch_f64<0, true>(ctx, in, out, c0, P, cnt, aligned, G, s);
            else if (out_mode == 1) rc = launch_f64<1, true>(ctx, in, out, c0, P, cnt, aligned, G, s);
            else                    rc = launch_f64<2, true>(ctx, in, out, c0, P, cnt, aligned, G, s);
        } else {
            if (out_mode == 1)      rc = launch_f64<1, false>(ctx, in, out, c0, P, cnt, aligned, G, s);
            else                    rc = launch_f64<2, false>(ctx, in, out, c0, P, cnt, aligned, G, s);
        }
        LO_TRY(rc);
    }
    return LO_OK;
}

// the argument checks of hist_u8_impl, which enqueue nothing
int check_hist_u8(const lo_table *in, const int32_t *col_idx, int32_t k, const uint64_t *counts_dev, bool group) {
    if (!in) return fail(LO_ERR_INVALID, "input table is NULL");
    if (in->dtype != LO_U8) return fail(LO_ERR_INVALID, "input table must be LO_U8 (got dtype %d)", in->dtype);
    LO_TRY(check_cols(in, col_idx, k));
    if (!counts_dev && !group) return fail(LO_ERR_INVALID, "counts_dev is NULL");
    if (group && k > lo::kMaxColsU8) return fail(LO_ERR_INVALID, "a group step takes k <= %d byte columns (got %d)", lo::kMaxColsU8, k);
    return LO_OK;
}

int hist_u8_impl(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                 uint64_t *counts_dev, cudaStream_t s, const lo::GroupStep *group = nullptr) {
    LO_TRY(check_hist_u8(in, col_idx, k, counts_dev, group != nullptr));
    if (in->nrows == 0 && !group) return LO_OK;
    const lo::GroupStep &G = group ? *group : kNoGroup;
    const bool aligned = ((uintptr_t)in->base % 16 == 0) && (in->pitch % 16 == 0);
    // chunk of a column per CTA, a multiple of the 32 Ki-row round: long chunks amortise the 64 KiB clear + fold
    // (up to 8 rounds, one chunk per column on short shards)
    const int64_t slots = (int64_t)ctx->sm_count * 3;
    int64_t want = (in->nrows * (int64_t)std::min<int32_t>(k, lo::kMaxColsU8)) / slots;
    want = std::max<int64_t>(lo::kU8LRoundRows, std::min<int64_t>(want, 8 * (int64_t)lo::kU8LRoundRows));
    const int64_t chunk_rows = (want / lo::kU8LRoundRows) * lo::kU8LRoundRows;
    const unsigned chunks_per_col = (unsigned)((in->nrows + chunk_rows - 1) / chunk_rows);
    for (int32_t c0 = 0; c0 < k; c0 += lo::kMaxColsU8) {
        lo::ColsU8 P;
        P.k = std::min<int32_t>(lo::kMaxColsU8, k - c0);
        for (int j = 0; j < P.k; ++j) P.col[j] = col_idx[c0 + j];
        const unsigned long long blocks = (unsigned long long)chunks_per_col * (unsigned)P.k;
        if (blocks > 0x7fffffffull) return fail(LO_ERR_INVALID, "table too large for one launch");
        unsigned long long *cnt = (unsigned long long *)counts_dev + (int64_t)c0 * 256;
        const uint8_t *ib = (const uint8_t *)in->base;
        const long long ip = in->pitch, nr = in->nrows;
        LO_CUDA(launch_kernel(aligned ? lo::k_hist_u8_cols_lanes<true> : lo::k_hist_u8_cols_lanes<false>, (unsigned)blocks,
                              (unsigned)lo::kU8LThreads, (size_t)lo::kU8LSmemBytes, s, G.overlap != 0,
                              ib, ip, nr, chunks_per_col, (long long)chunk_rows, cnt, P, G));
        LO_CUDA(launched(ctx, 1));
    }
    return LO_OK;
}

int ensure_stage(StageSet *st, size_t in_bytes, size_t out_bytes, size_t ncounts) {
    if (in_bytes > st->in_bytes) {
        for (int i = 0; i < kSlots; ++i) {
            if (st->in[i]) cudaFree(st->in[i]);
            st->in[i] = nullptr;
        }
        st->in_bytes = 0;
        for (int i = 0; i < kSlots; ++i) LO_CUDA(cudaMalloc((void **)&st->in[i], in_bytes));
        st->in_bytes = in_bytes;
    }
    if (out_bytes > st->out_bytes) {
        for (int i = 0; i < kSlots; ++i) {
            if (st->out[i]) cudaFree(st->out[i]);
            st->out[i] = nullptr;
        }
        st->out_bytes = 0;
        for (int i = 0; i < kSlots; ++i) LO_CUDA(cudaMalloc((void **)&st->out[i], out_bytes));
        st->out_bytes = out_bytes;
    }
    if (ncounts > st->counts_n) {
        if (st->counts) cudaFree(st->counts);
        st->counts = nullptr;
        st->counts_n = 0;
        LO_CUDA(cudaMalloc((void **)&st->counts, ncounts * sizeof(unsigned long long)));
        st->counts_n = ncounts;
    }
    return LO_OK;
}

void stage_set_destroy(StageSet *st) {
    if (!st) return;
    for (int i = 0; i < kSlots; ++i) {
        if (st->in[i]) cudaFree(st->in[i]);
        if (st->out[i]) cudaFree(st->out[i]);
        if (st->ev_h2d[i]) cudaEventDestroy(st->ev_h2d[i]);
        if (st->ev_k[i]) cudaEventDestroy(st->ev_k[i]);
        if (st->ev_d2h[i]) cudaEventDestroy(st->ev_d2h[i]);
    }
    if (st->counts) cudaFree(st->counts);
    if (st->compute) cudaStreamDestroy(st->compute);
    if (st->h2d) cudaStreamDestroy(st->h2d);
    if (st->d2h) cudaStreamDestroy(st->d2h);
    delete st;
}

int stage_set_create(StageSet **out) {
    StageSet *st = new (std::nothrow) StageSet;
    if (!st) return fail(LO_ERR_NOMEM, "out of host memory");
    auto setup = [&]() -> int {
        LO_CUDA(cudaStreamCreateWithFlags(&st->compute, cudaStreamNonBlocking));
        LO_CUDA(cudaStreamCreateWithFlags(&st->h2d, cudaStreamNonBlocking));
        LO_CUDA(cudaStreamCreateWithFlags(&st->d2h, cudaStreamNonBlocking));
        for (int i = 0; i < kSlots; ++i) {
            LO_CUDA(cudaEventCreateWithFlags(&st->ev_h2d[i], cudaEventDisableTiming));
            LO_CUDA(cudaEventCreateWithFlags(&st->ev_k[i], cudaEventDisableTiming));
            LO_CUDA(cudaEventCreateWithFlags(&st->ev_d2h[i], cudaEventDisableTiming));
        }
        return LO_OK;
    };
    const int rc = setup();
    if (rc != LO_OK) { const std::string msg = g_err; stage_set_destroy(st); g_err = msg; return rc; }
    *out = st;
    return LO_OK;
}

// borrow a stage set for the duration of one *_host call
struct StageLease {
    lo_ctx *ctx;
    StageSet *st = nullptr;
    explicit StageLease(lo_ctx *c) : ctx(c) {}
    int acquire() {
        std::unique_lock<std::mutex> lk(ctx->pool_mu);
        for (;;) {
            if (!ctx->free_sets.empty()) { st = ctx->free_sets.back(); ctx->free_sets.pop_back(); return LO_OK; }
            if (ctx->nsets < kMaxStageSets) { ctx->nsets += 1; break; }
            ctx->pool_cv.wait(lk);
        }
        lk.unlock();
        const int rc = stage_set_create(&st);
        if (rc != LO_OK) { std::lock_guard<std::mutex> g(ctx->pool_mu); ctx->nsets -= 1; ctx->pool_cv.notify_one(); }
        return rc;
    }
    ~StageLease() {
        if (!st) return;
        { std::lock_guard<std::mutex> g(ctx->pool_mu); ctx->free_sets.push_back(st); }
        ctx->pool_cv.notify_one();
    }
};

// rows per chunk of the *_host pipeline: ~LOEXEC_CHUNK_MB (default 512) MiB of input per chunk, whole tiles
int64_t chunk_rows_for(int64_t nrows, int32_t k, size_t elem_bytes, int64_t tile_rows) {
    size_t mb = 256;   // large enough that per-copy submission cost is small against the PCIe transfer itself
    if (const char *e = getenv("LOEXEC_CHUNK_MB")) {
        long v = atol(e);
        if (v >= 1 && v <= 8192) mb = (size_t)v;
    }
    const int64_t target = (int64_t)((mb << 20) / ((size_t)k * elem_bytes));
    int64_t rows = std::max<int64_t>(tile_rows, (target / tile_rows) * tile_rows);
    return std::min(rows, ((nrows + tile_rows - 1) / tile_rows) * tile_rows);
}

// min / max / count of the finite cast values of k resident columns: one launch per column into out_dev[3*j ..]
int launch_minmax(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k, unsigned long long *out_dev, cudaStream_t s) {
    if (in->nrows == 0) return LO_OK;
    for (int j = 0; j < k; ++j) {
        dim3 grid((unsigned)std::min<int64_t>((in->nrows + 2047) / 2048, ctx->sm_count * 4), 1);
        lo::k_minmax_cast<<<grid, 256, 0, s>>>(in->base + (int64_t)col_idx[j] * in->pitch, in->pitch, in->nrows, out_dev + 3 * j);
        LO_CUDA(launched(ctx, 1));
    }
    return LO_OK;
}

// One call of an entry point that runs its kernels once, not in chunks: its stream, its first error, its scratch, its
// kernel time (summed over timed sections) and its launch count.  Once a step has failed every later step does
// nothing.  finish() frees the scratch, drains the stream and reports the first error ("<call>: <CUDA error string>",
// LO_ERR_NOMEM for an allocation, LO_ERR_CUDA otherwise) or fills lo_host_timing.
// Scratch is allocated and freed in stream order (cudaMallocAsync / cudaFreeAsync on the call's stream), so a call
// neither synchronises the device (cudaFree does) nor touches the legacy default stream (cudaMemcpy does): other
// jobs' streams keep running.
struct HostCall {
    lo_ctx *ctx;
    const char *name;
    cudaStream_t s;
    int rc = LO_OK;
    std::string msg;
    std::vector<void *> scratch, kept;
    std::vector<cudaEvent_t> marks;          // start, stop, start, stop, ... of the timed sections
    double h2d = 0, d2h = 0;
    const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    const int64_t launches0;
    const bool timed;                        // false: nobody reads the frame's lo_host_timing, so mark() records nothing

    HostCall(lo_ctx *c, const char *call, bool timed = true)
        : ctx(c), name(call), s(c->stream), launches0(c->launches.load()), timed(timed) {}
    ~HostCall() {
        release(scratch);
        for (cudaEvent_t ev : marks) cudaEventDestroy(ev);
    }
    bool ok() const { return rc == LO_OK; }
    void latch(cudaError_t e) {
        if (!ok() || e == cudaSuccess) return;
        rc = e == cudaErrorMemoryAllocation ? LO_ERR_NOMEM : LO_ERR_CUDA;
        msg = std::string(name) + ": " + cudaGetErrorString(e);
    }
    template <typename F> void run(F f) { if (ok()) latch(f()); }               // f returns a cudaError_t
    template <typename F> void check(F f) { if (ok() && (rc = f()) != LO_OK) msg = g_err; }   // f returns an LO_* code
    // f enqueues n kernels: <<<>>> launches, or CUB calls that return their cudaError_t
    template <typename F> void launch(int n, F f) {
        if (!ok()) return;
        if constexpr (std::is_void_v<decltype(f())>) f(); else latch(f());
        if (ok()) latch(launched(ctx, n));
    }
    template <typename T> void alloc(T **p, size_t bytes) {
        run([&] { return cudaMallocAsync((void **)p, bytes ? bytes : 1, s); });
        if (ok()) scratch.push_back(*p);
    }
    // p outlives a successful call (the caller owns it then); a failed call frees it with the scratch
    void keep(const void *p) {
        auto it = std::find(scratch.begin(), scratch.end(), p);
        if (it != scratch.end()) { kept.push_back(*it); scratch.erase(it); }
    }
    void drop(const void *p) {               // free one scratch buffer before the call ends
        auto it = std::find(scratch.begin(), scratch.end(), p);
        if (it != scratch.end()) { cudaFreeAsync(*it, s); scratch.erase(it); }
    }
    void to_dev(void *d, const void *h, size_t bytes) {
        if (!ok() || !bytes) return;
        latch(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
        h2d += (double)bytes;
    }
    void to_host(void *h, const void *d, size_t bytes) {
        if (!ok() || !bytes) return;
        latch(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s));
        d2h += (double)bytes;
    }
    void memset(void *d, int v, size_t bytes) { run([&] { return cudaMemsetAsync(d, v, bytes, s); }); }
    void sync() { run([&] { return cudaStreamSynchronize(s); }); }
    void mark() {                            // start or end of a timed section
        if (timed) run([&] {
            cudaEvent_t ev = nullptr;
            const cudaError_t e = cudaEventCreate(&ev);
            if (e != cudaSuccess) return e;
            marks.push_back(ev);
            return cudaEventRecord(ev, s);
        });
    }
    void release(std::vector<void *> &v) {
        for (void *p : v) cudaFreeAsync(p, s);
        v.clear();
    }
    int finish(lo_host_timing *timing) {
        release(scratch);
        latch(cudaStreamSynchronize(s));
        if (!ok()) {
            release(kept);
            return fail(rc, "%s", msg.c_str());
        }
        if (timing) {
            double kernel_ms = 0;
            for (size_t i = 0; i + 1 < marks.size(); i += 2) {
                float t = 0.f;
                if (cudaEventElapsedTime(&t, marks[i], marks[i + 1]) == cudaSuccess) kernel_ms += t;
            }
            timing->total_ms  = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            timing->h2d_bytes = h2d;
            timing->d2h_bytes = d2h;
            timing->launches  = ctx->launches.load() - launches0;
            timing->kernel_ms = kernel_ms;
        }
        return LO_OK;
    }
};

// ---- text columns from the host: the Arrow large_string layout of lo_parse_number_to_table (loexec.h) -------------
constexpr int kGroupRowBits = 31;            // the text group-by keeps a row index beside a 33-bit tag in one slot
constexpr int kAnyRowBits = 63;

// Refuses, in this order: n outside [0, 2^row_bits) before offsets is read, NULL offsets, offsets[n] < offsets[0], NULL
// chars with bytes to copy, both forms of validity, a negative bit offset.  check_ascending walks the offsets between.
int check_text_in(const uint8_t *chars, const int64_t *offsets, const lo_validity *validity, int64_t n, int row_bits) {
    if (n < 0 || n >> row_bits) return fail(LO_ERR_INVALID, "n = %lld: 0 to 2^%d-1 rows per call", (long long)n, row_bits);
    if (!offsets) return fail(LO_ERR_INVALID, "offsets is NULL");
    const int64_t nbytes = offsets[n] - offsets[0];
    if (nbytes < 0 || (nbytes > 0 && !chars)) return fail(LO_ERR_INVALID, "bad offsets / chars");
    if (validity && validity->mask && validity->bitmap) return fail(LO_ERR_INVALID, "validity: mask or bitmap, not both");
    if (validity && validity->bitmap && validity->bit_offset < 0) return fail(LO_ERR_INVALID, "validity: bit_offset < 0");
    return LO_OK;
}

int check_ascending(const int64_t *offsets, int64_t n) {
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i + 1] < offsets[i]) return fail(LO_ERR_INVALID, "offsets must be non-decreasing (row %lld)", (long long)i);
    return LO_OK;
}

// the host bytes of a checked validity that cover n cells: the n mask bytes, or the bitmap bytes holding bits
// bit_offset .. bit_offset + n - 1; none without validity
const uint8_t *validity_span(const lo_validity *v, int64_t n, size_t *bytes) {
    const bool mask = v && v->mask && n > 0, bitmap = v && v->bitmap && n > 0;
    *bytes = mask ? (size_t)n : bitmap ? (size_t)(((v->bit_offset + n - 1) >> 3) - (v->bit_offset >> 3) + 1) : 0;
    return mask ? v->mask : bitmap ? v->bitmap + (v->bit_offset >> 3) : nullptr;
}

// a text column on the device, as the text kernels take it: staged for one call (stage_text) or resident (lo_text)
struct TextCols {
    uint8_t *chars = nullptr;                // chars[offsets[0] .. offsets[n])
    long long *offsets = nullptr;
    uint8_t *mask = nullptr, *bitmap = nullptr;   // at most one: validity_span's bytes
    int bit0 = 0;                            // cell 0's bit in bitmap[0]
};

// A checked text column copied into c's scratch.  rebased NULL: the offsets are copied as given; else they start at 0
// on the device, rebased on the host into *rebased when offsets[0] != 0 (kept by the caller until the call synchronises).
TextCols stage_text(HostCall &c, const uint8_t *chars, const int64_t *offsets, const lo_validity *validity, int64_t n,
                    std::vector<int64_t> *rebased) {
    TextCols d;
    const size_t nbytes = (size_t)(offsets[n] - offsets[0]);
    size_t vbytes = 0;
    const uint8_t *valid = validity_span(validity, n, &vbytes);
    uint8_t **d_valid = vbytes && validity->mask ? &d.mask : &d.bitmap;
    c.alloc(&d.chars, nbytes);
    c.alloc(&d.offsets, (size_t)(n + 1) * 8);
    if (vbytes) c.alloc(d_valid, vbytes);
    c.to_dev(d.chars, chars + offsets[0], nbytes);
    if (rebased && offsets[0] != 0) {
        rebased->resize(n + 1);
        for (int64_t i = 0; i <= n; ++i) (*rebased)[i] = offsets[i] - offsets[0];
    }
    c.to_dev(d.offsets, rebased && !rebased->empty() ? rebased->data() : offsets, (size_t)(n + 1) * 8);
    c.to_dev(*d_valid, valid, vbytes);
    if (d.bitmap) d.bit0 = (int)(validity->bit_offset & 7);
    return d;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int lo_abi_version(void) { return LO_ABI_VERSION; }

const char *lo_last_error(void) { return g_err.c_str(); }

int lo_device_count(int *out) {
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        *out = 0;
        return fail(LO_ERR_NO_DEVICE, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    *out = n;
    return LO_OK;
}

int lo_init(int device, lo_ctx **out) {
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(LO_ERR_NO_DEVICE, "no CUDA device (%s); libloexec has no CPU fallback",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    if (device < 0 || device >= n) return fail(LO_ERR_INVALID, "device %d outside [0, %d)", device, n);
    cudaDeviceProp prop;
    LO_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(LO_ERR_NO_DEVICE, "device %d is sm_%d%d; libloexec is built for sm_90a only", device,
                    prop.major, prop.minor);
    // the byte-histogram kernel puts the start of dynamic shared memory (after this reserve) in an immediate offset
    int reserved = 0;
    LO_CUDA(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, device));
    if (reserved != LO_SMEM_WINDOW_BASE)
        return fail(LO_ERR_NO_DEVICE, "device %d reserves %d bytes of shared memory per block, the kernels assume %d",
                    device, reserved, LO_SMEM_WINDOW_BASE);
    LO_CUDA(cudaSetDevice(device));
    lo_ctx *ctx = new (std::nothrow) lo_ctx;
    if (!ctx) return fail(LO_ERR_NOMEM, "out of host memory");
    ctx->device    = device;
    ctx->sm_count  = prop.multiProcessorCount;
    ctx->hbm_bytes = prop.totalGlobalMem;
    ctx->stream = nullptr;
    auto setup = [&]() -> int {
        LO_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        LO_CUDA(cudaStreamCreateWithFlags(&ctx->edge_stream, cudaStreamNonBlocking));
        // scratch of the parser / group-by calls comes from the device's stream-ordered pool: keep up to 8 GiB of it
        // mapped between calls (the default threshold of 0 hands everything back at every synchronise, and the next
        // call pays the mapping again)
        cudaMemPool_t pool = nullptr;
        LO_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        uint64_t keep = 8ull << 30;
        if (const char *e = getenv("LOEXEC_POOL_KEEP_MB")) keep = (uint64_t)std::max<long long>(0, atoll(e)) << 20;
        LO_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
        return configure_kernels();
    };
    const int rc = setup();
    if (rc != LO_OK) {              // keep the error message, release whatever was created
        const std::string msg = g_err;
        lo_shutdown(ctx);
        g_err = msg;
        return rc;
    }
    *out = ctx;
    return LO_OK;
}

int lo_shutdown(lo_ctx *ctx) {
    if (!ctx) return LO_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (StageSet *st : ctx->free_sets) stage_set_destroy(st);
    ctx->free_sets.clear();
    if (ctx->edge_stream) {
        for (const auto &t : ctx->edge_tables) edge_retire(ctx, t.get());
        cudaStreamSynchronize(ctx->edge_stream);
        cudaStreamDestroy(ctx->edge_stream);
    }
    ctx->edge_tables.clear();
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return LO_OK;
}

int lo_ctx_device(const lo_ctx *ctx, int *device, int *sm_count, size_t *hbm_bytes) {
    if (!ctx) return fail(LO_ERR_INVALID, "ctx is NULL");
    if (device) *device = ctx->device;
    if (sm_count) *sm_count = ctx->sm_count;
    if (hbm_bytes) *hbm_bytes = ctx->hbm_bytes;
    return LO_OK;
}

int lo_sync(lo_ctx *ctx, void *stream) {
    LO_TRY(check_ctx(ctx));
    LO_CUDA(cudaStreamSynchronize(pick(ctx, stream)));
    return LO_OK;
}

int lo_launch_count(const lo_ctx *ctx, int64_t *out) {
    if (!ctx || !out) return fail(LO_ERR_INVALID, "NULL argument");
    *out = ctx->launches.load(std::memory_order_relaxed);
    return LO_OK;
}

int lo_host_alloc(lo_ctx *ctx, size_t bytes, void **out) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (bytes == 0) return LO_OK;
    LO_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
    return LO_OK;
}

int lo_host_alloc_flags(lo_ctx *ctx, size_t bytes, int32_t flags, void **out) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    if (flags & ~LO_HOST_WRITE_COMBINED) return fail(LO_ERR_INVALID, "unknown flags 0x%x", flags);
    *out = nullptr;
    if (bytes == 0) return LO_OK;
    LO_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable | ((flags & LO_HOST_WRITE_COMBINED) ? cudaHostAllocWriteCombined : 0)));
    return LO_OK;
}

int lo_host_free(lo_ctx *ctx, void *p) {
    LO_TRY(check_ctx(ctx));
    if (p) LO_CUDA(cudaFreeHost(p));
    return LO_OK;
}

// ---- tables -------------------------------------------------------------------------------------
int lo_table_alloc(lo_ctx *ctx, int dtype, int64_t nrows, int32_t ncols, lo_table **out) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    const size_t es = dtype_size(dtype);
    if (!es) return fail(LO_ERR_INVALID, "unknown dtype %d", dtype);
    if (nrows < 0 || ncols <= 0) return fail(LO_ERR_INVALID, "bad shape %lld x %d", (long long)nrows, ncols);
    const int64_t pitch = (int64_t)(((size_t)nrows * es + 255) / 256 * 256);
    lo_table *t = new (std::nothrow) lo_table;
    if (!t) return fail(LO_ERR_NOMEM, "out of host memory");
    t->dtype = dtype; t->nrows = nrows; t->ncols = ncols; t->pitch = pitch;
    t->base = nullptr; t->owned = true; t->device = ctx->device;
    const size_t bytes = std::max<size_t>((size_t)pitch * (size_t)ncols, 256);
    cudaError_t e = cudaMalloc((void **)&t->base, bytes);
    if (e != cudaSuccess) {
        delete t;
        cudaGetLastError();
        return fail(LO_ERR_NOMEM, "cudaMalloc(%zu bytes) for a %lld x %d table: %s", bytes, (long long)nrows,
                    ncols, cudaGetErrorString(e));
    }
    *out = t;
    return LO_OK;
}

int lo_table_wrap(lo_ctx *ctx, int dtype, int64_t nrows, int32_t ncols, void *base_dev, int64_t pitch_bytes,
                  lo_table **out) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    const size_t es = dtype_size(dtype);
    if (!es) return fail(LO_ERR_INVALID, "unknown dtype %d", dtype);
    if (nrows < 0 || ncols <= 0) return fail(LO_ERR_INVALID, "bad shape %lld x %d", (long long)nrows, ncols);
    if (!base_dev && nrows > 0) return fail(LO_ERR_INVALID, "base_dev is NULL");
    if (pitch_bytes < (int64_t)((size_t)nrows * es))
        return fail(LO_ERR_INVALID, "pitch %lld smaller than a column (%lld bytes)", (long long)pitch_bytes,
                    (long long)((size_t)nrows * es));
    if ((uintptr_t)base_dev % es || pitch_bytes % (int64_t)es)
        return fail(LO_ERR_ALIGNMENT, "base / pitch not aligned to the element size %zu", es);
    lo_table *t = new (std::nothrow) lo_table;
    if (!t) return fail(LO_ERR_NOMEM, "out of host memory");
    t->dtype = dtype; t->nrows = nrows; t->ncols = ncols; t->pitch = pitch_bytes;
    t->base = (char *)base_dev; t->owned = false; t->device = ctx->device;
    *out = t;
    return LO_OK;
}

int lo_table_free(lo_ctx *ctx, lo_table *t) {
    LO_TRY(check_ctx(ctx));
    if (!t) return LO_OK;
    if (t->owned && t->base) LO_CUDA(cudaFree(t->base));
    delete t;
    return LO_OK;
}

int lo_table_info(const lo_table *t, int *dtype, int64_t *nrows, int32_t *ncols, int64_t *pitch_bytes,
                  void **base_dev) {
    if (!t) return fail(LO_ERR_INVALID, "table is NULL");
    if (dtype) *dtype = t->dtype;
    if (nrows) *nrows = t->nrows;
    if (ncols) *ncols = t->ncols;
    if (pitch_bytes) *pitch_bytes = t->pitch;
    if (base_dev) *base_dev = t->base;
    return LO_OK;
}

static int check_range(const lo_table *t, int32_t col, int64_t row0, int64_t nrows) {
    if (!t) return fail(LO_ERR_INVALID, "table is NULL");
    if (col < 0 || col >= t->ncols) return fail(LO_ERR_INVALID, "column %d outside [0, %d)", col, t->ncols);
    if (row0 < 0 || nrows < 0 || row0 + nrows > t->nrows)
        return fail(LO_ERR_INVALID, "rows [%lld, %lld) outside [0, %lld)", (long long)row0,
                    (long long)(row0 + nrows), (long long)t->nrows);
    return LO_OK;
}

int lo_table_upload_col(lo_ctx *ctx, lo_table *t, int32_t col, int64_t row0, const void *host, int64_t nrows) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_range(t, col, row0, nrows));
    if (nrows == 0) return LO_OK;
    if (!host) return fail(LO_ERR_INVALID, "host is NULL");
    const size_t es = dtype_size(t->dtype);
    // on the context's stream and waited for: a pageable cudaMemcpy on the NULL stream may return before the DMA has
    // finished and is not ordered with the non-blocking streams the kernels run on
    LO_CUDA(cudaMemcpyAsync(t->base + (int64_t)col * t->pitch + row0 * (int64_t)es, host, (size_t)nrows * es,
                            cudaMemcpyHostToDevice, ctx->stream));
    LO_CUDA(cudaStreamSynchronize(ctx->stream));
    return LO_OK;
}

int lo_table_download_col(lo_ctx *ctx, const lo_table *t, int32_t col, int64_t row0, void *host, int64_t nrows,
                          void *stream) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_range(t, col, row0, nrows));
    if (nrows == 0) return LO_OK;
    if (!host) return fail(LO_ERR_INVALID, "host is NULL");
    const size_t es = dtype_size(t->dtype);
    cudaStream_t s = pick(ctx, stream);     // waits for this stream only: other streams' kernels keep running
    LO_CUDA(cudaMemcpyAsync(host, t->base + (int64_t)col * t->pitch + row0 * (int64_t)es, (size_t)nrows * es,
                            cudaMemcpyDeviceToHost, s));
    LO_CUDA(cudaStreamSynchronize(s));
    return LO_OK;
}

int lo_table_copy_col(lo_ctx *ctx, const lo_table *src, int32_t src_col, lo_table *dst, int32_t dst_col) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_range(src, src_col, 0, 0));
    LO_TRY(check_range(dst, dst_col, 0, 0));
    if (src->device != ctx->device || dst->device != ctx->device)
        return fail(LO_ERR_INVALID, "tables live on devices %d and %d, the context on %d", src->device, dst->device, ctx->device);
    if (src->dtype != dst->dtype || src->nrows != dst->nrows)
        return fail(LO_ERR_INVALID, "tables differ: dtype %d / %d, rows %lld / %lld", src->dtype, dst->dtype,
                    (long long)src->nrows, (long long)dst->nrows);
    if (src->nrows == 0) return LO_OK;
    const int64_t bytes = src->nrows * (int64_t)dtype_size(src->dtype);
    LO_CUDA(cudaMemcpyAsync(dst->base + (int64_t)dst_col * dst->pitch, src->base + (int64_t)src_col * src->pitch,
                            (size_t)bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    LO_CUDA(cudaStreamSynchronize(ctx->stream));
    return LO_OK;
}

int lo_table_fill_synthetic_dev(lo_ctx *ctx, lo_table *t, int kind, uint64_t seed, int64_t row_offset,
                                double lo_v, double hi_v, void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!t) return fail(LO_ERR_INVALID, "table is NULL");
    if (t->nrows == 0) return LO_OK;
    cudaStream_t s = pick(ctx, stream);
    const int grid = ctx->sm_count * 8;
    if (kind == LO_SYNTH_MNIST_U8) {
        if (t->dtype != LO_U8) return fail(LO_ERR_INVALID, "LO_SYNTH_MNIST_U8 needs an LO_U8 table");
        lo::k_fill_u8_mnist<<<grid, 256, 0, s>>>((uint8_t *)t->base, t->pitch, t->nrows, t->ncols, seed, row_offset);
    } else if (kind >= LO_SYNTH_UNIFORM && kind <= LO_SYNTH_CONSTCOL) {
        if (t->dtype != LO_F64) return fail(LO_ERR_INVALID, "f64 generators need an LO_F64 table");
        if (!(hi_v > lo_v) || !std::isfinite(lo_v) || !std::isfinite(hi_v) || hi_v == 0.0)
            return fail(LO_ERR_INVALID, "generator range must be finite with hi > lo and hi != 0");
        lo::k_fill_f64<<<grid, 256, 0, s>>>((double *)t->base, t->pitch / 8, t->nrows, t->ncols, kind, seed,
                                            row_offset, lo_v, hi_v);
    } else {
        return fail(LO_ERR_INVALID, "unknown generator kind %d", kind);
    }
    LO_CUDA(launched(ctx, 1));
    return LO_OK;
}

int lo_table_checksum(lo_ctx *ctx, const lo_table *t, int32_t col, int64_t row_offset, uint64_t *out) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_range(t, col, 0, 0));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    if (t->dtype == LO_I32) return fail(LO_ERR_INVALID, "table dtype LO_I32: the checksum reads LO_F64, LO_F32 and LO_U8 slabs");
    HostCall c(ctx, "checksum");
    unsigned long long *d = nullptr, h = 0;
    c.alloc(&d, 8);
    c.memset(d, 0, 8);
    if (t->nrows > 0)
        c.launch(1, [&] {
            const char *p = t->base + (int64_t)col * t->pitch;
            const int grid = ctx->sm_count * 8;
            if (t->dtype == LO_F64)      lo::k_checksum<double><<<grid, 256, 0, c.s>>>((const double *)p, t->nrows, row_offset, d);
            else if (t->dtype == LO_F32) lo::k_checksum<float><<<grid, 256, 0, c.s>>>((const float *)p, t->nrows, row_offset, d);
            else                         lo::k_checksum<uint8_t><<<grid, 256, 0, c.s>>>((const uint8_t *)p, t->nrows, row_offset, d);
        });
    c.to_host(&h, d, 8);
    LO_TRY(c.finish(nullptr));
    *out = h;
    return LO_OK;
}

int lo_selftest_fastdiv(lo_ctx *ctx, float lo_v, float hi_v, int32_t nbins, int *fast_path_used,
                        uint64_t *mismatches) {
    LO_TRY(check_ctx(ctx));
    if (!mismatches) return fail(LO_ERR_INVALID, "mismatches is NULL");
    lo_hist_spec spec = {nbins, 0, &lo_v, &hi_v};   // flags = 0
    float w = 0.f;
    LO_TRY(check_spec(&spec, 1, &w));
    if (fast_path_used) *fast_path_used = fastdiv_ok(w) ? 1 : 0;
    HostCall c(ctx, "selftest");
    unsigned long long *d = nullptr, h = 0;
    c.alloc(&d, 8);
    c.memset(d, 0, 8);
    c.launch(1, [&] { lo::k_selftest_fastdiv<<<ctx->sm_count * 16, 256, 0, c.s>>>(lo_v, hi_v, w, nbins, d); });
    c.to_host(&h, d, 8);
    LO_TRY(c.finish(nullptr));
    *mismatches = h;
    return LO_OK;
}

int lo_hist_edges(float lo_v, float hi_v, int32_t nbins, float *edges) {
    if (!edges) return fail(LO_ERR_INVALID, "edges is NULL");
    lo_hist_spec spec = {nbins, 0, &lo_v, &hi_v};
    float w = 0.f;
    LO_TRY(check_spec(&spec, 1, &w));
    hist_edges(lo_v, hi_v, w, nbins, edges);
    return LO_OK;
}

int lo_edge_tables_info(lo_ctx *ctx, int32_t *tables, uint64_t *bytes, int64_t *divide_launches) {
    if (!ctx) return fail(LO_ERR_INVALID, "ctx is NULL");
    std::lock_guard<std::mutex> g(ctx->edge_mu);
    uint64_t b = 0;
    for (const auto &t : ctx->edge_tables) b += t->bytes;
    if (tables) *tables = (int32_t)ctx->edge_tables.size();
    if (bytes) *bytes = b;
    if (divide_launches) *divide_launches = ctx->divide_launches.load(std::memory_order_relaxed);
    return LO_OK;
}

int lo_selftest_edges(lo_ctx *ctx, float lo_v, float hi_v, int32_t nbins, int *edges_used, uint64_t *mismatches) {
    LO_TRY(check_ctx(ctx));
    if (!mismatches) return fail(LO_ERR_INVALID, "mismatches is NULL");
    if (nbins > LO_TILE_BINS) return fail(LO_ERR_INVALID, "nbins = %d: the edge-table kernels take <= %d", nbins, LO_TILE_BINS);
    lo_hist_spec spec = {nbins, 0, &lo_v, &hi_v};
    float w = 0.f;
    LO_TRY(check_spec(&spec, 1, &w));
    if (edges_used) *edges_used = edges_ok(w) ? 1 : 0;
    std::vector<float> h((size_t)nbins + 1);
    hist_edges(lo_v, hi_v, w, nbins, h.data());
    HostCall c(ctx, "selftest");
    unsigned long long *d = nullptr, bad = 0;
    c.alloc(&d, 8 + h.size() * 4);
    float *E = reinterpret_cast<float *>(d + 1);
    c.to_dev(E, h.data(), h.size() * 4);
    c.memset(d, 0, 8);
    c.launch(1, [&] { lo::k_selftest_edges<<<ctx->sm_count * 16, 256, 0, c.s>>>(lo_v, hi_v, w, nbins, E, d); });
    c.to_host(&bad, d, 8);
    LO_TRY(c.finish(nullptr));
    *mismatches = bad;
    return LO_OK;
}

// per-column min / max / count of the finite cast values of RESIDENT columns; out_dev: uint64[3*k], zeroed here.
// Decode on the host with lo_minmax_decode.
int lo_minmax_cast_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k, uint64_t *out_dev, void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!in || in->dtype != LO_F64) return fail(LO_ERR_INVALID, "input table must be LO_F64");
    LO_TRY(check_cols(in, col_idx, k));
    if (!out_dev) return fail(LO_ERR_INVALID, "out_dev is NULL");
    cudaStream_t s = pick(ctx, stream);
    LO_CUDA(cudaMemsetAsync(out_dev, 0, (size_t)k * 24, s));
    return launch_minmax(ctx, in, col_idx, k, (unsigned long long *)out_dev, s);
}

// raw[3*k] (as downloaded from lo_minmax_cast_dev) -> mins / maxs / nfinite
int lo_minmax_decode(const uint64_t *raw, int32_t k, float *mins, float *maxs, uint64_t *nfinite) {
    if (!raw || !mins || !maxs || !nfinite || k < 0) return fail(LO_ERR_INVALID, "bad arguments");
    for (int j = 0; j < k; ++j) {
        nfinite[j] = raw[(size_t)j * 3 + 2];
        // the device kept min as ~ordered (so that zero-initialised memory is the identity) and max as ordered
        uint32_t omin = ~(uint32_t)raw[(size_t)j * 3 + 0], omax = (uint32_t)raw[(size_t)j * 3 + 1];
        auto unorder = [](uint32_t o) { uint32_t b = (o & 0x80000000u) ? (o ^ 0x80000000u) : ~o; float f; memcpy(&f, &b, 4); return f; };
        mins[j] = nfinite[j] ? unorder(omin) : 0.f;
        maxs[j] = nfinite[j] ? unorder(omax) : 0.f;
    }
    return LO_OK;
}

// ---- hot path, device resident ------------------------------------------------------------------
int lo_project_cast_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k, lo_table *out,
                        void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "output table is NULL");
    return project_cast_hist_impl(ctx, in, col_idx, k, out, nullptr, nullptr, pick(ctx, stream));
}

int lo_project_cast_hist_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k, lo_table *out,
                             const lo_hist_spec *spec, uint64_t *counts_dev, void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!spec) return fail(LO_ERR_INVALID, "spec is NULL (use lo_project_cast_dev for projection only)");
    return project_cast_hist_impl(ctx, in, col_idx, k, out, spec, counts_dev, pick(ctx, stream));
}

int lo_hist_u8_cols_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k, uint64_t *counts_dev,
                        void *stream) {
    LO_TRY(check_ctx(ctx));
    return hist_u8_impl(ctx, in, col_idx, k, counts_dev, pick(ctx, stream));
}

int lo_counts_alloc(lo_ctx *ctx, int64_t n, uint64_t **out_dev) {
    LO_TRY(check_ctx(ctx));
    if (!out_dev || n <= 0) return fail(LO_ERR_INVALID, "bad arguments");
    LO_CUDA(cudaMalloc((void **)out_dev, (size_t)n * 8));
    // zeroed on the context's stream and waited for, so launches on ANY stream after this call see zeros
    // (a NULL-stream cudaMemset is not ordered with cudaStreamNonBlocking streams)
    LO_CUDA(cudaMemsetAsync(*out_dev, 0, (size_t)n * 8, ctx->stream));
    LO_CUDA(cudaStreamSynchronize(ctx->stream));
    return LO_OK;
}

int lo_counts_free(lo_ctx *ctx, uint64_t *counts_dev) {
    LO_TRY(check_ctx(ctx));
    if (counts_dev) LO_CUDA(cudaFree(counts_dev));
    return LO_OK;
}

int lo_counts_zero_dev(lo_ctx *ctx, uint64_t *counts_dev, int64_t n, void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!counts_dev || n <= 0) return fail(LO_ERR_INVALID, "bad arguments");
    LO_CUDA(cudaMemsetAsync(counts_dev, 0, (size_t)n * 8, pick(ctx, stream)));
    return LO_OK;
}

int lo_counts_download(lo_ctx *ctx, const uint64_t *counts_dev, int64_t n, uint64_t *host, void *stream) {
    LO_TRY(check_ctx(ctx));
    if (!counts_dev || !host || n <= 0) return fail(LO_ERR_INVALID, "bad arguments");
    cudaStream_t s = pick(ctx, stream);
    LO_CUDA(cudaMemcpyAsync(host, counts_dev, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    LO_CUDA(cudaStreamSynchronize(s));
    return LO_OK;
}

// ---- hot path, host buffers ---------------------------------------------------------------------
// Three-stream pipeline over row chunks; chunk c uses staging slot c % kSlots:
//   h2d stream : wait(kernel of chunk c-kSlots done) -> k column copies             -> ev_h2d[slot]
//   compute    : wait(ev_h2d[slot]), wait(d2h of chunk c-kSlots done) -> kernel     -> ev_k[slot]
//   d2h stream : wait(ev_k[slot]) -> k column copies back                           -> ev_d2h[slot]
// `launch(tin, tout_or_null, counts_dev)` enqueues the kernel(s) of one chunk on ctx->stream.
// counts_target: device matrix the kernels accumulate into (NULL: the context's own scratch, zeroed here and
// downloaded into counts_host at the end; non-NULL: a group member's accumulate matrix, merged by the caller).
}  // extern "C"

namespace {

// One chunk of k host columns <-> k staging slabs.  Host columns that sit at a constant stride (one 2-D array, the
// usual case: a numpy matrix, an Arrow table's buffers from one allocation) go as ONE strided 2-D copy per run instead
// of one copy per column: 784 byte columns x 5 chunks would be 3 920 small submissions; a run is one.
// Columns that are separate allocations can also sit at a constant stride (page-locked buffers allocated one after
// another).  The runtime can reject a 2-D copy over such a run with cudaErrorInvalidValue, an argument check made
// before anything is enqueued; the run is then copied column by column.
int copy_cols(char *dev_base, int64_t dev_pitch, const void *const *host_cols, int64_t host_off, size_t bytes, int32_t k,
              bool to_device, cudaStream_t s) {
    for (int32_t j = 0; j < k;) {
        int32_t e = j + 1;
        const ptrdiff_t stride = (e < k) ? (const char *)host_cols[e] - (const char *)host_cols[j] : 0;
        if (stride >= (ptrdiff_t)bytes && stride <= (ptrdiff_t)0x7fffffff && dev_pitch <= 0x7fffffffll)   // cudaMemcpy2D pitch limit
            while (e < k && (const char *)host_cols[e] - (const char *)host_cols[e - 1] == stride) ++e;
        else
            e = j + 1;
        if (e - j >= 2) {
            char *d = dev_base + (int64_t)j * dev_pitch;
            char *h = (char *)host_cols[j] + host_off;
            const cudaError_t r = to_device
                ? cudaMemcpy2DAsync(d, (size_t)dev_pitch, h, (size_t)stride, bytes, (size_t)(e - j), cudaMemcpyHostToDevice, s)
                : cudaMemcpy2DAsync(h, (size_t)stride, d, (size_t)dev_pitch, bytes, (size_t)(e - j), cudaMemcpyDeviceToHost, s);
            if (r == cudaSuccess) { j = e; continue; }
            if (r != cudaErrorInvalidValue) LO_CUDA(r);
            (void)cudaGetLastError();
        }
        for (; j < e; ++j) {
            char *d = dev_base + (int64_t)j * dev_pitch;
            char *h = (char *)host_cols[j] + host_off;
            if (to_device) LO_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
            else           LO_CUDA(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s));
        }
    }
    return LO_OK;
}

template <typename Launch>
int host_pipeline(lo_ctx *ctx, const void *const *in_cols, int in_dtype, int64_t nrows, int32_t k,
                  void *const *out_cols, int out_dtype, int64_t tile_rows, size_t ncounts, uint64_t *counts_host,
                  lo_host_timing *timing, Launch launch, unsigned long long *counts_target = nullptr) {
    const auto t0 = std::chrono::steady_clock::now();
    const int64_t launches0 = ctx->launches.load();
    const size_t ies = dtype_size(in_dtype), oes = out_cols ? dtype_size(out_dtype) : 0;
    double h2d = 0, d2h = 0;
    if (counts_host && ncounts && !counts_target) memset(counts_host, 0, ncounts * 8);
    if (nrows > 0) {
        StageLease lease(ctx);
        LO_TRY(lease.acquire());
        StageSet *st = lease.st;
        auto body = [&]() -> int {
            const int64_t crows = chunk_rows_for(nrows, k, ies, tile_rows);
            const int64_t in_pitch  = (int64_t)(((size_t)crows * ies + 255) / 256 * 256);
            const int64_t out_pitch = (int64_t)(((size_t)crows * oes + 255) / 256 * 256);
            LO_TRY(ensure_stage(st, (size_t)in_pitch * k, out_cols ? (size_t)out_pitch * k : 0, counts_target ? 0 : ncounts));
            unsigned long long *cdev = counts_target ? counts_target : st->counts;
            if (ncounts && !counts_target) LO_CUDA(cudaMemsetAsync(cdev, 0, ncounts * 8, st->compute));
            const int64_t nchunks = (nrows + crows - 1) / crows;
            for (int64_t c = 0; c < nchunks; ++c) {
                const int slot = (int)(c % kSlots);
                const int64_t r0 = c * crows, n = std::min(crows, nrows - r0);
                if (c >= kSlots) LO_CUDA(cudaStreamWaitEvent(st->h2d, st->ev_k[slot], 0));
                LO_TRY(copy_cols(st->in[slot], in_pitch, in_cols, r0 * (int64_t)ies, (size_t)n * ies, k, true, st->h2d));
                h2d += (double)n * ies * k;
                LO_CUDA(cudaEventRecord(st->ev_h2d[slot], st->h2d));
                LO_CUDA(cudaStreamWaitEvent(st->compute, st->ev_h2d[slot], 0));
                if (c >= kSlots && out_cols) LO_CUDA(cudaStreamWaitEvent(st->compute, st->ev_d2h[slot], 0));
                lo_table tin  = {in_dtype, n, k, in_pitch, st->in[slot], false, ctx->device};
                lo_table tout = {out_dtype, n, k, out_pitch, out_cols ? st->out[slot] : nullptr, false, ctx->device};
                LO_TRY(launch(&tin, out_cols ? &tout : nullptr, cdev, st->compute));
                LO_CUDA(cudaEventRecord(st->ev_k[slot], st->compute));
                if (out_cols) {
                    LO_CUDA(cudaStreamWaitEvent(st->d2h, st->ev_k[slot], 0));
                    LO_TRY(copy_cols(st->out[slot], out_pitch, (const void *const *)out_cols, r0 * (int64_t)oes, (size_t)n * oes, k,
                                     false, st->d2h));
                    d2h += (double)n * oes * k;
                    LO_CUDA(cudaEventRecord(st->ev_d2h[slot], st->d2h));
                }
            }
            if (ncounts && counts_host && !counts_target) {
                LO_CUDA(cudaMemcpyAsync(counts_host, cdev, ncounts * 8, cudaMemcpyDeviceToHost, st->compute));
                d2h += (double)ncounts * 8;
            }
            return LO_OK;
        };
        const int rc = body();
        // success or failure: nothing may still be reading the caller's buffers or the staging slots when the
        // stage set goes back to the pool (on failure the message of the FIRST error is kept)
        const std::string first = g_err;
        const cudaError_t e1 = cudaStreamSynchronize(st->compute), e2 = cudaStreamSynchronize(st->d2h),
                          e3 = cudaStreamSynchronize(st->h2d);
        if (rc != LO_OK) { g_err = first; return rc; }
        if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)
            return fail(LO_ERR_CUDA, "host pipeline: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2 != cudaSuccess ? e2 : e3));
    }
    if (timing) {
        timing->total_ms  = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        timing->h2d_bytes = h2d;
        timing->d2h_bytes = d2h;
        timing->launches  = ctx->launches.load() - launches0;
        timing->kernel_ms = 0.0;      // chunks overlap their copies: there is no separate kernel time to report
    }
    return LO_OK;
}

int check_host_cols(const void *const *cols, int64_t nrows, int32_t k, const char *what) {
    if (k <= 0) return fail(LO_ERR_INVALID, "k must be > 0 (got %d)", k);
    if (nrows < 0) return fail(LO_ERR_INVALID, "nrows < 0");
    if (!cols) return fail(LO_ERR_INVALID, "%s is NULL", what);
    for (int j = 0; j < k; ++j)
        if (nrows > 0 && !cols[j]) return fail(LO_ERR_INVALID, "%s[%d] is NULL", what, j);
    return LO_OK;
}

// the arguments of lo_project_cast_hist_host and lo_group_project_cast_hist_host (at most max_k columns), and the
// column list 0 .. k-1 their pipelines project from the staged chunk
int check_project_host(const double *const *in_cols, int64_t nrows, int32_t k, float *const *out_cols,
                       const lo_hist_spec *spec, const uint64_t *counts, int32_t max_k, std::vector<int32_t> &ident) {
    LO_TRY(check_host_cols((const void *const *)in_cols, nrows, k, "in_cols"));
    if (out_cols) LO_TRY(check_host_cols((const void *const *)out_cols, nrows, k, "out_cols"));
    if (!out_cols && !spec) return fail(LO_ERR_INVALID, "nothing to do: no out_cols and no spec");
    if (spec && !counts) return fail(LO_ERR_INVALID, "counts is NULL");
    if (k > max_k) return fail(LO_ERR_INVALID, "k must be <= %d", max_k);
    std::vector<float> w(k);
    if (spec) LO_TRY(check_spec(spec, k, w.data()));
    ident.resize(k);
    for (int j = 0; j < k; ++j) ident[j] = j;
    return LO_OK;
}

// The output checks of every lo_value_counts_* call that returns groups, in the order they refuse: a negative capacity
// and a NULL ndistinct, after which *ndistinct is 0 until the groups are counted ...
int check_ndistinct(int64_t capacity, int64_t *ndistinct) {
    if (capacity < 0) return fail(LO_ERR_INVALID, "negative size");
    if (!ndistinct) return fail(LO_ERR_INVALID, "ndistinct is NULL");
    *ndistinct = 0;
    return LO_OK;
}

// ... then, once there is something to count, NULL outputs with room for groups
int check_groups_out(int64_t capacity, const void *keys_out, const uint64_t *counts_out) {
    if (capacity > 0 && (!keys_out || !counts_out)) return fail(LO_ERR_INVALID, "NULL argument");
    return LO_OK;
}

// The device half of the hash group-by of n rows.  launch(keys, counts, slots, out, out_n) enqueues the nlaunch kernels
// that count into a table of `slots` slots (keys all ones, counts zero), then compact at most out_n groups into
// out[0 .. out_n) (keys) and out[out_n .. 2 out_n) (counts) and the number of groups into out[2 out_n].  Returns out,
// in c's scratch; the table goes back to the pool in stream order.
template <typename Launch>
unsigned long long *count_groups(HostCall &c, int64_t n, size_t out_n, Launch launch, int nlaunch = 2) {
    unsigned long long slots = 1024;
    while (slots < 2ull * (unsigned long long)n) slots <<= 1;
    unsigned long long *d_keys = nullptr, *d_counts = nullptr, *d_out = nullptr;
    c.alloc(&d_keys, slots * 8);
    c.alloc(&d_counts, slots * 8);
    c.alloc(&d_out, (2 * out_n + 1) * 8);
    c.mark();
    c.memset(d_keys, 0xFF, slots * 8);
    c.memset(d_counts, 0, slots * 8);
    c.memset(d_out + 2 * out_n, 0, 8);
    c.launch(nlaunch, [&] { launch(d_keys, d_counts, slots, d_out, out_n); });
    c.mark();
    c.drop(d_keys);
    c.drop(d_counts);
    return d_out;
}

// The end of every call that returns at most `capacity` of the nd groups it found: the first min(nd, capacity) 8-byte
// words of each {host output, device column} pair copied out and the call finished.  More groups than capacity is
// refused after *ndistinct is set, so the caller can retry larger.
int finish_groups(HostCall &c, unsigned long long nd, int64_t capacity,
                  std::initializer_list<std::pair<void *, const void *>> outs, int64_t *ndistinct, lo_host_timing *timing) {
    const size_t take = (size_t)std::min<unsigned long long>(nd, (unsigned long long)capacity);
    for (const auto &[host, dev] : outs) c.to_host(host, dev, take * 8);
    LO_TRY(c.finish(timing));
    *ndistinct = (int64_t)nd;
    if ((int64_t)nd > capacity)
        return fail(LO_ERR_INVALID, "%llu distinct keys do not fit the caller's capacity %lld", nd, (long long)capacity);
    return LO_OK;
}

// The host half: the groups of count_groups' out (out_n = capacity), their number read first.
int copy_groups(HostCall &c, const unsigned long long *out, int64_t capacity, void *keys_out, uint64_t *counts_out,
                int64_t *ndistinct, lo_host_timing *timing) {
    unsigned long long nd = 0;
    c.to_host(&nd, out + 2 * capacity, 8);
    c.sync();
    return finish_groups(c, nd, capacity, {{keys_out, out}, {counts_out, out + capacity}}, ndistinct, timing);
}

// The rest of a lo_value_counts_* call once its input is on the device: at most `capacity` groups, copied out.
template <typename Launch>
int value_counts_tail(HostCall &c, int64_t n, void *keys_out, uint64_t *counts_out, int64_t capacity, int64_t *ndistinct,
                      lo_host_timing *timing, Launch launch, int nlaunch = 2) {
    const unsigned long long *out = count_groups(c, n, (size_t)capacity, launch, nlaunch);
    return copy_groups(c, out, capacity, keys_out, counts_out, ndistinct, timing);
}

// blocks of 256 threads for n items, at most 8 per SM
int grid_for(const lo_ctx *ctx, int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8); }

// count_groups of the n cells of a text column on the device (offsets[0] == 0; validity as k_hash_count_str reads
// it): the keys are the groups' representative rows
unsigned long long *count_text_groups(HostCall &c, const TextCols &t, int64_t n, size_t out_n) {
    return count_groups(c, n, out_n,
        [&](unsigned long long *slots_keys, unsigned long long *counts, unsigned long long slots, unsigned long long *out, size_t) {
            lo::k_hash_count_str<<<grid_for(c.ctx, n), 256, 0, c.s>>>(t.chars, t.offsets, n, t.mask, t.bitmap, t.bit0,
                                                                       slots_keys, counts, slots - 1);
            lo::k_hash_compact_str<<<c.ctx->sm_count * 8, 256, 0, c.s>>>(slots_keys, counts, slots, (long long *)out,
                                                                          out + out_n, (unsigned long long)out_n, out + 2 * out_n);
        });
}

// the groups of a text column already on the device: the call of lo_value_counts_str_host after its copies, and all of
// lo_value_counts_text
int value_counts_str_tail(HostCall &c, const TextCols &t, int64_t n, int64_t *rep_rows_out, uint64_t *counts_out,
                          int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    const unsigned long long *out = count_text_groups(c, t, n, (size_t)capacity);
    return copy_groups(c, out, capacity, rep_rows_out, counts_out, ndistinct, timing);
}

// value_counts_tail of rows [0, n) of a number column already on the device: the call of lo_value_counts_f64_host after
// its copy, and all of lo_value_counts_f64_table.  A 16-byte aligned column takes k_group_f64's 16-byte loads.
int value_counts_f64_tail(HostCall &c, const double *d_val, int64_t n, double *keys_out, uint64_t *counts_out,
                          int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    return value_counts_tail(c, n, keys_out, counts_out, capacity, ndistinct, timing,
        [&](unsigned long long *keys, unsigned long long *counts, unsigned long long slots, unsigned long long *out, size_t out_n) {
            const int grid = (int)std::min<int64_t>((n + 511) / 512, (int64_t)c.ctx->sm_count * 8);
            if ((uintptr_t)d_val % 16 == 0)
                lo::k_group_f64<true><<<grid, 256, 0, c.s>>>(d_val, n, keys, counts, slots - 1);
            else
                lo::k_group_f64<false><<<grid, 256, 0, c.s>>>(d_val, n, keys, counts, slots - 1);
            lo::k_hash_compact<<<c.ctx->sm_count * 8, 256, 0, c.s>>>(keys, counts, slots, out, out + out_n,
                                                                      (unsigned long long)out_n, out + 2 * out_n);
        });
}

}  // namespace

static_assert(lo::kStrStageSlots == LO_TEXT_STAGE_SLOTS, "loexec.h documents the text group-by's stage size");

// one text column resident in HBM (lo_text_upload): chars, offsets rebased to 0, the validity as it was given (n mask
// bytes, or the bitmap bytes covering the column with the first cell at bit bit0), all from the stream-ordered pool
struct lo_text {
    lo_ctx *ctx;
    TextCols cols;
    int64_t n, nbytes, nulls;
    size_t device_bytes;
};

extern "C" {

int lo_project_cast_hist_host(lo_ctx *ctx, const double *const *in_cols, int64_t nrows, int32_t k,
                              float *const *out_cols, const lo_hist_spec *spec, uint64_t *counts,
                              lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    std::vector<int32_t> ident;
    LO_TRY(check_project_host(in_cols, nrows, k, out_cols, spec, counts, INT32_MAX, ident));
    const size_t ncounts = spec ? (size_t)k * (size_t)spec->nbins : 0;
    return host_pipeline(ctx, (const void *const *)in_cols, LO_F64, nrows, k, (void *const *)out_cols, LO_F32,
                         lo::kTileRows, ncounts, counts, timing,
                         [&](lo_table *tin, lo_table *tout, unsigned long long *cdev, cudaStream_t cs) {
                             return project_cast_hist_impl(ctx, tin, ident.data(), k, tout, spec, (uint64_t *)cdev, cs);
                         });
}

int lo_hist_u8_cols_host(lo_ctx *ctx, const uint8_t *const *in_cols, int64_t nrows, int32_t k, uint64_t *counts,
                         lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_host_cols((const void *const *)in_cols, nrows, k, "in_cols"));
    if (!counts) return fail(LO_ERR_INVALID, "counts is NULL");
    std::vector<int32_t> ident(k);
    for (int j = 0; j < k; ++j) ident[j] = j;
    return host_pipeline(ctx, (const void *const *)in_cols, LO_U8, nrows, k, nullptr, LO_U8, lo::kU8HostChunkRows,
                         (size_t)k * 256, counts, timing, [&](lo_table *tin, lo_table *, unsigned long long *cdev, cudaStream_t cs) {
                             return hist_u8_impl(ctx, tin, ident.data(), k, (uint64_t *)cdev, cs);
                         });
}

// exact value counts of dictionary-encoded columns: counts[c] = #{r : codes[r] == c}
int lo_value_counts_u32_host(lo_ctx *ctx, const uint32_t *codes, int64_t nrows, uint32_t ncodes, uint64_t *counts,
                             lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (nrows < 0 || ncodes == 0) return fail(LO_ERR_INVALID, "bad arguments (nrows %lld, ncodes %u)", (long long)nrows, ncodes);
    if ((nrows > 0 && !codes) || !counts) return fail(LO_ERR_INVALID, "NULL argument");
    const void *cols[1] = {codes};
    // counts buffer layout: [ncodes counts][1 out-of-range flag]
    std::vector<uint64_t> tmp((size_t)ncodes + 1);
    int rc = host_pipeline(ctx, cols, LO_U32, nrows, 1, nullptr, LO_U32, 1 << 16, (size_t)ncodes + 1, tmp.data(), timing,
                           [&](lo_table *tin, lo_table *, unsigned long long *cdev, cudaStream_t cs) {
                               const int grid = ctx->sm_count * 8;
                               lo::k_count_codes_u32<<<grid, 256, 0, cs>>>(
                                   (const uint32_t *)tin->base, tin->nrows, ncodes, cdev);
                               LO_CUDA(launched(ctx, 1));
                               return LO_OK;
                           });
    LO_TRY(rc);
    if (tmp[ncodes] != 0) return fail(LO_ERR_INVALID, "%llu codes were >= ncodes (%u)", (unsigned long long)tmp[ncodes], ncodes);
    memcpy(counts, tmp.data(), (size_t)ncodes * 8);
    return LO_OK;
}

// exact value counts of one numeric column (GPU hash group-by).  keys_out / counts_out: host arrays of
// `capacity` entries; *ndistinct receives the number of distinct keys (may exceed capacity: then only the first
// `capacity` groups were written and the call fails with LO_ERR_INVALID so the caller can retry larger).
int lo_value_counts_f64_host(lo_ctx *ctx, const double *values, int64_t n, double *keys_out, uint64_t *counts_out,
                             int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "negative size");
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (n == 0) return LO_OK;
    if (!values) return fail(LO_ERR_INVALID, "NULL argument");
    LO_TRY(check_groups_out(capacity, keys_out, counts_out));
    HostCall c(ctx, "value_counts_f64");
    double *d_val = nullptr;
    c.alloc(&d_val, (size_t)n * 8);
    c.to_dev(d_val, values, (size_t)n * 8);
    return value_counts_f64_tail(c, d_val, n, keys_out, counts_out, capacity, ndistinct, timing);
}

// the same on rows [0, nrows) of column `col` of a device table: nothing crosses PCIe but the groups
int lo_value_counts_f64_table(lo_ctx *ctx, const lo_table *t, int32_t col, double *keys_out, uint64_t *counts_out,
                              int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!t) return fail(LO_ERR_INVALID, "table is NULL");
    if (t->device != ctx->device) return fail(LO_ERR_INVALID, "table lives on device %d, the context on %d", t->device, ctx->device);
    if (t->dtype != LO_F64) return fail(LO_ERR_INVALID, "table dtype %d is not LO_F64", t->dtype);
    if (col < 0 || col >= t->ncols) return fail(LO_ERR_INVALID, "column %d outside [0, %d)", col, t->ncols);
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (t->nrows == 0) return LO_OK;
    LO_TRY(check_groups_out(capacity, keys_out, counts_out));
    HostCall c(ctx, "value_counts_f64_table");
    return value_counts_f64_tail(c, (const double *)(t->base + (int64_t)col * t->pitch), t->nrows, keys_out, counts_out,
                                 capacity, ndistinct, timing);
}

// exact value counts of one TEXT column (cells = chars[offsets[i] .. offsets[i+1])): GPU hash group-by on the bytes.
// rep_rows_out[g] = row index of one member of group g (the caller reads the key from its own cell), counts_out[g].
int lo_value_counts_str_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n, int64_t *rep_rows_out,
                             uint64_t *counts_out, int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "negative size");
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (n == 0) return LO_OK;
    LO_TRY(check_groups_out(capacity, rep_rows_out, counts_out));
    LO_TRY(check_text_in(chars, offsets, nullptr, n, kGroupRowBits));
    if (offsets[0] != 0) return fail(LO_ERR_INVALID, "offsets[0] must be 0");
    LO_TRY(check_ascending(offsets, n));
    HostCall c(ctx, "value_counts_str");
    const TextCols d = stage_text(c, chars, offsets, nullptr, n, nullptr);    // offsets[0] is 0: copied as given
    return value_counts_str_tail(c, d, n, rep_rows_out, counts_out, capacity, ndistinct, timing);
}

// ---- text columns resident in HBM ---------------------------------------------------------------------------------
int lo_text_upload(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, const lo_validity *validity, int64_t n,
                   lo_text **out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    LO_TRY(check_text_in(chars, offsets, validity, n, kGroupRowBits));
    LO_TRY(check_ascending(offsets, n));
    const int64_t nbytes = offsets[n] - offsets[0];
    size_t valid_bytes = 0;
    validity_span(validity, n, &valid_bytes);
    const size_t need = (size_t)std::max<int64_t>(nbytes, 1) + (size_t)(n + 1) * 8 + valid_bytes;
    size_t free_b = 0, total_b = 0;
    const cudaError_t e = cudaMemGetInfo(&free_b, &total_b);
    if (e != cudaSuccess) return fail(LO_ERR_CUDA, "cudaMemGetInfo: %s", cudaGetErrorString(e));
    if (need > free_b)
        return fail(LO_ERR_NOMEM, "text_upload: the column needs %zu bytes of device memory, %zu are free", need, free_b);
    int64_t nulls = 0;                       // counted here: the host holds the validity already
    if (validity && validity->mask) {
        for (int64_t i = 0; i < n; ++i) nulls += validity->mask[i] == 0;
    } else if (validity && validity->bitmap) {
        for (int64_t i = 0; i < n; ++i) {
            const int64_t b = validity->bit_offset + i;
            nulls += ((validity->bitmap[b >> 3] >> (b & 7)) & 1) == 0;
        }
    }
    std::unique_ptr<lo_text> t(new (std::nothrow) lo_text);
    if (!t) return fail(LO_ERR_NOMEM, "out of host memory");
    HostCall c(ctx, "text_upload");
    std::vector<int64_t> rebased;
    const TextCols d = stage_text(c, chars, offsets, validity, n, &rebased);
    for (const void *p : {(const void *)d.chars, (const void *)d.offsets, (const void *)d.mask, (const void *)d.bitmap})
        c.keep(p);
    LO_TRY(c.finish(timing));                // synchronises: the host buffers may go
    *t = lo_text{ctx, d, n, nbytes, nulls, need};
    *out = t.release();
    return LO_OK;
}

int lo_text_info(const lo_text *t, int64_t *n, int64_t *nbytes, int64_t *nulls, size_t *device_bytes) {
    if (!t) return fail(LO_ERR_INVALID, "text is NULL");
    if (n) *n = t->n;
    if (nbytes) *nbytes = t->nbytes;
    if (nulls) *nulls = t->nulls;
    if (device_bytes) *device_bytes = t->device_bytes;
    return LO_OK;
}

int lo_text_free(lo_ctx *ctx, lo_text *t) {
    if (!t) return LO_OK;
    LO_TRY(check_ctx(ctx));
    if (t->ctx != ctx) return fail(LO_ERR_INVALID, "text belongs to another context");
    for (void *p : {(void *)t->cols.chars, (void *)t->cols.offsets, (void *)t->cols.mask, (void *)t->cols.bitmap})
        if (p) cudaFreeAsync(p, ctx->stream);
    delete t;
    return LO_OK;
}

int lo_value_counts_text(lo_ctx *ctx, const lo_text *t, int64_t *rep_rows_out, uint64_t *counts_out, int64_t capacity,
                         int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!t) return fail(LO_ERR_INVALID, "text is NULL");
    if (t->ctx != ctx) return fail(LO_ERR_INVALID, "text belongs to another context");
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (t->n == t->nulls) return LO_OK;      // no cell to count (n == 0 included)
    LO_TRY(check_groups_out(capacity, rep_rows_out, counts_out));
    HostCall c(ctx, "value_counts_text");
    return value_counts_str_tail(c, t->cols, t->n, rep_rows_out, counts_out, capacity, ndistinct, timing);
}

}  // extern "C"

namespace {

// The refusals of every call on a text column cut into row-range shards, in this order: a NULL root, nshards outside
// [1, LO_GROUP_MAX_DEVICES], NULL shards or row0, then shard by shard a NULL shard and a row0 that is negative or inside
// the shard before.
int check_shards(const lo_ctx *root, const lo_text *const *shards, const int64_t *row0, int32_t nshards) {
    if (!root) return fail(LO_ERR_INVALID, "root is NULL");
    static_assert(lo::kMaxPeers + 1 == LO_GROUP_MAX_DEVICES, "a group's devices: the root and its peers");
    if (nshards < 1 || nshards > LO_GROUP_MAX_DEVICES)
        return fail(LO_ERR_INVALID, "nshards = %d: 1 to %d shards", nshards, LO_GROUP_MAX_DEVICES);
    if (!shards || !row0) return fail(LO_ERR_INVALID, "shards or row0 is NULL");
    for (int i = 0; i < nshards; ++i) {
        if (!shards[i]) return fail(LO_ERR_INVALID, "shards[%d] is NULL", i);
        if (row0[i] < 0) return fail(LO_ERR_INVALID, "row0[%d] = %lld is negative", i, (long long)row0[i]);
        if (i > 0 && row0[i] < row0[i - 1] + shards[i - 1]->n)
            return fail(LO_ERR_INVALID, "row0[%d] = %lld: shard %d ends at row %lld (shards are disjoint and in row order)",
                        i, (long long)row0[i], i - 1, (long long)(row0[i - 1] + shards[i - 1]->n));
    }
    return LO_OK;
}

// The offsets of a key column of the cells at nd rows of a text column on c's device: the exclusive scan of their byte
// lengths, nd + 1 of them (the last is their bytes).  Two launches.
long long *key_offsets(HostCall &c, const TextCols &t, const unsigned long long *rows, int64_t nd) {
    long long *key_off = nullptr;
    size_t scan_bytes = 0;
    void *tmp = nullptr;
    c.alloc(&key_off, (size_t)(nd + 1) * 8);
    c.run([&] { return cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, key_off, nd + 1, c.s); });
    c.alloc(&tmp, scan_bytes);
    c.memset(key_off + nd, 0, 8);            // the scan's last input
    c.launch(1, [&] { lo::k_gather_lens<<<grid_for(c.ctx, nd), 256, 0, c.s>>>(t.offsets, (const long long *)rows, nd, key_off); });
    c.launch(1, [&] { return cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, key_off, nd + 1, c.s); });
    c.drop(tmp);
    return key_off;
}

// A call on one text column cut into checked row-range shards, each resident on its own context, whose groups are
// merged on root's context.  Each shard works on an untimed call frame of its own, on its context's stream; the root's
// frame `c` times the call.  Each step is enqueued on every shard before the host waits on any, so shards on different
// devices run at once:
//   1. each: the caller lists every shard's groups on its device, one row of each group;
//   2. pack_keys: the host reads each shard's group count; the byte lengths of its groups' cells and their exclusive
//      scan; the host reads its key bytes; k_gather_cells packs the keys, rebases their offsets into the concatenated
//      column and makes the rows global;
//   3. send_keys: the root waits on each shard's event and copies the packed pieces over with cudaMemcpyPeerAsync;
//   4. wait_root: once the root has read the pieces, each shard's stream waits on the root's, so a shard's scratch is
//      freed after the root has read it;
//   5. finish: the root's frame first, then every shard's.
// X is the caller's own state of a shard.
template <typename X>
struct ShardFrame {
    struct Shard : X {
        const lo_text *t;
        int64_t row0;
        int64_t live;                                // n - nulls: at most this many groups
        std::unique_ptr<HostCall> c;
        unsigned long long nd = 0;                   // its groups
        long long *key_off = nullptr;                // the packed key column of its groups: nd + 1 offsets, then the bytes
        uint8_t *key_chars = nullptr;
        cudaEvent_t gathered = nullptr;              // the packed pieces are ready to copy
        long long bytes = 0, group0 = 0, byte0 = 0;  // its bytes, and where its pieces start in the concatenated column
    };
    lo_ctx *root;
    HostCall c;
    std::vector<Shard> sh;                           // the shards with a row, in row order
    long long groups = 0, bytes = 0;                 // summed over the shards
    cudaEvent_t root_read = nullptr;                 // wait_root's event on root's stream

    // own(i): the caller's state of shards[i]
    template <typename Own>
    ShardFrame(lo_ctx *root_, const char *name, const lo_text *const *shards, const int64_t *row0, int32_t nshards, Own own)
        : root(root_), c(root_, name) {
        for (int i = 0; i < nshards; ++i)
            if (shards[i]->n > 0)
                sh.push_back(Shard{own(i), shards[i], row0[i], shards[i]->n - shards[i]->nulls,
                                   std::make_unique<HostCall>(shards[i]->ctx, name, false)});
    }

    bool ok() const { return c.ok() && std::all_of(sh.begin(), sh.end(), [](const Shard &s) { return s.c->ok(); }); }

    // step(s, its call frame) for every shard with a cell, in row order, on the shard's device, until the root or a
    // shard fails
    template <typename Step> void each(Step step) {
        for (Shard &s : sh) {
            if (!ok()) return;
            if (!s.live) continue;
            s.c->run([&] { return cudaSetDevice(s.t->ctx->device); });
            step(s, *s.c);
        }
    }

    // listed(s) = {the rows in s of its groups, on its device; the word there that holds their number}
    template <typename Listed> void pack_keys(Listed listed) {
        each([&](Shard &s, HostCall &sc) { sc.to_host(&s.nd, listed(s).second, 8); sc.sync(); });
        each([&](Shard &s, HostCall &sc) { s.key_off = key_offsets(sc, s.t->cols, listed(s).first, (int64_t)s.nd); });
        each([&](Shard &s, HostCall &sc) {
            sc.to_host(&s.bytes, s.key_off + s.nd, 8);
            sc.sync();
            s.group0 = groups;
            s.byte0 = bytes;
            groups += (long long)s.nd;
            bytes += s.bytes;
        });
        if (ok() && groups >> 31)            // the merge's slot word keeps a 31-bit key index, and codes are int32
            c.check([&] { return fail(LO_ERR_INVALID, "the shards hold %lld groups: at most 2^31-1 can be merged", groups); });
        each([&](Shard &s, HostCall &sc) {   // pack the keys
            sc.alloc(&s.key_chars, (size_t)s.bytes);
            sc.launch(1, [&] {
                lo::k_gather_cells<<<grid_for(sc.ctx, (int64_t)s.nd + 1), 256, 0, sc.s>>>(s.t->cols.chars, s.t->cols.offsets,
                    (long long *)listed(s).first, (long long)s.nd, s.key_off, s.key_chars, s.row0, s.byte0);
            });
            sc.run([&] { return cudaEventCreateWithFlags(&s.gathered, cudaEventDisableTiming); });
            sc.run([&] { return cudaEventRecord(s.gathered, sc.s); });
        });
    }

    // On root's device: chars and offsets receive the concatenated key column (offsets[groups] = bytes), and each of
    // `cols` one 8-byte word per group, cols[j] taking words(s)[j] .. + nd of every shard s.
    template <size_t N, typename Words>
    void send_keys(uint8_t *&chars, long long *&offsets, std::array<unsigned long long *, N> &cols, Words words) {
        c.run([&] { return cudaSetDevice(root->device); });
        c.alloc(&chars, (size_t)bytes);
        c.alloc(&offsets, (size_t)(groups + 1) * 8);
        for (unsigned long long *&col : cols) c.alloc(&col, (size_t)groups * 8);
        for (Shard &s : sh) {
            if (!s.live) continue;
            const int dev = s.t->ctx->device;
            c.run([&] { return cudaStreamWaitEvent(c.s, s.gathered, 0); });
            // nd + 1 offsets: the last is the next shard's first (the same value), or offsets[groups]
            c.run([&] { return cudaMemcpyPeerAsync(offsets + s.group0, root->device, s.key_off, dev, (s.nd + 1) * 8, c.s); });
            for (size_t j = 0; j < N; ++j)
                c.run([&] { return cudaMemcpyPeerAsync(cols[j] + s.group0, root->device, words(s)[j], dev, s.nd * 8, c.s); });
            if (s.bytes) c.run([&] { return cudaMemcpyPeerAsync(chars + s.byte0, root->device, s.key_chars, dev, s.bytes, c.s); });
        }
    }

    // every shard's stream waits on what root's stream has enqueued so far: its reads of the pieces, and what the shards
    // read back from it
    void wait_root() {
        c.run([&] { return cudaEventCreateWithFlags(&root_read, cudaEventDisableTiming); });
        c.run([&] { return cudaEventRecord(root_read, c.s); });
        for (Shard &s : sh)
            if (s.live && c.ok()) s.c->run([&] { return cudaStreamWaitEvent(s.c->s, root_read, 0); });
    }

    // After the root's frame has finished with `rc` (it has synchronised: nothing of it reads a shard any more): frees
    // every shard's scratch.  The root's error is the call's, else the first shard's in row order; root's device is
    // current again.
    int finish(int rc) {
        std::string msg = g_err;
        for (Shard &s : sh) {
            cudaSetDevice(s.t->ctx->device);
            const int r = s.c->finish(nullptr);
            if (rc == LO_OK && r != LO_OK) { rc = r; msg = g_err; }
            if (s.gathered) cudaEventDestroy(s.gathered);
        }
        if (root_read) cudaEventDestroy(root_read);
        cudaSetDevice(root->device);
        g_err = msg;
        return rc;
    }
};

// lo_value_counts_text_shards' own state of a shard: count_text_groups' out, rows [0, live), counts [live, 2 live),
// their number [2 live]
struct CountShard {
    unsigned long long *grp = nullptr;
};

}  // namespace

extern "C" {

// Value counts of one text column cut into row-range shards, each resident on its own context (loexec.h), in the steps
// of ShardFrame: each shard counts and compacts its cells (count_text_groups) and packs its groups' keys; the root
// copies the keys with their rows and counts over and merges them (k_hash_sum_str, k_hash_compact_str, k_take_rows).
int lo_value_counts_text_shards(lo_ctx *root, const lo_text *const *shards, const int64_t *row0, int32_t nshards,
                                int64_t *rep_rows_out, uint64_t *counts_out, int64_t capacity, int64_t *ndistinct,
                                lo_host_timing *timing) {
    LO_TRY(check_shards(root, shards, row0, nshards));
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (std::none_of(shards, shards + nshards, [](const lo_text *t) { return t->n > t->nulls; })) return LO_OK;
    LO_TRY(check_groups_out(capacity, rep_rows_out, counts_out));
    LO_TRY(check_ctx(root));
    ShardFrame<CountShard> f(root, "value_counts_text_shards", shards, row0, nshards, [](int) { return CountShard{}; });
    f.each([](auto &s, HostCall &sc) { s.grp = count_text_groups(sc, s.t->cols, s.t->n, (size_t)s.live); });
    f.pack_keys([](auto &s) { return std::pair(s.grp, s.grp + 2 * s.live); });
    if (!f.ok()) return f.finish(f.c.finish(nullptr));
    HostCall &c = f.c;
    const long long groups = f.groups;
    uint8_t *chars = nullptr;
    long long *offsets = nullptr;
    std::array<unsigned long long *, 2> cols{};     // the groups' global rows and their counts
    f.send_keys(chars, offsets, cols, [](auto &s) { return std::array{s.grp, s.grp + s.live}; });
    f.wait_root();
    const long long *rows = (const long long *)cols[0];
    const unsigned long long *weight = cols[1];
    const int rc = value_counts_tail(c, groups, rep_rows_out, counts_out, capacity, ndistinct, timing,
        [&](unsigned long long *slots_keys, unsigned long long *counts, unsigned long long slots, unsigned long long *out, size_t out_n) {
            lo::k_hash_sum_str<<<grid_for(root, groups), 256, 0, c.s>>>(chars, offsets, weight, groups, slots_keys,
                                                                         counts, slots - 1);
            lo::k_hash_compact_str<<<root->sm_count * 8, 256, 0, c.s>>>(slots_keys, counts, slots, (long long *)out,
                                                                         out + out_n, (unsigned long long)out_n,
                                                                         out + 2 * out_n);
            lo::k_take_rows<<<root->sm_count * 8, 256, 0, c.s>>>((long long *)out, rows, out + 2 * out_n,
                                                                  (unsigned long long)out_n);
        }, 3);
    return f.finish(rc);
}

}  // extern "C"

// ---- dictionary codes of resident text columns (lo_text_codes, lo_text_codes_shards) ------------------------------
namespace {

// The output of a codes call on text column t: column `col` of an LO_I32 table of t->n rows on t's device.
int check_codes_out(const lo_text *t, const lo_table *out, int32_t col, const char *name) {
    if (!out) return fail(LO_ERR_INVALID, "%s is NULL", name);
    if (out->dtype != LO_I32) return fail(LO_ERR_INVALID, "%s: dtype %d is not LO_I32", name, out->dtype);
    if (col < 0 || col >= out->ncols) return fail(LO_ERR_INVALID, "%s: column %d outside [0, %d)", name, col, out->ncols);
    if (out->nrows != t->n)
        return fail(LO_ERR_INVALID, "%s has %lld rows, its text column %lld", name, (long long)out->nrows, (long long)t->n);
    if (out->device != t->ctx->device)
        return fail(LO_ERR_INVALID, "%s lives on device %d, its text column on %d", name, out->device, t->ctx->device);
    return LO_OK;
}

int *codes_col(const lo_table *out, int32_t col) { return (int *)(out->base + (int64_t)col * out->pitch); }

// the bits a radix sort of rows up to max_row orders (at least 1)
int row_bits(int64_t max_row) {
    int b = 1;
    while (b < 63 && (max_row >> b)) ++b;
    return b;
}

// a table of at least twice as many slots as groups, 1024 or more (count_groups' sizing)
unsigned long long slots_for(int64_t groups) {
    unsigned long long s = 1024;
    while (s < 2ull * (unsigned long long)groups) s <<= 1;
    return s;
}

// One column's table of a codes call and the groups listed from it
struct CodesTable {
    unsigned long long *keys = nullptr;       // the slot words
    unsigned long long *first = nullptr;      // per slot: k_hash_count_str's counts, then the first row, then the code
    unsigned long long nslots = 0;
    unsigned long long *grp_first = nullptr;  // k_compact_first: the groups' first rows [0, cap), their number at [cap]
    unsigned *grp_slot = nullptr;             // and their slots
};

// The column's half of a codes call on c's stream, for a text column of n rows, `live` of them not null: the table
// k_hash_count_str builds, the slot pass into `codes` and the compaction of the occupied slots with their first rows.
// Three launches.
void codes_slots(HostCall &c, const TextCols &t, int64_t n, int64_t live, int *codes, CodesTable &T) {
    T.nslots = slots_for(live);
    const unsigned long long mask = T.nslots - 1;
    c.alloc(&T.keys, T.nslots * 8);
    c.alloc(&T.first, T.nslots * 8);
    c.alloc(&T.grp_first, (size_t)(live + 1) * 8);
    c.alloc(&T.grp_slot, (size_t)live * 4);
    c.memset(T.keys, 0xFF, T.nslots * 8);
    c.memset(T.first, 0, T.nslots * 8);
    c.memset(T.grp_first + live, 0, 8);
    c.launch(1, [&] {
        lo::k_hash_count_str<<<grid_for(c.ctx, n), 256, 0, c.s>>>(t.chars, t.offsets, n, t.mask, t.bitmap, t.bit0, T.keys,
                                                                   T.first, mask);
    });
    c.memset(T.first, 0xFF, T.nslots * 8);    // the counts are not needed: the same words keep the first rows
    c.launch(1, [&] {
        lo::k_text_slots<<<grid_for(c.ctx, n), 256, 0, c.s>>>(t.chars, t.offsets, n, t.mask, t.bitmap, t.bit0, T.keys, mask,
                                                               T.first, codes);
    });
    c.launch(1, [&] {
        lo::k_compact_first<<<c.ctx->sm_count * 8, 256, 0, c.s>>>(T.keys, T.first, T.nslots, T.grp_first, T.grp_slot,
                                                                   (unsigned long long)live, T.grp_first + live);
    });
}

// Orders nd groups (first rows and slots as k_compact_first lists them) by first row: sorted_first receives the first
// rows in code order and slot_code[slot] each group's code.  Two launches: the radix sort over the rows' low `bits`
// bits (first rows are unique per group, so no tie is left to the sort) and k_rank_slots.
void order_groups(HostCall &c, const unsigned long long *first, const unsigned *slot, int64_t nd, int bits,
                  unsigned long long *sorted_first, unsigned long long *slot_code) {
    unsigned *sorted_slot = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    c.alloc(&sorted_slot, (size_t)nd * 4);
    c.run([&] { return cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, first, sorted_first, slot, sorted_slot, nd, 0, bits, c.s); });
    c.alloc(&tmp, tmp_bytes);
    c.launch(1, [&] { return cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, first, sorted_first, slot, sorted_slot, nd, 0, bits, c.s); });
    c.launch(1, [&] { lo::k_rank_slots<<<grid_for(c.ctx, nd), 256, 0, c.s>>>(sorted_slot, nullptr, nd, slot_code); });
    c.drop(tmp);
    c.drop(sorted_slot);
}

// lo_text_codes_shards' own state of a shard
struct CodesShard {
    int *codes;                              // its column of out[i]
    CodesTable T;
    int *key_code = nullptr;                 // the global codes of its groups, copied back from the root
    cudaEvent_t taken = nullptr;             // the shard has copied its codes from the root
};

}  // namespace

extern "C" {

int lo_text_codes(lo_ctx *ctx, const lo_text *t, lo_table *out, int32_t col, int64_t *first_rows_out, int64_t capacity,
                  int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!t) return fail(LO_ERR_INVALID, "text is NULL");
    if (t->ctx != ctx) return fail(LO_ERR_INVALID, "text belongs to another context");
    LO_TRY(check_codes_out(t, out, col, "out"));
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (capacity > 0 && !first_rows_out) return fail(LO_ERR_INVALID, "NULL argument: first_rows_out with capacity > 0");
    HostCall c(ctx, "text_codes");
    int *codes = codes_col(out, col);
    const int64_t live = t->n - t->nulls;
    if (live == 0) {                         // no cell to number (n == 0 included): every row is -1
        c.memset(codes, 0xFF, (size_t)t->n * 4);
        return c.finish(timing);
    }
    CodesTable T;
    c.mark();
    codes_slots(c, t->cols, t->n, live, codes, T);
    c.mark();
    unsigned long long nd = 0, *sorted = nullptr;
    c.to_host(&nd, T.grp_first + live, 8);
    c.sync();
    c.alloc(&sorted, nd * 8);
    c.mark();
    order_groups(c, T.grp_first, T.grp_slot, (int64_t)nd, row_bits(t->n - 1), sorted, T.first);
    c.launch(1, [&] {
        lo::k_remap_codes<<<grid_for(ctx, t->n), 256, 0, c.s>>>(codes, t->n, t->cols.mask, t->cols.bitmap, t->cols.bit0, T.first);
    });
    c.mark();
    return finish_groups(c, nd, capacity, {{first_rows_out, sorted}}, ndistinct, timing);   // codes written all the same
}

// Codes of one text column cut into row-range shards, each resident on its own context (loexec.h), in the steps of
// ShardFrame, the keys' first rows made global being their weights:
//   1. each shard's table, slot pass and compaction (codes_slots); each shard packs its groups' keys;
//   2. the root copies the keys with their first rows over, merges them with k_hash_min_str (each group's lowest
//      global first row, each key's slot), compacts and orders the groups, and remaps its key slots to codes;
//   3. each shard copies its keys' codes back, writes them to its own slots (k_rank_slots) and remaps its rows.
// The root's scratch is freed after every shard has taken its codes; a shard's after the root's step 2.
int lo_text_codes_shards(lo_ctx *root, const lo_text *const *shards, const int64_t *row0, int32_t nshards,
                         lo_table *const *out, int32_t col, int64_t *first_rows_out, int64_t capacity, int64_t *ndistinct,
                         lo_host_timing *timing) {
    LO_TRY(check_shards(root, shards, row0, nshards));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    for (int i = 0; i < nshards; ++i) {
        char name[16];
        snprintf(name, sizeof name, "out[%d]", i);
        LO_TRY(check_codes_out(shards[i], out[i], col, name));
    }
    LO_TRY(check_ndistinct(capacity, ndistinct));
    if (capacity > 0 && !first_rows_out) return fail(LO_ERR_INVALID, "NULL argument: first_rows_out with capacity > 0");
    LO_TRY(check_ctx(root));
    ShardFrame<CodesShard> f(root, "text_codes_shards", shards, row0, nshards,
                             [&](int i) { return CodesShard{codes_col(out[i], col)}; });
    for (auto &s : f.sh)                     // a shard without a cell: every row is -1, no launch
        if (!s.live && f.ok()) {
            s.c->run([&] { return cudaSetDevice(s.t->ctx->device); });
            s.c->memset(s.codes, 0xFF, (size_t)s.t->n * 4);
        }
    f.each([](auto &s, HostCall &sc) { codes_slots(sc, s.t->cols, s.t->n, s.live, s.codes, s.T); });
    f.pack_keys([](auto &s) { return std::pair(s.T.grp_first, s.T.grp_first + s.live); });
    HostCall &c = f.c;
    const long long groups = f.groups;
    int64_t max_row = 0;
    for (const auto &s : f.sh)
        if (s.live) max_row = s.row0 + s.t->n - 1;
    unsigned long long nd = 0, *sorted = nullptr;
    if (f.ok() && groups > 0) {              // 2. merge and order the keys on the root
        uint8_t *chars = nullptr;
        long long *offsets = nullptr;
        std::array<unsigned long long *, 1> cols{};     // the keys' global first rows
        f.send_keys(chars, offsets, cols, [](auto &s) { return std::array{s.T.grp_first}; });
        const unsigned long long *weight = cols[0];
        unsigned *key_slot = nullptr;
        c.alloc(&key_slot, (size_t)groups * 4);
        CodesTable R;
        R.nslots = slots_for(groups);
        c.alloc(&R.keys, R.nslots * 8);
        c.alloc(&R.first, R.nslots * 8);
        c.alloc(&R.grp_first, (size_t)(groups + 1) * 8);
        c.alloc(&R.grp_slot, (size_t)groups * 4);
        c.mark();
        c.memset(R.keys, 0xFF, R.nslots * 8);
        c.memset(R.first, 0xFF, R.nslots * 8);
        c.memset(R.grp_first + groups, 0, 8);
        c.launch(1, [&] {
            lo::k_hash_min_str<<<grid_for(root, groups), 256, 0, c.s>>>(chars, offsets, weight, groups, R.keys, R.first,
                                                                         R.nslots - 1, key_slot);
        });
        c.launch(1, [&] {
            lo::k_compact_first<<<root->sm_count * 8, 256, 0, c.s>>>(R.keys, R.first, R.nslots, R.grp_first, R.grp_slot,
                                                                      (unsigned long long)groups, R.grp_first + groups);
        });
        c.mark();
        c.to_host(&nd, R.grp_first + groups, 8);
        c.sync();
        c.alloc(&sorted, nd * 8);
        c.mark();
        order_groups(c, R.grp_first, R.grp_slot, (int64_t)nd, row_bits(max_row), sorted, R.first);
        c.launch(1, [&] {   // key i's slot -> its code, in place
            lo::k_remap_codes<<<grid_for(root, groups), 256, 0, c.s>>>((int *)key_slot, groups, nullptr, nullptr, 0, R.first);
        });
        c.mark();
        f.wait_root();
        f.each([&](auto &s, HostCall &sc) {  // 3. each shard's codes back, onto its slots and rows
            const int64_t snd = (int64_t)s.nd;
            sc.alloc(&s.key_code, (size_t)snd * 4);
            sc.run([&] {
                return cudaMemcpyPeerAsync(s.key_code, s.t->ctx->device, key_slot + s.group0, root->device, (size_t)snd * 4, sc.s);
            });
            sc.run([&] { return cudaEventCreateWithFlags(&s.taken, cudaEventDisableTiming); });
            sc.run([&] { return cudaEventRecord(s.taken, sc.s); });
            sc.launch(1, [&] { lo::k_rank_slots<<<grid_for(sc.ctx, snd), 256, 0, sc.s>>>(s.T.grp_slot, s.key_code, snd, s.T.first); });
            sc.launch(1, [&] {
                lo::k_remap_codes<<<grid_for(sc.ctx, s.t->n), 256, 0, sc.s>>>(s.codes, s.t->n, s.t->cols.mask, s.t->cols.bitmap,
                                                                                s.t->cols.bit0, s.T.first);
            });
        });
        c.run([&] { return cudaSetDevice(root->device); });
        for (auto &s : f.sh)                 // the root's scratch is freed after every shard has read its codes
            if (s.taken) c.run([&] { return cudaStreamWaitEvent(c.s, s.taken, 0); });
    }
    const int rc = f.finish(f.ok() ? finish_groups(c, nd, capacity, {{first_rows_out, sorted}}, ndistinct, timing)
                                   : c.finish(nullptr));
    for (auto &s : f.sh)
        if (s.taken) cudaEventDestroy(s.taken);
    return rc;
}

// text -> number for one column of cells (R-semantics "number" cast).  chars: all cells back to back;
// offsets[i] .. offsets[i+1] delimit cell i.  values[i] = the binary64 CPython's float() returns,
// status[i] in {0 float, 1 integer-valued, 2 empty string, 3 invalid (ValueError), 4 not decidable on device}.
int lo_parse_number_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n, double *values,
                         uint8_t *status, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n == 0) return LO_OK;
    if (!values || !status) return fail(LO_ERR_INVALID, "NULL argument");
    LO_TRY(check_text_in(chars, offsets, nullptr, n, kAnyRowBits));
    LO_TRY(check_ascending(offsets, n));
    HostCall c(ctx, "parse_number");
    std::vector<int64_t> rebased;
    const TextCols d = stage_text(c, chars, offsets, nullptr, n, &rebased);
    uint8_t *d_status = nullptr;
    unsigned long long *d_val = nullptr;
    c.alloc(&d_val, (size_t)n * 8);
    c.alloc(&d_status, (size_t)n);
    c.mark();
    c.launch(1, [&] {
        const int grid = (int)std::min<int64_t>((n + 127) / 128, (int64_t)ctx->sm_count * 16);
        lo::k_parse_number<<<grid, 128, 0, c.s>>>(d.chars, d.offsets, n, d_val, d_status);
    });
    c.mark();
    c.to_host(values, d_val, (size_t)n * 8);
    c.to_host(status, d_status, (size_t)n);
    return c.finish(timing);
}

// text -> number straight into rows [row0, row0 + n) of one f64 table column: the same parse, no per-row status; the
// call's summary instead (first invalid / unsupported row, null + empty cells, all valid cells integer valued).
int lo_parse_number_to_table(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, const lo_validity *validity,
                             int64_t n, lo_table *out, int32_t col, int64_t row0, lo_parse_summary *summary,
                             lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!summary) return fail(LO_ERR_INVALID, "summary is NULL");
    *summary = lo_parse_summary{-1, -1, 0, 1, 0};
    if (!out || out->dtype != LO_F64) return fail(LO_ERR_INVALID, "output table must be LO_F64");
    LO_TRY(check_range(out, col, row0, n));
    if (n == 0) return LO_OK;
    LO_TRY(check_text_in(chars, offsets, validity, n, kAnyRowBits));
    // No check_ascending and no host rebase: a sharded parse hands every shard a slice of one offsets array, and either
    // would be one more host pass over it per shard.  The kernel rebases the offsets and reports a cell whose offsets
    // leave [offsets[0], offsets[n]] or run backwards as unsupported.
    HostCall c(ctx, "parse_number_to_table");
    const TextCols d = stage_text(c, chars, offsets, validity, n, nullptr);
    unsigned long long *d_sum = nullptr;
    c.alloc(&d_sum, 4 * 8);
    c.memset(d_sum, 0xFF, 2 * 8);
    c.memset(d_sum + 2, 0, 2 * 8);
    unsigned long long *dst = (unsigned long long *)(out->base + (int64_t)col * out->pitch) + row0;
    c.mark();
    c.launch(1, [&] {
        const int grid = (int)std::min<int64_t>((n + 127) / 128, (int64_t)ctx->sm_count * 16);
        lo::k_parse_number_to_col<<<grid, 128, 0, c.s>>>(d.chars, d.offsets, n, d.mask, d.bitmap, d.bit0, dst, d_sum);
    });
    c.mark();
    unsigned long long sum[4] = {~0ull, ~0ull, 0, 0};
    c.to_host(sum, d_sum, sizeof(sum));
    LO_TRY(c.finish(timing));
    summary->first_invalid = sum[0] < (unsigned long long)n ? (int64_t)sum[0] : -1;
    summary->first_unsupported = sum[1] < (unsigned long long)n ? (int64_t)sum[1] : -1;
    summary->nulls = (int64_t)sum[2];
    summary->all_integer = sum[3] == 0;
    return LO_OK;
}

// number -> text for one column (R-semantics "string" cast): cell lengths, an exclusive scan of them into the Arrow
// offsets, then every cell's text at its offset.  The offsets come back before the text is made, so the caller's
// capacity is checked against the exact size and the device text buffer is allocated at that size.
int lo_format_number_host(lo_ctx *ctx, const double *values, const uint8_t *status, int64_t n, int64_t *offsets,
                          uint8_t *chars, int64_t chars_capacity, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0 || chars_capacity < 0) return fail(LO_ERR_INVALID, "negative size");
    if (!offsets) return fail(LO_ERR_INVALID, "offsets is NULL");
    if (!chars && chars_capacity) return fail(LO_ERR_INVALID, "chars is NULL with chars_capacity %lld", (long long)chars_capacity);
    offsets[0] = 0;
    if (n == 0) return LO_OK;
    if (!values || !status) return fail(LO_ERR_INVALID, "NULL argument");
    HostCall c(ctx, "format_number");
    unsigned long long *d_val = nullptr, *d_bad = nullptr;
    uint8_t *d_status = nullptr, *d_chars = nullptr;
    long long *d_off = nullptr;
    void *d_tmp = nullptr;
    size_t tmp_bytes = 0;
    const int grid = (int)std::min<int64_t>((n + 127) / 128, (int64_t)ctx->sm_count * 16);
    c.run([&] { return cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_off, n + 1, c.s); });
    c.alloc(&d_val, (size_t)n * 8);
    c.alloc(&d_status, (size_t)n);
    c.alloc(&d_off, (size_t)(n + 1) * 8);
    c.alloc(&d_bad, 8);
    c.alloc(&d_tmp, tmp_bytes);
    c.to_dev(d_val, values, (size_t)n * 8);
    c.to_dev(d_status, status, (size_t)n);
    c.memset(d_bad, 0xFF, 8);
    c.memset(d_off + n, 0, 8);           // the scan's last input: offsets[n] = total
    c.mark();
    c.launch(1, [&] { lo::k_format_number_len<<<grid, 128, 0, c.s>>>(d_val, d_status, n, d_off, d_bad); });
    c.launch(1, [&] { return cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_off, n + 1, c.s); });
    c.mark();
    unsigned long long bad = ~0ull;
    c.to_host(offsets, d_off, (size_t)(n + 1) * 8);
    c.to_host(&bad, d_bad, 8);
    c.sync();
    const int64_t total = c.ok() ? offsets[n] : 0;
    if (bad >= (unsigned long long)n && chars && total <= chars_capacity && total > 0) {
        c.alloc(&d_chars, (size_t)total);
        c.mark();
        c.launch(1, [&] { lo::k_format_number_write<<<grid, 128, 0, c.s>>>(d_val, d_status, n, d_off, d_chars); });
        c.mark();
        c.to_host(chars, d_chars, (size_t)total);
    }
    LO_TRY(c.finish(timing));
    if (bad < (unsigned long long)n) {
        const long long row = (long long)bad;
        if (status[row] > LO_NUM_EMPTY)
            return fail(LO_ERR_INVALID, "row %lld: status %u is not LO_NUM_FLOAT, LO_NUM_INTEGER or LO_NUM_EMPTY", row, (unsigned)status[row]);
        return fail(LO_ERR_INVALID, "row %lld: LO_NUM_INTEGER value %.17g is not finite and integral", row, values[row]);
    }
    if (chars && total > chars_capacity)
        return fail(LO_ERR_INVALID, "the text takes %lld bytes, chars_capacity is %lld", (long long)total, (long long)chars_capacity);
    return LO_OK;
}

// lo_parse_number_to_table with a resident text column as the input: the same kernel over the column's device chars,
// offsets (rebased to 0 when it was made) and validity, so no cell crosses PCIe
int lo_parse_text_to_table(lo_ctx *ctx, const lo_text *src, lo_table *out, int32_t col, lo_parse_summary *summary,
                           lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!summary) return fail(LO_ERR_INVALID, "summary is NULL");
    *summary = lo_parse_summary{-1, -1, 0, 1, 0};
    if (!src) return fail(LO_ERR_INVALID, "text is NULL");
    if (src->ctx != ctx) return fail(LO_ERR_INVALID, "text belongs to another context");
    if (!out || out->dtype != LO_F64) return fail(LO_ERR_INVALID, "output table must be LO_F64");
    if (out->device != ctx->device) return fail(LO_ERR_INVALID, "table lives on device %d, the context on %d", out->device, ctx->device);
    LO_TRY(check_range(out, col, 0, 0));
    if (src->n != out->nrows)
        return fail(LO_ERR_INVALID, "text of %lld cells for a table of %lld rows", (long long)src->n, (long long)out->nrows);
    const int64_t n = src->n;
    if (n == 0) return LO_OK;
    HostCall c(ctx, "parse_text_to_table");
    const TextCols &d = src->cols;
    unsigned long long *d_sum = nullptr;
    c.alloc(&d_sum, 4 * 8);
    c.memset(d_sum, 0xFF, 2 * 8);
    c.memset(d_sum + 2, 0, 2 * 8);
    unsigned long long *dst = (unsigned long long *)(out->base + (int64_t)col * out->pitch);
    c.mark();
    c.launch(1, [&] {
        const int grid = (int)std::min<int64_t>((n + 127) / 128, (int64_t)ctx->sm_count * 16);
        lo::k_parse_number_to_col<<<grid, 128, 0, c.s>>>(d.chars, d.offsets, n, d.mask, d.bitmap, d.bit0, dst, d_sum);
    });
    c.mark();
    unsigned long long sum[4] = {~0ull, ~0ull, 0, 0};
    c.to_host(sum, d_sum, sizeof(sum));
    LO_TRY(c.finish(timing));
    summary->first_invalid = sum[0] < (unsigned long long)n ? (int64_t)sum[0] : -1;
    summary->first_unsupported = sum[1] < (unsigned long long)n ? (int64_t)sum[1] : -1;
    summary->nulls = (int64_t)sum[2];
    summary->all_integer = sum[3] == 0;
    return LO_OK;
}

// lo_format_number_host of one resident f64 column into a new resident text column: the statuses come from the two
// flag arrays on the device, the lengths, their scan and the text stay there; only the flags and the total cross PCIe
int lo_format_table_to_text(lo_ctx *ctx, const lo_table *in, int32_t col, const lo_validity *valid,
                            const lo_validity *is_int, lo_text **out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!out) return fail(LO_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (!in || in->dtype != LO_F64) return fail(LO_ERR_INVALID, "input table must be LO_F64");
    if (in->device != ctx->device) return fail(LO_ERR_INVALID, "table lives on device %d, the context on %d", in->device, ctx->device);
    LO_TRY(check_range(in, col, 0, 0));
    const int64_t n = in->nrows;
    if (n >> kGroupRowBits) return fail(LO_ERR_INVALID, "n = %lld: 0 to 2^%d-1 rows per text column", (long long)n, kGroupRowBits);
    for (const lo_validity *v : {valid, is_int}) {
        if (v && v->mask && v->bitmap) return fail(LO_ERR_INVALID, "validity: mask or bitmap, not both");
        if (v && v->bitmap && v->bit_offset < 0) return fail(LO_ERR_INVALID, "validity: bit_offset < 0");
    }
    std::unique_ptr<lo_text> t(new (std::nothrow) lo_text);
    if (!t) return fail(LO_ERR_NOMEM, "out of host memory");
    HostCall c(ctx, "format_table_to_text");
    const unsigned long long *d_val = (const unsigned long long *)(in->base + (int64_t)col * in->pitch);
    lo::CellFlags flags[2] = {{nullptr, nullptr, 0}, {nullptr, nullptr, 0}};
    const lo_validity *src[2] = {valid, is_int};
    for (int k = 0; k < 2; ++k) {            // the flags' host bytes, staged as stage_text stages a validity
        size_t bytes = 0;
        const uint8_t *h = validity_span(src[k], n, &bytes);
        if (!bytes) continue;
        uint8_t *d = nullptr;
        c.alloc(&d, bytes);
        c.to_dev(d, h, bytes);
        if (src[k]->mask) flags[k].mask = d;
        else flags[k] = lo::CellFlags{nullptr, d, (int)(src[k]->bit_offset & 7)};
    }
    long long *d_off = nullptr;
    unsigned long long *d_bad = nullptr;
    uint8_t *d_chars = nullptr;
    void *d_tmp = nullptr;
    size_t tmp_bytes = 0;
    const int grid = (int)std::min<int64_t>(std::max<int64_t>((n + 127) / 128, 1), (int64_t)ctx->sm_count * 16);
    c.run([&] { return cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_off, n + 1, c.s); });
    c.alloc(&d_off, (size_t)(n + 1) * 8);
    c.alloc(&d_bad, 8);
    c.alloc(&d_tmp, tmp_bytes);
    c.memset(d_bad, 0xFF, 8);
    c.memset(d_off + n, 0, 8);           // the scan's last input: offsets[n] = total
    c.mark();
    if (n) c.launch(1, [&] { lo::k_format_col_len<<<grid, 128, 0, c.s>>>(d_val, flags[0], flags[1], n, d_off, d_bad); });
    c.launch(1, [&] { return cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_off, n + 1, c.s); });
    c.mark();
    unsigned long long bad = ~0ull;
    long long total = 0;
    c.to_host(&total, d_off + n, 8);
    c.to_host(&bad, d_bad, 8);
    c.sync();
    if (bad < (unsigned long long)n) {
        double v = 0;
        c.to_host(&v, d_val + bad, 8);
        LO_TRY(c.finish(nullptr));
        return fail(LO_ERR_INVALID, "row %lld: an is_int value %.17g is not finite and integral", (long long)bad, v);
    }
    c.alloc(&d_chars, (size_t)total);
    c.mark();
    if (total > 0)
        c.launch(1, [&] { lo::k_format_col_write<<<grid, 128, 0, c.s>>>(d_val, flags[0], flags[1], n, d_off, d_chars); });
    c.mark();
    c.keep(d_off);
    c.keep(d_chars);
    LO_TRY(c.finish(timing));
    TextCols cols;
    cols.chars = d_chars;
    cols.offsets = d_off;
    *t = lo_text{ctx, cols, n, (int64_t)total, 0, (size_t)std::max<long long>(total, 1) + (size_t)(n + 1) * 8};
    *out = t.release();
    return LO_OK;
}

// a resident text column's cells back into host Arrow large_string buffers: offsets (n + 1, from 0) and the chars
int lo_text_download(lo_ctx *ctx, const lo_text *t, int64_t *offsets, uint8_t *chars, int64_t chars_capacity,
                     lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!t) return fail(LO_ERR_INVALID, "text is NULL");
    if (t->ctx != ctx) return fail(LO_ERR_INVALID, "text belongs to another context");
    if (!offsets) return fail(LO_ERR_INVALID, "offsets is NULL");
    if (chars_capacity < t->nbytes || (t->nbytes && !chars))
        return fail(LO_ERR_INVALID, "the text takes %lld bytes, chars_capacity is %lld", (long long)t->nbytes,
                    (long long)chars_capacity);
    HostCall c(ctx, "text_download");
    c.to_host(offsets, t->cols.offsets, (size_t)(t->n + 1) * 8);
    c.to_host(chars, t->cols.chars, (size_t)t->nbytes);
    return c.finish(timing);
}

// per-column min / max of the CAST fp32 values, ignoring NaN and +-inf (the range pre-pass when a
// histogram request carries no range); nfinite[j] = how many values took part
int lo_minmax_cast_host(lo_ctx *ctx, const double *const *in_cols, int64_t nrows, int32_t k, float *mins, float *maxs,
                        uint64_t *nfinite, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_host_cols((const void *const *)in_cols, nrows, k, "in_cols"));
    if (!mins || !maxs || !nfinite) return fail(LO_ERR_INVALID, "NULL argument");
    // counts buffer layout per column: [ordered-uint min][ordered-uint max][count]
    std::vector<uint64_t> tmp((size_t)k * 3);
    int rc = host_pipeline(ctx, (const void *const *)in_cols, LO_F64, nrows, k, nullptr, LO_F32, lo::kTileRows,
                           (size_t)k * 3, tmp.data(), timing, [&](lo_table *tin, lo_table *, unsigned long long *cdev, cudaStream_t cs) {
                               dim3 grid((unsigned)std::min<int64_t>((tin->nrows + 2047) / 2048, ctx->sm_count * 4), (unsigned)k);
                               lo::k_minmax_cast<<<grid, 256, 0, cs>>>(
                                   (const char *)tin->base, tin->pitch, tin->nrows, cdev);
                               LO_CUDA(launched(ctx, 1));
                               return LO_OK;
                           });
    LO_TRY(rc);
    return lo_minmax_decode(tmp.data(), k, mins, maxs, nfinite);
}

}  // extern "C"

namespace {

// a source column of lo_assemble_rows: NULL, dtype, device, column and rows checked; *p receives its descriptor
int check_assemble_src(const lo_ctx *ctx, const lo_table *t, int32_t col, int64_t n, const char *name, lo::AsmSrc *p) {
    if (!t) return fail(LO_ERR_INVALID, "%s is NULL", name);
    if (t->dtype != LO_F64 && t->dtype != LO_I32) return fail(LO_ERR_INVALID, "%s must be LO_F64 or LO_I32 (dtype %d)", name, t->dtype);
    if (t->device != ctx->device) return fail(LO_ERR_INVALID, "%s lives on device %d, the context on %d", name, t->device, ctx->device);
    if (col < 0 || col >= t->ncols) return fail(LO_ERR_INVALID, "%s: column %d outside [0, %d)", name, col, t->ncols);
    if (t->nrows != n)
        return fail(LO_ERR_INVALID, "%s has %lld rows, the first source %lld", name, (long long)t->nrows, (long long)n);
    p->p = t->base + (int64_t)col * t->pitch;
    p->i32 = t->dtype == LO_I32;
    p->vec = (uintptr_t)p->p % 16 == 0;
    return LO_OK;
}

// an LO_F32 / LO_F64 table of the feature-matrix calls: NULL, dtype (0: either float dtype), device and size checked
int check_float_table(const lo_ctx *ctx, const lo_table *t, int dtype, int64_t need, const char *name) {
    if (!t) return fail(LO_ERR_INVALID, "%s is NULL", name);
    if (dtype ? t->dtype != dtype : t->dtype != LO_F32 && t->dtype != LO_F64)
        return fail(LO_ERR_INVALID, "%s must be %s (dtype %d)", name,
                    dtype == LO_F32 ? "LO_F32" : dtype == LO_F64 ? "LO_F64" : "LO_F32 or LO_F64", t->dtype);
    if (t->device != ctx->device) return fail(LO_ERR_INVALID, "%s lives on device %d, the context on %d", name, t->device, ctx->device);
    if (t->nrows < need)
        return fail(LO_ERR_INVALID, "%s holds %lld elements, %lld needed", name, (long long)t->nrows, (long long)need);
    return LO_OK;
}

// n rows of k values at stride ld: ld >= k, n >= 0 and n * ld representable
int check_matrix_shape(int64_t ld, int32_t k, int64_t n) {
    if (ld < k) return fail(LO_ERR_INVALID, "ld = %lld is less than k = %d", (long long)ld, k);
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    if (n > 0 && ld > (INT64_MAX / 2) / n) return fail(LO_ERR_INVALID, "n * ld overflows (ld = %lld)", (long long)ld);
    return LO_OK;
}

// The lowest refused cell of a call (lo::cell_key): a word armed to ~0 on the call's stream that the kernels lower, read
// back with the call's outputs.  After c.finish, found() fills info's bad_row / bad_col when a cell was refused.
struct RefusedCell {
    unsigned long long *word = nullptr, key = ~0ull;
    void arm(HostCall &c) {
        c.alloc(&word, 8);
        c.memset(word, 0xFF, 8);
    }
    void read(HostCall &c) { if (word) c.to_host(&key, word, 8); }
    template <typename Info> bool found(int32_t k, Info *info) const {
        if (key == ~0ull) return false;
        lo::cell_of_key(key, k, &info->bad_row, &info->bad_col);
        return true;
    }
};

constexpr int64_t kAsmMaxK = 65535ll * lo::kAsmCols;    // chunks on the grid's y dimension

template <typename T>
void launch_assemble(HostCall &c, bool skip, const lo::AsmSrc *src, int k, const lo::AsmSrc &label, int64_t n, T *x,
                     int64_t ld, T *y, long long *kept, const unsigned *bits, const unsigned long long *off,
                     unsigned long long *err) {
    const dim3 grid((unsigned)((n + lo::kAsmRows - 1) / lo::kAsmRows), (unsigned)((k + lo::kAsmCols - 1) / lo::kAsmCols));
    c.launch(1, [&] {
        if (skip) lo::k_assemble_rows<T, true><<<grid, lo::kAsmThreads, 0, c.s>>>(src, k, label, n, x, ld, y, kept, bits, off, nullptr);
        else      lo::k_assemble_rows<T, false><<<grid, lo::kAsmThreads, 0, c.s>>>(src, k, label, n, x, ld, y, nullptr, nullptr, nullptr, err);
    });
}

}  // namespace

extern "C" {

int lo_assemble_rows(lo_ctx *ctx, const lo_table *const *src, const int32_t *src_col, int32_t k, const lo_table *label,
                     int32_t label_col, int32_t mode, lo_table *x, int64_t ld, lo_table *y, int64_t *kept_rows,
                     lo_assemble_info *info, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!info) return fail(LO_ERR_INVALID, "info is NULL");
    *info = lo_assemble_info{0, -1, -1, 0};
    if (!src || !src_col) return fail(LO_ERR_INVALID, "src or src_col is NULL");
    if (k < 1 || k > kAsmMaxK) return fail(LO_ERR_INVALID, "k = %d outside [1, %lld]", k, (long long)kAsmMaxK);
    if (mode != LO_INVALID_ERROR && mode != LO_INVALID_SKIP && mode != LO_INVALID_KEEP)
        return fail(LO_ERR_INVALID, "unknown mode %d", mode);
    if (!src[0]) return fail(LO_ERR_INVALID, "src[0] is NULL");
    const int64_t n = src[0]->nrows;
    std::vector<lo::AsmSrc> desc((size_t)k);
    for (int j = 0; j < k; ++j) {
        char name[24];
        snprintf(name, sizeof name, "src[%d]", j);
        LO_TRY(check_assemble_src(ctx, src[j], src_col[j], n, name, &desc[j]));
    }
    lo::AsmSrc lab = {nullptr, 0, 0};
    if (label) LO_TRY(check_assemble_src(ctx, label, label_col, n, "label", &lab));
    if (!x) return fail(LO_ERR_INVALID, "x is NULL");
    if (x->dtype != LO_F32 && x->dtype != LO_F64) return fail(LO_ERR_INVALID, "x must be LO_F32 or LO_F64 (dtype %d)", x->dtype);
    LO_TRY(check_matrix_shape(ld, k, n));
    LO_TRY(check_float_table(ctx, x, x->dtype, n * ld, "x"));
    if (!label != !y) return fail(LO_ERR_INVALID, "y and label go together");
    if (y) LO_TRY(check_float_table(ctx, y, x->dtype, n, "y"));
    HostCall c(ctx, "assemble_rows");
    if (n == 0) return c.finish(timing);
    const bool skip = mode == LO_INVALID_SKIP, err_mode = mode == LO_INVALID_ERROR;
    const int64_t ntiles = (n + lo::kAsmRows - 1) / lo::kAsmRows;
    lo::AsmSrc *d_src = nullptr;
    unsigned long long *off = nullptr;
    unsigned *bits = nullptr;
    long long *kept = nullptr;
    RefusedCell bad;
    c.alloc(&d_src, (size_t)k * sizeof(lo::AsmSrc));
    c.to_dev(d_src, desc.data(), (size_t)k * sizeof(lo::AsmSrc));
    if (err_mode) bad.arm(c);
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    if (skip) {
        c.alloc(&bits, (size_t)ntiles * lo::kAsmWords * 4);
        c.alloc(&off, (size_t)(ntiles + 1) * 8);
        if (kept_rows) c.alloc(&kept, (size_t)n * 8);
        c.memset(off + ntiles, 0, 8);
        c.run([&] { return cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, off, ntiles + 1, c.s); });
        c.alloc(&tmp, tmp_bytes);
    }
    c.mark();
    if (skip) {
        c.launch(1, [&] {
            lo::k_assemble_valid<<<(unsigned)ntiles, lo::kAsmThreads, 0, c.s>>>(d_src, k, lab, n, bits, off);
        });
        c.launch(1, [&] { return cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, off, ntiles + 1, c.s); });
    }
    if (x->dtype == LO_F32)
        launch_assemble(c, skip, d_src, k, lab, n, (float *)x->base, ld, y ? (float *)y->base : nullptr, kept, bits, off, bad.word);
    else
        launch_assemble(c, skip, d_src, k, lab, n, (double *)x->base, ld, y ? (double *)y->base : nullptr, kept, bits, off, bad.word);
    c.mark();
    unsigned long long nkept = (unsigned long long)n;
    if (skip) {
        c.to_host(&nkept, off + ntiles, 8);
        c.sync();
        if (kept_rows) c.to_host(kept_rows, kept, nkept * 8);
    }
    bad.read(c);
    LO_TRY(c.finish(timing));
    if (bad.found(k, info))
        return fail(LO_ERR_INVALID, "invalid cell (NaN or code -1) in row %lld, %s %d", (long long)info->bad_row,
                    info->bad_col == k ? "the label, source" : "source", info->bad_col);
    info->nkept = (int64_t)nkept;
    if (kept_rows && !skip)
        for (int64_t i = 0; i < n; ++i) kept_rows[i] = i;
    return LO_OK;
}

}  // extern "C"

static_assert(lo::kNbMaxClasses == LO_NB_MAX_CLASSES && lo::kNbMaxTheta == LO_NB_MAX_THETA, "loexec.h documents the caps");

namespace {

// the matrix x (n rows of k, stride ld) and, when given, its labels y of the same dtype
int check_nb_matrix(const lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const lo_table *y) {
    if (k < 1) return fail(LO_ERR_INVALID, "k = %d: at least one feature", k);
    LO_TRY(check_matrix_shape(ld, k, n));
    LO_TRY(check_float_table(ctx, x, 0, n * ld, "x"));
    if (y) LO_TRY(check_float_table(ctx, y, x->dtype, n, "y"));
    return LO_OK;
}

// a class or label table: count in [1, LO_NB_MAX_CLASSES], strictly ascending, no NaN; *direct: exactly 0 .. m-1
int check_nb_classes(const double *v, int32_t m, const char *name, int *direct) {
    if (!v) return fail(LO_ERR_INVALID, "%s is NULL", name);
    if (m < 1 || m > LO_NB_MAX_CLASSES) return fail(LO_ERR_INVALID, "%d %s outside [1, %d]", m, name, LO_NB_MAX_CLASSES);
    *direct = 1;
    for (int32_t i = 0; i < m; ++i) {
        if (v[i] != v[i] || (i > 0 && !(v[i] > v[i - 1])))
            return fail(LO_ERR_INVALID, "%s must be strictly ascending and not NaN (entry %d)", name, i);
        if (v[i] != (double)i) *direct = 0;
    }
    return LO_OK;
}

int check_nb_caps(int32_t nclasses, int32_t k) {
    if (nclasses < 1 || nclasses > LO_NB_MAX_CLASSES)
        return fail(LO_ERR_INVALID, "%d classes outside [1, %d]", nclasses, LO_NB_MAX_CLASSES);
    if ((int64_t)nclasses * k > LO_NB_MAX_THETA)
        return fail(LO_ERR_INVALID, "%d classes x %d features exceed LO_NB_MAX_THETA = %d", nclasses, k, LO_NB_MAX_THETA);
    return LO_OK;
}

// k_nb_sums over rows [row0, row1): one CTA per G * kNbRun rows, shape = {G, Q, kp, stride, vw}
template <typename T>
void launch_nb_sums(HostCall &c, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t row0, int64_t row1,
                    const double *cls, int32_t C, int direct, double *partial, unsigned long long *counts,
                    unsigned long long *err, const int (&shape)[5], int smem) {
    const int G = shape[0], Q = shape[1], kp = shape[2], stride = shape[3], vw = shape[4];
    const int64_t per_cta = (int64_t)G * lo::kNbRun, nct = (row1 - row0 + per_cta - 1) / per_cta;
    auto go = [&](auto kernel) {
        c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
        c.launch(1, [&] {
            kernel<<<(unsigned)nct, lo::kNbThreads, smem, c.s>>>((const T *)x->base, ld, k, (const T *)y->base, row0, row1,
                                                               cls, C, direct, G, Q, kp, stride, partial, counts, err);
        });
    };
    if (vw > 1) go(lo::k_nb_sums<T, 16 / (int)sizeof(T)>);
    else        go(lo::k_nb_sums<T, 1>);
}

// The m rows of `slots` partials at src added into dst (slots doubles) by k_nb_reduce levels of kNbFan, ping-ponging
// through buf[0] / buf[1] (each ceil(m / kNbFan) rows).
void nb_tree(HostCall &c, const double *src, int64_t m, size_t slots, double *dst, double *const (&buf)[2]) {
    for (int which = 0;; which ^= 1) {
        const int64_t m2 = (m + lo::kNbFan - 1) / lo::kNbFan;
        double *out = m2 == 1 ? dst : buf[which];
        const dim3 grid((unsigned)((slots + lo::kNbThreads - 1) / lo::kNbThreads), (unsigned)m2);
        c.launch(1, [&] { lo::k_nb_reduce<<<grid, lo::kNbThreads, 0, c.s>>>(src, m, (int)slots, out); });
        if (m2 == 1) return;
        src = out;
        m = m2;
    }
}

// check_ctx, then info cleared: no refused cell
int start_info(const lo_ctx *ctx, lo_nb_info *info) {
    LO_TRY(check_ctx(ctx));
    if (!info) return fail(LO_ERR_INVALID, "info is NULL");
    *info = lo_nb_info{-1, -1, 0};
    return LO_OK;
}

// The frame of the transform / evaluate entry points (lo_nb_predict, lo_lr_predict, lo_dt_predict, lo_gb_predict,
// lo_rf_predict), CO outputs per row.  Evaluate (confusion_out given) writes no rows: the kernel counts (label slot,
// prediction) into the neval x CO matrix (lo::Confusion) and lowers the refusal word for a label that is not in
// eval_labels.  Transform writes prob, pred and (when given) raw.  An entry point calls check_x, its model checks,
// check_out, opens its HostCall as call(prefix), stages its model, then stage, grid and its launch, and returns finish.
struct PredictFrame {
    const lo_table *y;
    const double *eval_labels;
    int32_t neval, CO = 0;
    int64_t *confusion_out;
    const bool eval;
    int direct = 0;
    std::string name;
    double *d_evl = nullptr;
    unsigned long long *conf = nullptr;
    RefusedCell bad;

    PredictFrame(const lo_table *y_, const double *labels, int32_t neval_, int64_t *confusion)
        : y(y_), eval_labels(labels), neval(neval_), confusion_out(confusion), eval(confusion != nullptr) {}
    // evaluate's y, then the matrix and (evaluate) its labels
    int check_x(const lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n) const {
        if (eval && !y) return fail(LO_ERR_INVALID, "evaluate needs y");
        return check_nb_matrix(ctx, x, ld, k, n, eval ? y : nullptr);
    }
    // the outputs of CO columns: evaluate's labels (confusion_out zeroed), or transform's tables (neval becomes 0)
    int check_out(const lo_ctx *ctx, int64_t n, int32_t co, const lo_table *prob, const lo_table *raw, const lo_table *pred) {
        CO = co;
        if (eval) {
            if (prob || raw || pred) return fail(LO_ERR_INVALID, "evaluate writes no rows: prob, raw and pred must be NULL");
            LO_TRY(check_nb_classes(eval_labels, neval, "eval_labels", &direct));
            std::fill(confusion_out, confusion_out + (size_t)neval * CO, (int64_t)0);
            return LO_OK;
        }
        if (y || eval_labels) return fail(LO_ERR_INVALID, "y and eval_labels go with confusion_out");
        neval = 0;
        if (n > 0 && CO > INT64_MAX / 8 / n) return fail(LO_ERR_INVALID, "n * C overflows");
        LO_TRY(check_float_table(ctx, prob, LO_F64, n * CO, "prob"));
        LO_TRY(check_float_table(ctx, pred, LO_F64, n, "pred"));
        if (raw) LO_TRY(check_float_table(ctx, raw, LO_F64, n * CO, "raw"));
        return LO_OK;
    }
    // the call's name: <prefix>_evaluate or <prefix>_predict
    const char *call(const char *prefix) {
        name = std::string(prefix) + (eval ? "_evaluate" : "_predict");
        return name.c_str();
    }
    // evaluate: the labels uploaded, the counts zeroed and the refusal word armed
    void stage(HostCall &c) {
        if (!eval) return;
        c.alloc(&d_evl, (size_t)neval * 8);
        c.alloc(&conf, (size_t)neval * CO * 8);
        c.to_dev(d_evl, eval_labels, (size_t)neval * 8);
        c.memset(conf, 0, (size_t)neval * CO * 8);
        bad.arm(c);
    }
    // The shared memory of a tree model's kernel (k_dt_predict, k_gb_predict, k_rf_predict): its model_bytes when they
    // fit lo::kDtTreeSmem beside evaluate's labels (*model_smem), then evaluate's counts when they fit too (*hist_smem);
    // returns the bytes
    int tree_smem(int64_t model_bytes, bool *model_smem, bool *hist_smem) const {
        const int64_t evl_bytes = (int64_t)neval * 8, hist_bytes = (int64_t)neval * CO * 4;
        *model_smem = model_bytes + evl_bytes <= lo::kDtTreeSmem;
        const int64_t fixed = (*model_smem ? model_bytes : 0) + evl_bytes;
        *hist_smem = eval && fixed + hist_bytes <= lo::kDtTreeSmem;
        return (int)(fixed + (*hist_smem ? hist_bytes : 0));
    }
    // CTAs of `threads` with smem bytes: as many as the SMs hold at once, at most `units`
    template <typename K> static int grid(HostCall &c, K kernel, int threads, int smem, int64_t units) {
        int per_sm = 0;
        c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
        c.run([&] { return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem); });
        return (int)std::min<int64_t>(units, (int64_t)c.ctx->sm_count * std::max(1, per_sm));
    }
    // evaluate's counts back; a refused label names its row, confusion_out zeroed
    int finish(HostCall &c, int32_t k, lo_nb_info *info, lo_host_timing *timing) {
        if (eval) c.to_host(confusion_out, conf, (size_t)neval * CO * 8);
        bad.read(c);
        LO_TRY(c.finish(timing));
        if (!bad.found(k, info)) return LO_OK;
        std::fill(confusion_out, confusion_out + (size_t)neval * CO, (int64_t)0);
        return fail(LO_ERR_INVALID, "row %lld: its label is not one of the evaluated labels", (long long)info->bad_row);
    }
};

// lo_nb_predict and lo_lr_predict: the model's C classes (lo::kLrBinomial: C = 1, two outputs per row) over every row,
// by k_nb_predict with the epilogue `mode`.  The arguments are checked here (ctx and info before).
int nb_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const double *pi, const double *theta,
               int32_t nclasses, int mode, double threshold, lo_table *prob, lo_table *raw, lo_table *pred,
               const lo_table *y, const double *eval_labels, int32_t neval, int64_t *confusion_out, lo_nb_info *info,
               lo_host_timing *timing, const char *prefix) {
    PredictFrame f(y, eval_labels, neval, confusion_out);
    LO_TRY(f.check_x(ctx, x, ld, k, n));
    const bool binomial = mode == lo::kLrBinomial;
    LO_TRY(check_nb_caps(binomial ? 2 : nclasses, k));
    if (!pi || !theta) return fail(LO_ERR_INVALID, "pi or theta is NULL");
    const int32_t C = nclasses;
    LO_TRY(f.check_out(ctx, n, binomial ? 2 : C, prob, raw, pred));
    HostCall c(ctx, f.call(prefix));
    if (n == 0) return c.finish(timing);
    // theta j-major for the blocks of classes; raws and the histogram in shared memory when they fit beside the tables
    std::vector<double> theta_t((size_t)k * C);
    for (int32_t cc = 0; cc < C; ++cc)
        for (int32_t j = 0; j < k; ++j) theta_t[(size_t)j * C + cc] = theta[(size_t)cc * k + j];
    const int64_t base = ((int64_t)k * C + C + lo::kNbTile * (lo::kNbChunk + 1) + f.neval) * 8;
    const int64_t raws_bytes = (int64_t)C * lo::kNbTile * 8, hist_bytes = (int64_t)f.neval * f.CO * 4;
    const bool raws_smem = base + raws_bytes <= lo::kNbSmemMax;
    const int64_t with_raws = base + (raws_smem ? raws_bytes : 0);
    const bool hist_smem = f.eval && with_raws + hist_bytes <= lo::kNbSmemMax;
    const int smem = (int)(with_raws + (hist_smem ? hist_bytes : 0));
    double *d_theta = nullptr, *d_pi = nullptr, *raws = nullptr;
    c.alloc(&d_theta, theta_t.size() * 8);
    c.alloc(&d_pi, (size_t)C * 8);
    c.to_dev(d_theta, theta_t.data(), theta_t.size() * 8);
    c.to_dev(d_pi, pi, (size_t)C * 8);
    f.stage(c);
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        const int grid = f.grid(c, kernel, lo::kNbTile, smem, (n + lo::kNbTile - 1) / lo::kNbTile);
        if (!raws_smem) c.alloc(&raws, (size_t)grid * raws_bytes);
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kNbTile, smem, c.s>>>((const T *)x->base, ld, k, n, d_theta, d_pi, C,
                                                     prob ? (double *)prob->base : nullptr, raw ? (double *)raw->base : nullptr,
                                                     pred ? (double *)pred->base : nullptr, y ? (const T *)y->base : nullptr,
                                                     f.d_evl, f.neval, f.direct, f.conf, raws, hist_smem ? 1 : 0,
                                                     f.bad.word, mode, threshold);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) {
        if (f.eval) go(lo::k_nb_predict<float, true>, 0.0f); else go(lo::k_nb_predict<float, false>, 0.0f);
    } else {
        if (f.eval) go(lo::k_nb_predict<double, true>, 0.0); else go(lo::k_nb_predict<double, false>, 0.0);
    }
    return f.finish(c, k, info, timing);
}

}  // namespace

extern "C" {

int lo_nb_labels(lo_ctx *ctx, const lo_table *y, int64_t n, double *labels_out, int64_t capacity, int64_t *nlabels,
                 lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    LO_TRY(check_float_table(ctx, y, 0, n, "y"));
    LO_TRY(check_ndistinct(capacity, nlabels));
    if (n == 0) return LO_OK;
    if (capacity > 0 && !labels_out) return fail(LO_ERR_INVALID, "labels_out is NULL");
    HostCall c(ctx, "nb_labels");
    const double *d_val = (const double *)y->base;
    if (y->dtype == LO_F32) {
        double *wide = nullptr;
        c.alloc(&wide, (size_t)n * 8);
        c.launch(1, [&] { lo::k_nb_widen<<<grid_for(ctx, n), 256, 0, c.s>>>((const float *)y->base, n, wide); });
        d_val = wide;
    }
    std::vector<uint64_t> counts((size_t)capacity);
    LO_TRY(value_counts_f64_tail(c, d_val, n, labels_out, counts.data(), capacity, nlabels, timing));
    std::sort(labels_out, labels_out + *nlabels, [](double a, double b) { return a < b || (b != b && a == a); });
    if (*nlabels > 0 && labels_out[*nlabels - 1] != labels_out[*nlabels - 1])
        return fail(LO_ERR_INVALID, "a label is NaN");
    return LO_OK;
}

int lo_nb_fit(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, const double *classes,
              int32_t nclasses, double *sums_out, int64_t *counts_out, lo_nb_info *info, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!info) return fail(LO_ERR_INVALID, "info is NULL");
    *info = lo_nb_info{-1, -1, 0};
    if (!y) return fail(LO_ERR_INVALID, "y is NULL");
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, y));
    LO_TRY(check_nb_caps(nclasses, k));
    int direct = 0;
    LO_TRY(check_nb_classes(classes, nclasses, "classes", &direct));
    if (!sums_out || !counts_out) return fail(LO_ERR_INVALID, "sums_out or counts_out is NULL");
    const int32_t C = nclasses;
    const size_t slots = (size_t)C * k;
    std::fill(sums_out, sums_out + slots, 0.0);
    std::fill(counts_out, counts_out + C, (int64_t)0);
    HostCall c(ctx, "nb_fit");
    if (n == 0) return c.finish(timing);
    // a 16-byte load per row and column group when every row starts 16-byte aligned; row groups as many as fit 256
    // threads and the copies' budget.  Column j of a class row at nb_col(j) (kp per row); the copy stride = 2 mod 16
    // doubles, so a warp's row groups and column groups use different banks.
    const size_t esz = x->dtype == LO_F32 ? 4 : 8;
    const int vw = (uintptr_t)x->base % 16 == 0 && (ld * (int64_t)esz) % 16 == 0 ? (int)(16 / esz) : 1;
    const int Q = (k + vw - 1) / vw, kp = lo::nb_col(Q * vw - 1) + 1;
    const int stride = C * kp + (int)(((2 - (int64_t)C * kp) % 16 + 16) % 16);
    int G = Q >= lo::kNbThreads ? 1 : lo::kNbThreads / Q;
    G = std::max(1, std::min<int>(G, lo::kNbSumsSmem / (stride * 8)));
    const int smem = G * stride * 8 + C * 8 + C * 4;
    const int shape[5] = {G, Q, kp, stride, vw};
    // Rows go in windows whose CTAs' partials fit kNbPartialBytes; each window's partials, then the windows' sums, are
    // added by the k_nb_reduce tree.  A sum thus takes at most kNbRun adds in a thread, 16 + G / 16 over the row groups
    // and kNbFan per tree level.
    const int64_t per_cta = (int64_t)G * lo::kNbRun;
    const int64_t wct = std::max<int64_t>(1, std::min<int64_t>(1 << 20, lo::kNbPartialBytes / (int64_t)(slots * 8)));
    const int64_t wrows = wct * per_cta, nw = (n + wrows - 1) / wrows;
    const int64_t nct = std::min(wct, (n + per_cta - 1) / per_cta);
    const int64_t level1 = (std::max(nct, nw) + lo::kNbFan - 1) / lo::kNbFan;
    double *d_cls = nullptr, *partial = nullptr, *wins = nullptr, *sums = nullptr, *buf[2] = {nullptr, nullptr};
    unsigned long long *counts = nullptr;
    RefusedCell bad;
    c.alloc(&d_cls, (size_t)C * 8);
    c.alloc(&partial, (size_t)nct * slots * 8);
    c.alloc(&wins, (size_t)nw * slots * 8);
    c.alloc(&buf[0], (size_t)level1 * slots * 8);
    c.alloc(&buf[1], (size_t)level1 * slots * 8);
    c.alloc(&sums, slots * 8);
    c.alloc(&counts, (size_t)C * 8);
    c.to_dev(d_cls, classes, (size_t)C * 8);
    c.memset(counts, 0, (size_t)C * 8);
    bad.arm(c);
    c.mark();
    for (int64_t w = 0; w < nw; ++w) {
        const int64_t r0 = w * wrows, r1 = std::min(n, r0 + wrows);
        if (x->dtype == LO_F32)
            launch_nb_sums<float>(c, x, ld, k, y, r0, r1, d_cls, C, direct, partial, counts, bad.word, shape, smem);
        else
            launch_nb_sums<double>(c, x, ld, k, y, r0, r1, d_cls, C, direct, partial, counts, bad.word, shape, smem);
        nb_tree(c, partial, (r1 - r0 + per_cta - 1) / per_cta, slots, wins + (size_t)w * slots, buf);
    }
    nb_tree(c, wins, nw, slots, sums, buf);
    c.mark();
    c.to_host(sums_out, sums, slots * 8);
    c.to_host(counts_out, counts, (size_t)C * 8);
    bad.read(c);
    LO_TRY(c.finish(timing));
    if (!bad.found(k, info)) return LO_OK;
    std::fill(sums_out, sums_out + slots, 0.0);
    std::fill(counts_out, counts_out + C, (int64_t)0);
    if (info->bad_col == k) return fail(LO_ERR_INVALID, "row %lld: its label is not one of the classes", (long long)info->bad_row);
    return fail(LO_ERR_INVALID, "row %lld, feature %d: negative or NaN (NaiveBayes needs values >= 0)",
                (long long)info->bad_row, info->bad_col);
}

int lo_nb_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const double *pi, const double *theta,
                  int32_t nclasses, lo_table *prob, lo_table *raw, lo_table *pred, const lo_table *y,
                  const double *eval_labels, int32_t neval, int64_t *confusion_out, lo_nb_info *info,
                  lo_host_timing *timing) {
    LO_TRY(start_info(ctx, info));
    return nb_predict(ctx, x, ld, k, n, pi, theta, nclasses, lo::kNbSoftmax, 0.0, prob, raw, pred, y, eval_labels, neval,
                      confusion_out, info, timing, "nb");
}

}  // extern "C"

static_assert(lo::kLrHist == LO_NB_MAX_CLASSES, "a label bin per class");

namespace {

// The largest power of two R <= kLrTileMax with fixed + R * per_row within kLrSmemMax; 0 when none is
int lr_rows(int64_t fixed, int64_t per_row) {
    int R = lo::kLrTileMax;
    while (R > 0 && fixed + R * per_row > lo::kLrSmemMax) R >>= 1;
    return R;
}

int lr_vw(const lo_table *x, int64_t ld) {
    const int64_t esz = x->dtype == LO_F32 ? 4 : 8;
    return (uintptr_t)x->base % 16 == 0 && (ld * esz) % 16 == 0 ? (int)(16 / esz) : 1;
}

// The shape of a stats pass over kc staged columns: one sum per column, G = 256 / kc row groups (at least 1), the min /
// max and the label bins of kLrSum beside them.  Every k fits (kc <= kLrStatCols).  R does not set a sum's order where
// G = 1, and where G > 1 it is kLrTileMax whether kLrSum's min / max are there or not.
lo::LrShape lr_stats_shape(const lo_table *x, int64_t ld, int kc, bool bins, int *smem) {
    lo::LrShape sh{};
    sh.S = kc;
    sh.kc = kc;
    sh.ks = kc | 1;
    sh.G = kc >= lo::kLrThreads ? 1 : lo::kLrThreads / kc;
    sh.vw = lr_vw(x, ld);
    const int64_t fixed = (int64_t)sh.G * kc * 8 * (bins ? 3 : 1) + (bins ? (lo::kLrHist + 1) * 4 : 0);
    const int64_t per_row = ((int64_t)sh.ks + 1) * 8;
    sh.R = lr_rows(fixed, per_row);
    *smem = (int)(fixed + sh.R * per_row);
    return sh;
}

// The shape of a loss / grad pass of a model of nc rows over k columns: S = 1 + nc (k + 1) sums in blocks of kLrBlockC x
// kLrBlockJ (plus the loss), G row groups so that about 256 threads own a block, the coefficients in shared memory when
// that leaves R >= min(32, R without them).  False when no tile fits (not within the caps: the widest, C' = 2 and
// k = 8192 in f64, fits at R = 1).
bool lr_model_shape(const lo_table *x, int64_t ld, int32_t k, int32_t nc, lo::LrShape *sh, int *smem) {
    *sh = lo::LrShape{};
    sh->S = 1 + nc * (k + 1);
    sh->kc = k;
    sh->ks = (k + 1) | 1;
    sh->vw = lr_vw(x, ld);
    sh->nbj = (k + 1 + lo::kLrBlockJ - 1) / lo::kLrBlockJ;
    sh->nb = (nc + lo::kLrBlockC - 1) / lo::kLrBlockC * sh->nbj + 1;
    sh->G = sh->nb >= lo::kLrThreads ? 1 : lo::kLrThreads / sh->nb;
    const int64_t fixed = (int64_t)sh->G * sh->S * 8, per_row = ((int64_t)sh->ks + 1 + nc + 1) * 8;
    const int64_t coef = (int64_t)nc * k * 8;
    const int bare = lr_rows(fixed, per_row), staged = lr_rows(fixed + coef, per_row);
    sh->cs = staged > 0 && staged >= std::min(32, bare) ? 1 : 0;
    sh->R = sh->cs ? staged : bare;
    *smem = (int)(fixed + (sh->cs ? coef : 0) + sh->R * per_row);
    return sh->R > 0;
}

// One pass over rows [0, n) whose CTAs each write `slots` partial sums: rows go in windows whose CTAs' partials fit
// kNbPartialBytes; launch(r0, r1, partial) runs the pass's kernel over a window, the k_nb_reduce tree adds its partials,
// then the windows' sums, into sums (device, `slots` doubles).
template <typename F>
void lr_windows(HostCall &c, int64_t n, size_t slots, double *sums, F launch) {
    const int64_t wct = std::max<int64_t>(1, std::min<int64_t>(1 << 20, lo::kNbPartialBytes / (int64_t)(slots * 8)));
    const int64_t wrows = wct * lo::kLrCtaRows, nw = (n + wrows - 1) / wrows;
    const int64_t nct = std::min(wct, (n + lo::kLrCtaRows - 1) / lo::kLrCtaRows);
    const int64_t level1 = (std::max(nct, nw) + lo::kNbFan - 1) / lo::kNbFan;
    double *partial = nullptr, *wins = nullptr, *buf[2] = {nullptr, nullptr};
    c.alloc(&partial, (size_t)nct * slots * 8);
    c.alloc(&wins, (size_t)nw * slots * 8);
    c.alloc(&buf[0], (size_t)level1 * slots * 8);
    c.alloc(&buf[1], (size_t)level1 * slots * 8);
    for (int64_t w = 0; w < nw; ++w) {
        const int64_t r0 = w * wrows, r1 = std::min(n, r0 + wrows);
        launch(r0, r1, partial);
        nb_tree(c, partial, (r1 - r0 + lo::kLrCtaRows - 1) / lo::kLrCtaRows, slots, wins + (size_t)w * slots, buf);
    }
    nb_tree(c, wins, nw, slots, sums, buf);
}

// one k_lr_stats pass over rows [0, n): sums (device, k doubles) of x (PASS kLrSum: also the columns' min / max in ext,
// the label bins and the refused cell) or of (x - mean)^2
template <typename T, int PASS>
void lr_stats_pass(HostCall &c, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, const double *mean,
                   double *sums, unsigned long long *hist, unsigned long long *ext, unsigned long long *err) {
    int smem = 0;
    const int kc = std::min<int>(k, lo::kLrStatCols);
    const lo::LrShape sh = lr_stats_shape(x, ld, kc, PASS == lo::kLrSum, &smem);
    auto kernel = lo::k_lr_stats<T, PASS>;
    c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
    lr_windows(c, n, (size_t)k, sums, [&](int64_t r0, int64_t r1, double *partial) {
        const dim3 grid((unsigned)((r1 - r0 + lo::kLrCtaRows - 1) / lo::kLrCtaRows), (unsigned)((k + kc - 1) / kc));
        c.launch(1, [&] {
            kernel<<<grid, lo::kLrThreads, smem, c.s>>>((const T *)x->base, ld, k, (const T *)y->base, r0, r1, mean, sh,
                                                        partial, hist, ext, err);
        });
    });
}

template <typename T, bool MULTI>
void lr_loss_grad_pass(HostCall &c, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n,
                       const double *coef, const double *icpt, int32_t nc, const lo::LrShape &sh, int smem,
                       double *sums) {
    const int S = sh.S;
    auto kernel = lo::k_lr_loss_grad<T, MULTI>;
    c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
    lr_windows(c, n, (size_t)S, sums, [&](int64_t r0, int64_t r1, double *partial) {
        const unsigned grid = (unsigned)((r1 - r0 + lo::kLrCtaRows - 1) / lo::kLrCtaRows);
        c.launch(1, [&] {
            kernel<<<grid, lo::kLrThreads, smem, c.s>>>((const T *)x->base, ld, k, (const T *)y->base, r0, r1, coef, icpt,
                                                        nc, sh, partial);
        });
    });
}

// the model of lo_lr_loss_grad / lo_lr_predict: C' = nclasses rows (1 when binomial) within the caps of lo_nb_predict;
// training (lo_lr_loss_grad) needs at least 2 classes when multinomial
int check_lr_model(int32_t nclasses, int32_t multinomial, int32_t k, bool training) {
    if (multinomial != 0 && multinomial != 1) return fail(LO_ERR_INVALID, "multinomial = %d: 0 or 1", multinomial);
    if (!multinomial && nclasses != 1)
        return fail(LO_ERR_INVALID, "a binomial model has one row of coefficients, not %d", nclasses);
    if (training && multinomial && nclasses < 2)
        return fail(LO_ERR_INVALID, "a multinomial model of %d class has nothing to train", nclasses);
    return check_nb_caps(multinomial ? nclasses : 2, k);
}

}  // namespace

extern "C" {

int lo_lr_stats_range(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n,
                      double *sum_out, double *m2_out, double *min_out, double *max_out, int64_t *label_counts_out,
                      lo_nb_info *info, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!info) return fail(LO_ERR_INVALID, "info is NULL");
    *info = lo_nb_info{-1, -1, 0};
    if (!y) return fail(LO_ERR_INVALID, "y is NULL");
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, y));
    if (k > LO_NB_MAX_THETA) return fail(LO_ERR_INVALID, "k = %d exceeds LO_NB_MAX_THETA = %d", k, LO_NB_MAX_THETA);
    if (!sum_out || !m2_out || !min_out || !max_out || !label_counts_out)
        return fail(LO_ERR_INVALID, "sum_out, m2_out, min_out, max_out or label_counts_out is NULL");
    auto clear = [&] {
        for (double *o : {sum_out, m2_out, min_out, max_out}) std::fill(o, o + k, 0.0);
        std::fill(label_counts_out, label_counts_out + LO_NB_MAX_CLASSES, (int64_t)0);
    };
    clear();
    HostCall c(ctx, "lr_stats");
    if (n == 0) return c.finish(timing);
    double *d_sum = nullptr, *d_mean = nullptr, *d_m2 = nullptr;
    unsigned long long *hist = nullptr, *ext = nullptr, over = 0;
    std::vector<unsigned long long> ordered((size_t)2 * k);
    RefusedCell bad;
    c.alloc(&d_sum, (size_t)k * 8);
    c.alloc(&d_mean, (size_t)k * 8);
    c.alloc(&d_m2, (size_t)k * 8);
    c.alloc(&hist, (lo::kLrHist + 1) * 8);
    c.alloc(&ext, (size_t)2 * k * 8);
    c.memset(hist, 0, (lo::kLrHist + 1) * 8);
    c.memset(ext, 0xff, (size_t)k * 8);                    // the identities: all ones for the min, 0 for the max
    c.memset(ext + k, 0, (size_t)k * 8);
    bad.arm(c);
    const bool f32 = x->dtype == LO_F32;
    c.mark();
    if (f32) lr_stats_pass<float, lo::kLrSum>(c, x, ld, k, y, n, nullptr, d_sum, hist, ext, bad.word);
    else     lr_stats_pass<double, lo::kLrSum>(c, x, ld, k, y, n, nullptr, d_sum, hist, ext, bad.word);
    c.mark();
    static_assert(sizeof(int64_t) == sizeof(unsigned long long), "the bins are read back as int64");
    c.to_host(sum_out, d_sum, (size_t)k * 8);
    c.to_host(ordered.data(), ext, (size_t)2 * k * 8);
    c.to_host(label_counts_out, hist, (size_t)lo::kLrHist * 8);
    c.to_host(&over, hist + lo::kLrHist, 8);
    bad.read(c);
    c.sync();
    if (c.ok() && bad.key == ~0ull && over == 0) {          // pass 2 about the means of pass 1
        std::vector<double> mean((size_t)k);
        for (int32_t j = 0; j < k; ++j) mean[j] = sum_out[j] / (double)n;
        c.to_dev(d_mean, mean.data(), (size_t)k * 8);
        c.mark();
        if (f32) lr_stats_pass<float, lo::kLrM2>(c, x, ld, k, y, n, d_mean, d_m2, nullptr, nullptr, nullptr);
        else     lr_stats_pass<double, lo::kLrM2>(c, x, ld, k, y, n, d_mean, d_m2, nullptr, nullptr, nullptr);
        c.mark();
        c.to_host(m2_out, d_m2, (size_t)k * 8);
    }
    LO_TRY(c.finish(timing));
    const bool refused = bad.found(k, info);
    if (!refused && over == 0) {
        // back from lo::lr_ordered; a column whose min equals its max (as doubles: -0 == +0) has m2 exactly 0, not the
        // n ulp^2 that its rounded mean sum / n leaves
        for (int32_t j = 0; j < k; ++j) {
            for (int side = 0; side < 2; ++side) {
                const unsigned long long o = ordered[(size_t)side * k + j];
                const unsigned long long b = o >> 63 ? o & ~(1ull << 63) : ~o;
                std::memcpy(side ? &max_out[j] : &min_out[j], &b, 8);
            }
            if (min_out[j] == max_out[j]) m2_out[j] = 0.0;
        }
        return LO_OK;
    }
    clear();
    if (!refused)
        return fail(LO_ERR_INVALID, "%llu rows have a label >= %d: more than LO_NB_MAX_CLASSES classes", over,
                    LO_NB_MAX_CLASSES);
    if (info->bad_col == k)
        return fail(LO_ERR_INVALID, "row %lld: its label is not an integer >= 0", (long long)info->bad_row);
    return fail(LO_ERR_INVALID, "row %lld, feature %d: NaN or infinite", (long long)info->bad_row, info->bad_col);
}

int lo_lr_stats(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, double *sum_out,
                double *m2_out, int64_t *label_counts_out, lo_nb_info *info, lo_host_timing *timing) {
    // the range's outputs for a k the call accepts (any other k is refused before they are touched)
    std::vector<double> least(k >= 1 && k <= LO_NB_MAX_THETA ? (size_t)k : 0), most(least.size());
    return lo_lr_stats_range(ctx, x, ld, k, y, n, sum_out, m2_out, least.data(), most.data(), label_counts_out, info,
                             timing);
}

int lo_lr_loss_grad(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, const double *coef,
                    const double *intercept, int32_t nclasses, int32_t multinomial, double *out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!y) return fail(LO_ERR_INVALID, "y is NULL");
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, y));
    LO_TRY(check_lr_model(nclasses, multinomial, k, true));
    if (!coef || !intercept || !out) return fail(LO_ERR_INVALID, "coef, intercept or out is NULL");
    const int32_t nc = nclasses;
    lo::LrShape sh;
    int smem = 0;
    if (!lr_model_shape(x, ld, k, nc, &sh, &smem))
        return fail(LO_ERR_INVALID, "%d classes x %d features: no tile fits the shared memory", nc, k);
    const size_t slots = 1 + (size_t)nc * (k + 1);
    std::fill(out, out + slots, 0.0);
    HostCall c(ctx, "lr_loss_grad");
    if (n == 0) return c.finish(timing);
    double *d_coef = nullptr, *d_icpt = nullptr, *d_out = nullptr;
    c.alloc(&d_coef, (size_t)nc * k * 8);
    c.alloc(&d_icpt, (size_t)nc * 8);
    c.alloc(&d_out, slots * 8);
    c.to_dev(d_coef, coef, (size_t)nc * k * 8);
    c.to_dev(d_icpt, intercept, (size_t)nc * 8);
    c.mark();
    if (x->dtype == LO_F32) {
        if (multinomial) lr_loss_grad_pass<float, true>(c, x, ld, k, y, n, d_coef, d_icpt, nc, sh, smem, d_out);
        else             lr_loss_grad_pass<float, false>(c, x, ld, k, y, n, d_coef, d_icpt, nc, sh, smem, d_out);
    } else {
        if (multinomial) lr_loss_grad_pass<double, true>(c, x, ld, k, y, n, d_coef, d_icpt, nc, sh, smem, d_out);
        else             lr_loss_grad_pass<double, false>(c, x, ld, k, y, n, d_coef, d_icpt, nc, sh, smem, d_out);
    }
    c.mark();
    c.to_host(out, d_out, slots * 8);
    return c.finish(timing);
}

int lo_lr_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const double *coef,
                  const double *intercept, int32_t nclasses, int32_t multinomial, double threshold, lo_table *prob,
                  lo_table *raw, lo_table *pred, const lo_table *y, const double *eval_labels, int32_t neval,
                  int64_t *confusion_out, lo_nb_info *info, lo_host_timing *timing) {
    LO_TRY(start_info(ctx, info));
    LO_TRY(check_lr_model(nclasses, multinomial, k, false));
    if (!multinomial && !(threshold >= 0.0 && threshold <= 1.0))
        return fail(LO_ERR_INVALID, "threshold %g outside [0, 1]", threshold);
    return nb_predict(ctx, x, ld, k, n, intercept, coef, nclasses, multinomial ? lo::kLrMultinomial : lo::kLrBinomial,
                      threshold, prob, raw, pred, y, eval_labels, neval, confusion_out, info, timing, "lr");
}

}  // extern "C"

static_assert(lo::kDtMaxBins == LO_DT_MAX_BINS && lo::kDtMaxClasses == LO_DT_MAX_CLASSES &&
              lo::kDtPassHist == LO_DT_PASS_HIST && lo::kGbWords == LO_GB_WORDS && lo::kRfMaxDraws == LO_RF_MAX_DRAWS,
              "loexec.h documents the tree's caps");

namespace {

// a table of `dtype` on the context's device holding at least `need` elements
int check_typed_table(const lo_ctx *ctx, const lo_table *t, int dtype, int64_t need, const char *name) {
    if (!t) return fail(LO_ERR_INVALID, "%s is NULL", name);
    if (t->dtype != dtype) return fail(LO_ERR_INVALID, "%s has dtype %d, %d expected", name, t->dtype, dtype);
    if (t->device != ctx->device) return fail(LO_ERR_INVALID, "%s lives on device %d, the context on %d", name, t->device, ctx->device);
    if (t->nrows < need)
        return fail(LO_ERR_INVALID, "%s holds %lld elements, %lld needed", name, (long long)t->nrows, (long long)need);
    return LO_OK;
}

// the nodes [lo, hi) of one tree: features in [-1, k), an internal node's children inside (i, hi)
int check_tree_nodes(const int32_t *feature, const int32_t *left, const int32_t *right, int32_t lo, int32_t hi, int32_t k) {
    for (int32_t i = lo; i < hi; ++i) {
        if (feature[i] < -1 || feature[i] >= k) return fail(LO_ERR_INVALID, "node %d: feature %d outside [-1, %d)", i, feature[i], k);
        if (feature[i] >= 0 && !(left[i] > i && left[i] < hi && right[i] > i && right[i] < hi))
            return fail(LO_ERR_INVALID, "node %d: children %d, %d must lie in (%d, %d)", i, left[i], right[i], i, hi);
    }
    return LO_OK;
}

// The trees of a forest of M nodes (lo_gb_predict, lo_rf_predict): tree t holds the nodes [start[t], start[t + 1]) (the
// last up to M), the first from node 0, each checked by check_tree_nodes and then, when weight is given, its weight[t]
int check_forest(const int32_t *start, int32_t ntrees, int32_t M, const int32_t *feature, const int32_t *left,
                 const int32_t *right, int32_t k, const double *weight) {
    for (int32_t t = 0; t < ntrees; ++t) {
        const int32_t lo = start[t], hi = t + 1 < ntrees ? start[t + 1] : M;
        if (t == 0 && lo != 0) return fail(LO_ERR_INVALID, "start[0] = %d: the first tree starts at node 0", lo);
        if (!(hi > lo && hi <= M)) return fail(LO_ERR_INVALID, "tree %d: nodes [%d, %d) of %d", t, lo, hi, M);
        LO_TRY(check_tree_nodes(feature, left, right, lo, hi, k));
        if (weight && !std::isfinite(weight[t])) return fail(LO_ERR_INVALID, "weight[%d] = %g is not finite", t, weight[t]);
    }
    return LO_OK;
}

// A tree's or a forest's node arrays on the device as the tree kernels read them: *ints = feature, left, right (M each)
// and start (ntrees: a forest's first nodes; 0 for one tree); *dbls = threshold (M), the per-node payload (pay values: a
// leaf value, class counts or votes) and weight (ntrees when given: GBT's forest)
void stage_nodes(HostCall &c, int32_t M, const int32_t *feature, const int32_t *left, const int32_t *right,
                 const double *threshold, const double *payload, size_t pay, int32_t ntrees, const int32_t *start,
                 const double *weight, int **ints, double **dbls) {
    const size_t nw = weight ? (size_t)ntrees : 0;
    c.alloc(ints, ((size_t)3 * M + ntrees) * 4);
    c.alloc(dbls, ((size_t)M + pay + nw) * 8);
    c.to_dev(*ints, feature, (size_t)M * 4);
    c.to_dev(*ints + M, left, (size_t)M * 4);
    c.to_dev(*ints + 2 * M, right, (size_t)M * 4);
    if (ntrees) c.to_dev(*ints + 3 * M, start, (size_t)ntrees * 4);
    c.to_dev(*dbls, threshold, (size_t)M * 8);
    c.to_dev(*dbls + M, payload, pay * 8);
    if (nw) c.to_dev(*dbls + M + pay, weight, nw * 8);
}

int check_dt_classes(int32_t nclasses) {
    if (nclasses < 1 || nclasses > LO_DT_MAX_CLASSES)
        return fail(LO_ERR_INVALID, "%d classes outside [1, LO_DT_MAX_CLASSES = %d]", nclasses, LO_DT_MAX_CLASSES);
    return LO_OK;
}

// The launch shape of a level of nnodes nodes (lo_dt_level, lo_gb_level, lo_rf_level with k its nodes' m features): a
// feature's histogram of one node takes cell = nbins * C counters of wbytes (lo_dt_level, lo_rf_level: u32 class counts;
// lo_gb_level: C = 5 u64 words); a CTA holds gn nodes x fc features of them within kDtHistSmem.  fc is a multiple of 16
// (16-byte code loads) when 16 cells fit and `vec`, else as many single features as fit (scalar loads); gn as many nodes
// as fit beside, and as keep the pass's u64 histogram within kDtPassHist.  passes = node groups, each one pass over the
// rows.
struct DtShape { int vec, fc, gn, passes, smem; };
DtShape dt_shape(int32_t k, int32_t nbins, int32_t C, int32_t nnodes, int32_t wbytes = 4, bool vec = true) {
    DtShape sh{};
    const int64_t cell = (int64_t)nbins * C * wbytes, cells = lo::kDtHistSmem / cell;
    const int64_t kpad = ((int64_t)k + lo::kDtVec - 1) / lo::kDtVec * lo::kDtVec;
    sh.vec = vec && cells >= lo::kDtVec;
    sh.fc = (int)(sh.vec ? std::min<int64_t>(kpad, cells / lo::kDtVec * lo::kDtVec) : std::min<int64_t>(k, cells));
    const int64_t by_smem = cells / sh.fc, by_pass = lo::kDtPassHist / ((int64_t)k * nbins * C * 8);
    sh.gn = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)std::max(nnodes, 1), by_smem, by_pass}));
    sh.passes = (std::max(nnodes, 1) + sh.gn - 1) / sh.gn;
    sh.smem = (int)((int64_t)sh.gn * sh.fc * cell);
    return sh;
}

template <typename K>
void dt_sort_columns(HostCall &c, const lo_table *x, int64_t ld, int64_t n, int32_t j0, int32_t kc, K *out, int32_t cap,
                     unsigned long long *count, unsigned long long *fkey, long long *fpos) {
    K *keys = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    c.alloc(&keys, (size_t)n * kc * sizeof(K));
    c.run([&] { return cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, keys, out, n, 0, (int)sizeof(K) * 8, c.s); });
    c.alloc(&tmp, tmp_bytes);
    c.mark();
    const int grid = (int)std::min<int64_t>((n * kc + lo::kDtThreads - 1) / lo::kDtThreads, (int64_t)c.ctx->sm_count * 8);
    c.launch(1, [&] {
        if constexpr (sizeof(K) == 4) lo::k_dt_keys<float><<<grid, lo::kDtThreads, 0, c.s>>>((const float *)x->base, ld, j0, kc, n, keys);
        else lo::k_dt_keys<double><<<grid, lo::kDtThreads, 0, c.s>>>((const double *)x->base, ld, j0, kc, n, keys);
    });
    for (int32_t j = 0; j < kc; ++j)
        c.launch(1, [&] {
            return cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, keys + (size_t)j * n, out + (size_t)j * n, n, 0,
                                                  (int)sizeof(K) * 8, c.s);
        });
    c.drop(keys);
    c.drop(tmp);
    const dim3 dgrid((unsigned)std::min<int64_t>((n + lo::kDtThreads - 1) / lo::kDtThreads, (int64_t)c.ctx->sm_count * 4),
                     (unsigned)kc);
    c.launch(1, [&] { lo::k_dt_distinct<K><<<dgrid, lo::kDtThreads, 0, c.s>>>(out, n, cap, count, fkey, fpos); });
    c.mark();
}

// the value of an order-preserving code (lo::dt_code), widened to f64
double dt_value(uint64_t code, bool f32) {
    if (f32) {
        const uint32_t o = (uint32_t)code, b = o >> 31 ? o & 0x7fffffffu : ~o;
        float v;
        std::memcpy(&v, &b, 4);
        return (double)v;
    }
    const uint64_t b = code >> 63 ? code & ~(1ull << 63) : ~code;
    double v;
    std::memcpy(&v, &b, 8);
    return v;
}

// The arguments every level pass checks (tree_level), in this order: k, kp, n, the code matrix, nbins, one
// node's histogram of kf features x nbins x C u64 within LO_DT_PASS_HIST, nnodes, route, the slot tables src / dst of
// `slots` entries (without src: route 0 and `roots` nodes, every row at its tree's root), the parents' splits, hist_out.
int check_level(const lo_ctx *ctx, const char *per_bin, int32_t C, const lo_table *codes, int64_t kp, int32_t k,
                int64_t n, int32_t nbins, int32_t kf, const lo_table *src, int32_t route, const lo_table *dst,
                int64_t slots, int32_t roots, int32_t nparents, const int32_t *splits, int32_t nnodes,
                const int64_t *hist_out) {
    if (k < 1) return fail(LO_ERR_INVALID, "k = %d: at least one feature", k);
    if (kp < k || kp % lo::kDtVec) return fail(LO_ERR_INVALID, "kp = %lld: a multiple of 16 >= k", (long long)kp);
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    LO_TRY(check_typed_table(ctx, codes, LO_U8, n * kp, "codes"));
    if ((uintptr_t)codes->base % 16) return fail(LO_ERR_INVALID, "codes must start 16-byte aligned");
    if (nbins < 1 || nbins > LO_DT_MAX_BINS) return fail(LO_ERR_INVALID, "nbins = %d outside [1, %d]", nbins, LO_DT_MAX_BINS);
    if ((int64_t)kf * nbins * C * 8 > LO_DT_PASS_HIST)
        return fail(LO_ERR_INVALID, "%d features x %d bins x %d %s: one node's histogram exceeds LO_DT_PASS_HIST = %lld "
                    "bytes", kf, nbins, C, per_bin, (long long)LO_DT_PASS_HIST);
    if (nnodes < 1) return fail(LO_ERR_INVALID, "nnodes = %d: at least one", nnodes);
    if (route != 0 && route != 1) return fail(LO_ERR_INVALID, "route = %d: 0 or 1", route);
    if (src) LO_TRY(check_typed_table(ctx, src, LO_I32, slots, "src"));
    else if (roots == 1 && (route || nnodes != 1))
        return fail(LO_ERR_INVALID, "without src every row is at the root: route 0, one node");
    else if (route || nnodes != roots)
        return fail(LO_ERR_INVALID, "without src every row is at its tree's root: route 0, %d nodes", roots);
    if (dst) LO_TRY(check_typed_table(ctx, dst, LO_I32, slots, "dst"));
    if (route) {
        if (nparents < 1 || !splits) return fail(LO_ERR_INVALID, "routing needs the parents' splits");
        for (int32_t p = 0; p < nparents; ++p) {
            const int32_t *s = splits + (size_t)p * 4;
            if (s[0] < 0) continue;
            if (s[0] >= k || s[1] < 0 || s[1] >= nbins || s[2] < -1 || s[2] >= nnodes || s[3] < -1 || s[3] >= nnodes)
                return fail(LO_ERR_INVALID, "split %d = (%d, %d, %d, %d) is out of range", p, s[0], s[1], s[2], s[3]);
        }
    }
    if (!hist_out) return fail(LO_ERR_INVALID, "hist_out is NULL");
    return LO_OK;
}

// the parents' splits (rows feature, bin, left, right) on the device as four arrays of np each (np 0: none)
int *level_splits(HostCall &c, int32_t np, const int32_t *splits) {
    if (!np) return nullptr;
    int *d_split = nullptr;
    std::vector<int32_t> soa((size_t)np * 4);
    for (int32_t p = 0; p < np; ++p)
        for (int f = 0; f < 4; ++f) soa[(size_t)f * np + p] = splits[(size_t)p * 4 + f];
    c.alloc(&d_split, soa.size() * 4);
    c.to_dev(d_split, soa.data(), soa.size() * 4);
    return d_split;
}

// One node-group pass of a level as tree_level hands it to its caller's launch: the grid, the shared-memory bytes and
// stream, the slots read (from, routed when how) and written (to), the parents' splits as the four arrays of
// level_splits, the node group [g0, g0 + gn), and the histogram and refusal word the kernel writes.
struct LevelPass {
    dim3 grid;
    int smem;
    cudaStream_t s;
    const int *from;
    int how;
    int *to;
    const int *sfeat, *sbin, *left, *right;
    int g0, gn;
    unsigned long long *hist, *err;
};

// The frame of one tree level (lo_dt_level, lo_gb_level, lo_rf_level): C u64 words per (node, feature, bin) of the kf
// features each node counts, in hist_out, counted one node group of the launch shape at a time.  What differs is passed
// in: kf (k, or lo_rf_level's m), the slot tables' length and roots (n and 1, or ntrees * n and ntrees), the counters'
// width wbytes and `vec` of dt_shape, `check` (the caller's checks after check_level), `prefix` shared-memory bytes
// before the histogram, and `go(c, sh, run)`, which uploads the caller's own tables and picks the kernel for run(kernel,
// launch), launch(const LevelPass &) enqueuing one pass.  run sizes the grid from occupancy over the chunks of sh.fc
// features, then per node group d_hist is zeroed, the pass enqueued and its per_node * gn words copied to hist_out.  The
// first pass routes (how = route) from src and writes dst; the later ones read the slots it wrote.  A refused cell
// (lo::cell_key; col k: the row's label or residual) zeroes hist_out and is raised as "row R: <refused>" or as a code
// >= nbins.
template <typename Check, typename Go>
int tree_level(lo_ctx *ctx, const char *name, const char *per_bin, const char *refused, int32_t C, int32_t wbytes,
               bool vec, const lo_table *codes, int64_t kp, int32_t k, int32_t kf, int64_t n, int32_t nbins,
               const lo_table *src, int32_t route, lo_table *dst, int64_t slots, int32_t roots, int32_t nparents,
               const int32_t *splits, int32_t nnodes, int64_t *hist_out, int32_t *shape_out, lo_host_timing *timing,
               int prefix, Check check, Go go) {
    LO_TRY(check_level(ctx, per_bin, C, codes, kp, k, n, nbins, kf, src, route, dst, slots, roots, nparents, splits,
                       nnodes, hist_out));
    LO_TRY(check());
    const DtShape sh = dt_shape(kf, nbins, C, nnodes, wbytes, vec);
    if (shape_out) {
        shape_out[0] = sh.vec;
        shape_out[1] = sh.fc;
        shape_out[2] = sh.gn;
        shape_out[3] = sh.passes;
    }
    if (sh.passes > 1 && !dst) return fail(LO_ERR_INVALID, "%d node groups need dst to keep the rows' slots", sh.passes);
    const size_t per_node = (size_t)kf * nbins * C;
    std::fill(hist_out, hist_out + per_node * nnodes, (int64_t)0);
    HostCall c(ctx, name);
    if (n == 0) return c.finish(timing);
    unsigned long long *d_hist = nullptr;
    RefusedCell bad;
    bad.arm(c);
    const int np = route ? nparents : 0;
    int *d_split = level_splits(c, np, splits);
    const int smem = prefix + sh.smem;
    go(c, sh, [&](auto kernel, auto launch) {
        c.alloc(&d_hist, per_node * sh.gn * 8);
        int per_sm = 0;
        c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
        c.run([&] { return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, lo::kDtThreads, smem); });
        const int nchunks = (kf + sh.fc - 1) / sh.fc;
        const int64_t want = (int64_t)c.ctx->sm_count * std::max(1, per_sm) / nchunks;
        const dim3 grid((unsigned)std::max<int64_t>(1, std::min<int64_t>((n + lo::kDtThreads - 1) / lo::kDtThreads, want)),
                        (unsigned)nchunks);
        c.mark();
        for (int pass = 0; pass < sh.passes; ++pass) {
            const int g0 = pass * sh.gn, gn = std::min(sh.gn, nnodes - g0);
            const int *from = pass == 0 ? (src ? (const int *)src->base : nullptr) : (const int *)dst->base;
            int *to = pass == 0 && dst ? (int *)dst->base : nullptr;
            c.memset(d_hist, 0, per_node * gn * 8);
            c.launch(1, [&] {
                launch(LevelPass{grid, smem, c.s, from, pass == 0 ? route : 0, to, d_split, d_split + np,
                                 d_split + 2 * np, d_split + 3 * np, g0, gn, d_hist, bad.word});
            });
            c.to_host(hist_out + per_node * g0, d_hist, per_node * gn * 8);
            c.sync();                                   // d_hist is reused by the next pass
        }
        c.mark();
    });
    bad.read(c);
    LO_TRY(c.finish(timing));
    if (bad.key == ~0ull) return LO_OK;
    std::fill(hist_out, hist_out + per_node * nnodes, (int64_t)0);
    int64_t row = 0;
    int32_t col = 0;
    lo::cell_of_key(bad.key, k, &row, &col);
    if (col == k) return fail(LO_ERR_INVALID, "row %lld: %s", (long long)row, refused);
    return fail(LO_ERR_INVALID, "row %lld, feature %d: code >= nbins = %d", (long long)row, col, nbins);
}

// lo_dt_level's and lo_rf_level's refusal of a label: "its label is not a class in [0, C)"
std::string not_a_class(int32_t C) { return "its label is not a class in [0, " + std::to_string(C) + ")"; }

// tree_level's `check` of lo_dt_level and lo_gb_level: nothing beyond check_level
int no_check() { return LO_OK; }

}  // namespace

extern "C" {

int lo_dt_sort(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, int32_t j0, int32_t kc, lo_table *keys,
               int32_t cap, int64_t *ndistinct_out, double *values_out, int64_t *counts_out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n >= (1ll << 31)) return fail(LO_ERR_INVALID, "n = %lld: CUB's sort takes fewer than 2^31 rows", (long long)n);
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, nullptr));
    if (j0 < 0 || kc < 1 || j0 + (int64_t)kc > k) return fail(LO_ERR_INVALID, "columns [%d, %d + %d) outside [0, %d)", j0, j0, kc, k);
    if (cap < 0 || cap > LO_DT_MAX_BINS + 1) return fail(LO_ERR_INVALID, "cap = %d outside [0, %d]", cap, LO_DT_MAX_BINS + 1);
    LO_TRY(check_typed_table(ctx, keys, x->dtype, n * kc, "keys"));
    if (!ndistinct_out || (cap > 0 && (!values_out || !counts_out)))
        return fail(LO_ERR_INVALID, "ndistinct_out, values_out or counts_out is NULL");
    std::fill(ndistinct_out, ndistinct_out + kc, (int64_t)0);
    HostCall c(ctx, "dt_sort");
    if (n == 0) return c.finish(timing);
    const bool f32 = x->dtype == LO_F32;
    const size_t slots = (size_t)kc * std::max(cap, 1);
    unsigned long long *count = nullptr, *fkey = nullptr;
    long long *fpos = nullptr;
    c.alloc(&count, (size_t)kc * 8);
    c.alloc(&fkey, slots * 8);
    c.alloc(&fpos, slots * 8);
    c.memset(count, 0, (size_t)kc * 8);
    if (f32) dt_sort_columns<unsigned>(c, x, ld, n, j0, kc, (unsigned *)keys->base, cap, count, fkey, fpos);
    else     dt_sort_columns<unsigned long long>(c, x, ld, n, j0, kc, (unsigned long long *)keys->base, cap, count, fkey, fpos);
    std::vector<unsigned long long> key(slots), cnt((size_t)kc);
    std::vector<long long> pos(slots);
    c.to_host(cnt.data(), count, (size_t)kc * 8);
    c.to_host(key.data(), fkey, slots * 8);
    c.to_host(pos.data(), fpos, slots * 8);
    LO_TRY(c.finish(timing));
    for (int32_t j = 0; j < kc; ++j) {
        const int64_t d = (int64_t)cnt[j];
        ndistinct_out[j] = d;
        if (d > cap) continue;
        // the run starts by position are the distinct values ascending; a run ends where the next starts
        std::vector<std::pair<long long, unsigned long long>> runs((size_t)d);
        for (int64_t i = 0; i < d; ++i) runs[i] = {pos[(size_t)j * cap + i], key[(size_t)j * cap + i]};
        std::sort(runs.begin(), runs.end());
        for (int64_t i = 0; i < d; ++i) {
            values_out[(size_t)j * cap + i] = dt_value(runs[i].second, f32);
            counts_out[(size_t)j * cap + i] = (i + 1 < d ? runs[i + 1].first : n) - runs[i].first;
        }
    }
    return LO_OK;
}

int lo_dt_rank(lo_ctx *ctx, const lo_table *keys, int64_t n, int32_t kc, int32_t m, const int32_t *cols,
               const uint64_t *probes, int64_t *lt_out, int64_t *le_out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!keys) return fail(LO_ERR_INVALID, "keys is NULL");
    if (keys->dtype != LO_F32 && keys->dtype != LO_F64) return fail(LO_ERR_INVALID, "keys must be LO_F32 or LO_F64");
    if (n < 0 || kc < 1 || m < 0) return fail(LO_ERR_INVALID, "n = %lld, kc = %d, m = %d", (long long)n, kc, m);
    LO_TRY(check_typed_table(ctx, keys, keys->dtype, n * kc, "keys"));
    if (m > 0 && (!cols || !probes || !lt_out || !le_out)) return fail(LO_ERR_INVALID, "cols, probes, lt_out or le_out is NULL");
    for (int32_t i = 0; i < m; ++i)
        if (cols[i] < 0 || cols[i] >= kc) return fail(LO_ERR_INVALID, "cols[%d] = %d outside [0, %d)", i, cols[i], kc);
    HostCall c(ctx, "dt_rank", timing != nullptr);
    if (m == 0 || n == 0) {
        std::fill(lt_out, lt_out + m, (int64_t)0);
        std::fill(le_out, le_out + m, (int64_t)0);
        return c.finish(timing);
    }
    int *d_cols = nullptr;
    unsigned long long *d_probe = nullptr;
    long long *d_lt = nullptr, *d_le = nullptr;
    c.alloc(&d_cols, (size_t)m * 4);
    c.alloc(&d_probe, (size_t)m * 8);
    c.alloc(&d_lt, (size_t)m * 8);
    c.alloc(&d_le, (size_t)m * 8);
    c.to_dev(d_cols, cols, (size_t)m * 4);
    c.to_dev(d_probe, probes, (size_t)m * 8);
    const unsigned grid = (unsigned)((m + lo::kDtThreads - 1) / lo::kDtThreads);
    c.mark();
    c.launch(1, [&] {
        if (keys->dtype == LO_F32)
            lo::k_dt_rank<unsigned><<<grid, lo::kDtThreads, 0, c.s>>>((const unsigned *)keys->base, n, m, d_cols, d_probe, d_lt, d_le);
        else
            lo::k_dt_rank<unsigned long long><<<grid, lo::kDtThreads, 0, c.s>>>((const unsigned long long *)keys->base, n, m,
                                                                               d_cols, d_probe, d_lt, d_le);
    });
    c.mark();
    c.to_host(lt_out, d_lt, (size_t)m * 8);
    c.to_host(le_out, d_le, (size_t)m * 8);
    return c.finish(timing);
}

int lo_dt_bin(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const double *thresholds,
              const int32_t *nthr, int32_t tstride, lo_table *codes, int64_t kp, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, nullptr));
    if (tstride < 1 || tstride > LO_DT_MAX_BINS - 1) return fail(LO_ERR_INVALID, "tstride = %d outside [1, %d]", tstride, LO_DT_MAX_BINS - 1);
    if (!thresholds || !nthr) return fail(LO_ERR_INVALID, "thresholds or nthr is NULL");
    for (int32_t j = 0; j < k; ++j) {
        if (nthr[j] < 0 || nthr[j] > tstride) return fail(LO_ERR_INVALID, "nthr[%d] = %d outside [0, %d]", j, nthr[j], tstride);
        for (int32_t i = 1; i < nthr[j]; ++i)
            if (!(thresholds[(size_t)j * tstride + i] >= thresholds[(size_t)j * tstride + i - 1]))
                return fail(LO_ERR_INVALID, "the thresholds of column %d are not ascending (or NaN)", j);
    }
    if (kp < k || kp % lo::kDtVec) return fail(LO_ERR_INVALID, "kp = %lld: a multiple of 16 >= k", (long long)kp);
    LO_TRY(check_typed_table(ctx, codes, LO_U8, n * kp, "codes"));
    if ((uintptr_t)codes->base % 16) return fail(LO_ERR_INVALID, "codes must start 16-byte aligned");
    HostCall c(ctx, "dt_bin");
    if (n == 0) return c.finish(timing);
    // column chunks of a multiple of 16 whose thresholds fit kDtBinSmem (at least 48 columns of 255 thresholds)
    const int kc = std::min<int>((k + lo::kDtVec - 1) / lo::kDtVec * lo::kDtVec,
                                 lo::kDtBinSmem / (tstride * 8 + 4) / lo::kDtVec * lo::kDtVec);
    const int smem = kc * tstride * 8 + kc * 4;
    double *d_thr = nullptr;
    int *d_n = nullptr;
    c.alloc(&d_thr, (size_t)k * tstride * 8);
    c.alloc(&d_n, (size_t)k * 4);
    c.to_dev(d_thr, thresholds, (size_t)k * tstride * 8);
    c.to_dev(d_n, nthr, (size_t)k * 4);
    const size_t esz = x->dtype == LO_F32 ? 4 : 8;
    const bool vec = (uintptr_t)x->base % 16 == 0 && (ld * (int64_t)esz) % 16 == 0;
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        c.run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
        const dim3 grid((unsigned)std::min<int64_t>((n * kc / (16 / esz) + lo::kDtThreads - 1) / lo::kDtThreads,
                                                    (int64_t)ctx->sm_count * 8),
                        (unsigned)((k + kc - 1) / kc));
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kDtThreads, smem, c.s>>>((const T *)x->base, ld, k, n, d_thr, d_n, tstride, kc,
                                                        (unsigned char *)codes->base, kp);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) {
        if (vec) go(lo::k_dt_bin<float, 4>, 0.0f); else go(lo::k_dt_bin<float, 1>, 0.0f);
    } else {
        if (vec) go(lo::k_dt_bin<double, 2>, 0.0); else go(lo::k_dt_bin<double, 1>, 0.0);
    }
    return c.finish(timing);
}

int lo_dt_level(lo_ctx *ctx, const lo_table *codes, int64_t kp, int32_t k, const lo_table *y, int64_t n, int32_t nbins,
                int32_t nclasses, const lo_table *src, int32_t route, lo_table *dst, int32_t nparents,
                const int32_t *splits, int32_t nnodes, int64_t *hist_out, int32_t *shape_out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    LO_TRY(check_float_table(ctx, y, 0, n, "y"));
    LO_TRY(check_dt_classes(nclasses));
    return tree_level(ctx, "dt_level", "classes", not_a_class(nclasses).c_str(), nclasses, 4, true, codes, kp, k, k, n,
                      nbins, src, route, dst, n, 1, nparents, splits, nnodes, hist_out, shape_out, timing, 0, no_check,
                      [&](HostCall &, const DtShape &sh, auto run) {
        auto go = [&](auto kernel, auto tag) {
            using T = decltype(tag);
            run(kernel, [&](const LevelPass &p) {
                kernel<<<p.grid, lo::kDtThreads, p.smem, p.s>>>((const unsigned char *)codes->base, kp, k,
                                                                (const T *)y->base, n, nbins, nclasses, p.from, p.how,
                                                                p.to, p.sfeat, p.sbin, p.left, p.right, p.g0, p.gn,
                                                                sh.fc, p.hist, p.err);
            });
        };
        if (y->dtype == LO_F32) {
            if (sh.vec) go(lo::k_dt_level<float, true>, 0.0f); else go(lo::k_dt_level<float, false>, 0.0f);
        } else {
            if (sh.vec) go(lo::k_dt_level<double, true>, 0.0); else go(lo::k_dt_level<double, false>, 0.0);
        }
    });
}

int lo_dt_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, int32_t nnodes, const int32_t *feature,
                  const double *threshold, const int32_t *left, const int32_t *right, const double *counts,
                  int32_t nclasses, lo_table *prob, lo_table *raw, lo_table *pred, const lo_table *y,
                  const double *eval_labels, int32_t neval, int64_t *confusion_out, lo_nb_info *info,
                  lo_host_timing *timing) {
    LO_TRY(start_info(ctx, info));
    PredictFrame f(y, eval_labels, neval, confusion_out);
    LO_TRY(f.check_x(ctx, x, ld, k, n));
    LO_TRY(check_dt_classes(nclasses));
    const int32_t C = nclasses, M = nnodes;
    if (M < 1 || !feature || !threshold || !left || !right || !counts)
        return fail(LO_ERR_INVALID, "a tree of %d nodes: feature, threshold, left, right and counts are needed", M);
    LO_TRY(check_tree_nodes(feature, left, right, 0, M, k));
    LO_TRY(f.check_out(ctx, n, C, prob, raw, pred));
    HostCall c(ctx, f.call("dt"));
    if (n == 0) return c.finish(timing);
    bool tree_smem, hist_smem;
    const int smem = f.tree_smem((int64_t)M * 8 + ((int64_t)3 * M + 1) / 2 * 8, &tree_smem, &hist_smem);
    int *d_int = nullptr;
    double *d_dbl = nullptr;
    stage_nodes(c, M, feature, left, right, threshold, counts, (size_t)M * C, 0, nullptr, nullptr, &d_int, &d_dbl);
    f.stage(c);
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        const int grid = f.grid(c, kernel, lo::kDtThreads, smem, (n + lo::kDtThreads - 1) / lo::kDtThreads);
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kDtThreads, smem, c.s>>>((const T *)x->base, ld, k, n, M, d_int, d_dbl, d_int + M, d_int + 2 * M,
                                                        d_dbl + M, C, tree_smem ? 1 : 0, prob ? (double *)prob->base : nullptr,
                                                        raw ? (double *)raw->base : nullptr,
                                                        pred ? (double *)pred->base : nullptr,
                                                        y ? (const T *)y->base : nullptr, f.d_evl, f.neval, f.direct, f.conf,
                                                        hist_smem ? 1 : 0, f.bad.word);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) {
        if (f.eval) go(lo::k_dt_predict<float, true>, 0.0f); else go(lo::k_dt_predict<float, false>, 0.0f);
    } else {
        if (f.eval) go(lo::k_dt_predict<double, true>, 0.0); else go(lo::k_dt_predict<double, false>, 0.0);
    }
    return f.finish(c, k, info, timing);
}

int lo_gb_level(lo_ctx *ctx, const lo_table *codes, int64_t kp, int32_t k, const lo_table *residual, int64_t n,
                int32_t nbins, const lo_table *src, int32_t route, lo_table *dst, int32_t nparents, const int32_t *splits,
                int32_t nnodes, uint64_t *words_out, int32_t *shape_out, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    LO_TRY(check_typed_table(ctx, residual, LO_F64, n, "residual"));
    return tree_level(ctx, "gb_level", "words", "its residual is NaN or outside [-4, 4]", LO_GB_WORDS, 8, true, codes, kp,
                      k, k, n, nbins, src, route, dst, n, 1, nparents, splits, nnodes,
                      reinterpret_cast<int64_t *>(words_out), shape_out, timing, 0, no_check,
                      [&](HostCall &, const DtShape &sh, auto run) {
        auto go = [&](auto kernel) {
            run(kernel, [&](const LevelPass &p) {
                kernel<<<p.grid, lo::kDtThreads, p.smem, p.s>>>((const unsigned char *)codes->base, kp, k,
                                                                (const double *)residual->base, n, nbins, p.from, p.how,
                                                                p.to, p.sfeat, p.sbin, p.left, p.right, p.g0, p.gn,
                                                                sh.fc, p.hist, p.err);
            });
        };
        if (sh.vec) go(lo::k_gb_level<true>); else go(lo::k_gb_level<false>);
    });
}

}  // extern "C"

namespace {

// a 128-bit sum of lo_gb_level's words at w (lo, hi) as an integer
__int128 gb_word(const uint64_t *w) { return (__int128)(((unsigned __int128)w[1] << 64) | w[0]); }

}  // namespace

extern "C" {

int lo_gb_stats(const uint64_t *words, int64_t nnodes, int32_t k, int32_t nbins, int32_t nsplits, double *left_out,
                double *right_out, double *total_out) {
    if (!words || !total_out || (nsplits > 0 && (!left_out || !right_out)))
        return fail(LO_ERR_INVALID, "words, left_out, right_out or total_out is NULL");
    if (nnodes < 0 || k < 1 || nbins < 1 || nbins > LO_DT_MAX_BINS || nsplits < 0 || nsplits >= nbins)
        return fail(LO_ERR_INVALID, "nnodes = %lld, k = %d, nbins = %d, nsplits = %d", (long long)nnodes, k, nbins, nsplits);
    const double scale = 0x1p-58;
    // (count, sum, sumsq) of integer sums: the count exact, Σq1 = Σ(q1 + 2^60) - 2^60 count, each rounded once
    auto put = [&](double *o, __int128 cnt, __int128 s1, __int128 s2) {
        o[0] = (double)cnt;
        o[1] = (double)(s1 - (cnt << 60)) * scale;
        o[2] = (double)s2 * scale;
    };
    const int W = LO_GB_WORDS;
    for (int64_t g = 0; g < nnodes; ++g) {
        const uint64_t *node = words + (size_t)g * k * nbins * W;
        __int128 tc = 0, t1 = 0, t2 = 0;
        for (int32_t b = 0; b < nbins; ++b) {           // every row of the node is in one bin of feature 0
            const uint64_t *w = node + (size_t)b * W;
            tc += (__int128)w[0];
            t1 += gb_word(w + 1);
            t2 += gb_word(w + 3);
        }
        put(total_out + g * 3, tc, t1, t2);
        for (int32_t j = 0; j < k && nsplits > 0; ++j) {
            __int128 lc = 0, l1 = 0, l2 = 0;
            for (int32_t i = 0; i < nsplits; ++i) {
                const uint64_t *w = node + ((size_t)j * nbins + i) * W;
                lc += (__int128)w[0];
                l1 += gb_word(w + 1);
                l2 += gb_word(w + 3);
                const size_t at = (((size_t)g * k + j) * nsplits + i) * 3;
                put(left_out + at, lc, l1, l2);
                put(right_out + at, tc - lc, t1 - l1, t2 - l2);
            }
        }
    }
    return LO_OK;
}

int lo_gb_update(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, int32_t nnodes,
                 const int32_t *feature, const double *threshold, const int32_t *left, const int32_t *right,
                 const double *value, double weight, lo_table *margin, lo_table *residual, lo_nb_info *info,
                 lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (!info) return fail(LO_ERR_INVALID, "info is NULL");
    *info = lo_nb_info{-1, -1, 0};
    if (!y) return fail(LO_ERR_INVALID, "y is NULL");
    LO_TRY(check_nb_matrix(ctx, x, ld, k, n, y));
    LO_TRY(check_typed_table(ctx, margin, LO_F64, n, "margin"));
    LO_TRY(check_typed_table(ctx, residual, LO_F64, n, "residual"));
    const int32_t M = nnodes;
    if (M < 0) return fail(LO_ERR_INVALID, "nnodes = %d is negative", M);
    if (M > 0) {
        if (!feature || !threshold || !left || !right || !value)
            return fail(LO_ERR_INVALID, "a tree of %d nodes: feature, threshold, left, right and value are needed", M);
        LO_TRY(check_tree_nodes(feature, left, right, 0, M, k));
        if (!std::isfinite(weight)) return fail(LO_ERR_INVALID, "weight %g is not finite", weight);
    }
    HostCall c(ctx, M ? "gb_update" : "gb_init");
    if (n == 0) return c.finish(timing);
    int *d_int = nullptr;
    double *d_dbl = nullptr;
    RefusedCell bad;
    bad.arm(c);
    if (M > 0) stage_nodes(c, M, feature, left, right, threshold, value, (size_t)M, 0, nullptr, nullptr, &d_int, &d_dbl);
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        int per_sm = 0;
        c.run([&] { return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, lo::kDtThreads, 0); });
        const int grid = (int)std::min<int64_t>((n + lo::kDtThreads - 1) / lo::kDtThreads,
                                                (int64_t)ctx->sm_count * std::max(1, per_sm));
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kDtThreads, 0, c.s>>>((const T *)x->base, ld, k, n, (const T *)y->base, M, d_int, d_dbl,
                                                     d_int ? d_int + M : nullptr, d_int ? d_int + 2 * M : nullptr,
                                                     d_dbl ? d_dbl + M : nullptr, weight, (double *)margin->base,
                                                     (double *)residual->base, bad.word);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) go(lo::k_gb_update<float>, 0.0f); else go(lo::k_gb_update<double>, 0.0);
    bad.read(c);
    LO_TRY(c.finish(timing));
    if (!bad.found(k, info)) return LO_OK;
    return fail(LO_ERR_INVALID, "row %lld: its label is not 0 or 1", (long long)info->bad_row);
}

int lo_gb_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, int32_t ntrees, const int32_t *start,
                  const double *weight, int32_t nnodes, const int32_t *feature, const double *threshold,
                  const int32_t *left, const int32_t *right, const double *value, lo_table *prob, lo_table *raw,
                  lo_table *pred, const lo_table *y, const double *eval_labels, int32_t neval, int64_t *confusion_out,
                  lo_nb_info *info, lo_host_timing *timing) {
    LO_TRY(start_info(ctx, info));
    PredictFrame f(y, eval_labels, neval, confusion_out);
    LO_TRY(f.check_x(ctx, x, ld, k, n));
    const int32_t M = nnodes;
    if (ntrees < 1 || M < ntrees || !start || !weight || !feature || !threshold || !left || !right || !value)
        return fail(LO_ERR_INVALID, "a forest of %d trees and %d nodes: start, weight, feature, threshold, left, right and "
                    "value are needed", ntrees, M);
    LO_TRY(check_forest(start, ntrees, M, feature, left, right, k, weight));
    LO_TRY(f.check_out(ctx, n, 2, prob, raw, pred));
    HostCall c(ctx, f.call("gb"));
    if (n == 0) return c.finish(timing);
    bool forest_smem, hist_smem;
    const int smem = f.tree_smem(((int64_t)2 * M + ntrees) * 8 + ((int64_t)3 * M + ntrees) * 4, &forest_smem, &hist_smem);
    int *d_int = nullptr;
    double *d_dbl = nullptr;
    stage_nodes(c, M, feature, left, right, threshold, value, (size_t)M, ntrees, start, weight, &d_int, &d_dbl);
    f.stage(c);
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        const int grid = f.grid(c, kernel, lo::kDtThreads, smem, (n + lo::kDtThreads - 1) / lo::kDtThreads);
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kDtThreads, smem, c.s>>>((const T *)x->base, ld, k, n, ntrees, M, d_int + 3 * M, d_dbl + 2 * M,
                                                        d_int, d_dbl, d_int + M, d_int + 2 * M, d_dbl + M,
                                                        forest_smem ? 1 : 0, prob ? (double *)prob->base : nullptr,
                                                        raw ? (double *)raw->base : nullptr,
                                                        pred ? (double *)pred->base : nullptr,
                                                        y ? (const T *)y->base : nullptr, f.d_evl, f.neval, f.direct, f.conf,
                                                        hist_smem ? 1 : 0, f.bad.word);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) {
        if (f.eval) go(lo::k_gb_predict<float, true>, 0.0f); else go(lo::k_gb_predict<float, false>, 0.0f);
    } else {
        if (f.eval) go(lo::k_gb_predict<double, true>, 0.0); else go(lo::k_gb_predict<double, false>, 0.0);
    }
    return f.finish(c, k, info, timing);
}

int lo_rf_level(lo_ctx *ctx, const lo_table *codes, int64_t kp, int32_t k, const lo_table *y, int64_t n, int64_t row0,
                int32_t nbins, int32_t nclasses, uint64_t seed, int32_t tree0, int32_t ntrees, const uint64_t *draw,
                int32_t ndraw, const int32_t *features, int32_t m, const lo_table *src, int32_t route, lo_table *dst,
                int32_t nparents, const int32_t *splits, int32_t nnodes, int64_t *hist_out, int32_t *shape_out,
                lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "n = %lld is negative", (long long)n);
    LO_TRY(check_float_table(ctx, y, 0, n, "y"));
    LO_TRY(check_dt_classes(nclasses));
    if (ntrees < 1 || tree0 < 0 || row0 < 0)
        return fail(LO_ERR_INVALID, "ntrees = %d, tree0 = %d, row0 = %lld: trees >= 1, indices >= 0", ntrees, tree0,
                    (long long)row0);
    if (n > INT64_MAX / ntrees) return fail(LO_ERR_INVALID, "ntrees * n overflows");
    if (ndraw < 1 || ndraw > LO_RF_MAX_DRAWS || !draw)
        return fail(LO_ERR_INVALID, "ndraw = %d outside [1, LO_RF_MAX_DRAWS = %d] (or draw NULL)", ndraw, LO_RF_MAX_DRAWS);
    for (int32_t j = 1; j < ndraw; ++j)
        if (draw[j] < draw[j - 1]) return fail(LO_ERR_INVALID, "draw is not ascending at %d", j);
    if (m < 1 || m > k) return fail(LO_ERR_INVALID, "m = %d features per node outside [1, k = %d]", m, k);
    auto check = [&] {
        if (!features) return fail(LO_ERR_INVALID, "features is NULL");
        for (int64_t i = 0; i < (int64_t)nnodes * m; ++i)
            if (features[i] < 0 || features[i] >= k)
                return fail(LO_ERR_INVALID, "features[%lld] = %d outside [0, %d)", (long long)i, features[i], k);
        return LO_OK;
    };
    return tree_level(ctx, "rf_level", "classes", not_a_class(nclasses).c_str(), nclasses, 4, false, codes, kp, k, m, n,
                      nbins, src, route, dst, n * ntrees, ntrees, nparents, splits, nnodes, hist_out, shape_out, timing,
                      ndraw * 8, check, [&](HostCall &c, const DtShape &sh, auto run) {
        unsigned long long *d_draw = nullptr;
        int *d_feat = nullptr;
        c.alloc(&d_draw, (size_t)ndraw * 8);
        c.alloc(&d_feat, (size_t)nnodes * m * 4);
        c.to_dev(d_draw, draw, (size_t)ndraw * 8);
        c.to_dev(d_feat, features, (size_t)nnodes * m * 4);
        auto go = [&](auto kernel, auto tag) {
            using T = decltype(tag);
            run(kernel, [&](const LevelPass &p) {
                kernel<<<p.grid, lo::kDtThreads, p.smem, p.s>>>((const unsigned char *)codes->base, kp, k,
                                                                (const T *)y->base, n, row0, nbins, nclasses,
                                                                (unsigned long long)seed, tree0, ntrees, d_draw, ndraw,
                                                                d_feat, m, p.from, p.how, p.to, p.sfeat, p.sbin, p.left,
                                                                p.right, p.g0, p.gn, sh.fc, p.hist, p.err);
            });
        };
        if (y->dtype == LO_F32) go(lo::k_rf_level<float>, 0.0f); else go(lo::k_rf_level<double>, 0.0);
    });
}

int lo_rf_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, int32_t ntrees, const int32_t *start,
                  int32_t nnodes, const int32_t *feature, const double *threshold, const int32_t *left,
                  const int32_t *right, const double *votes, int32_t nclasses, lo_table *prob, lo_table *raw,
                  lo_table *pred, const lo_table *y, const double *eval_labels, int32_t neval, int64_t *confusion_out,
                  lo_nb_info *info, lo_host_timing *timing) {
    LO_TRY(start_info(ctx, info));
    PredictFrame f(y, eval_labels, neval, confusion_out);
    LO_TRY(f.check_x(ctx, x, ld, k, n));
    LO_TRY(check_dt_classes(nclasses));
    const int32_t M = nnodes, C = nclasses;
    if (ntrees < 1 || M < ntrees || !start || !feature || !threshold || !left || !right || !votes)
        return fail(LO_ERR_INVALID, "a forest of %d trees and %d nodes: start, feature, threshold, left, right and votes "
                    "are needed", ntrees, M);
    LO_TRY(check_forest(start, ntrees, M, feature, left, right, k, nullptr));
    LO_TRY(f.check_out(ctx, n, C, prob, raw, pred));
    HostCall c(ctx, f.call("rf"));
    if (n == 0) return c.finish(timing);
    bool forest_smem, hist_smem;
    const int smem = f.tree_smem(((int64_t)M + (int64_t)M * C) * 8 + ((int64_t)3 * M + ntrees) * 4, &forest_smem,
                                 &hist_smem);
    int *d_int = nullptr;
    double *d_dbl = nullptr;
    stage_nodes(c, M, feature, left, right, threshold, votes, (size_t)M * C, ntrees, start, nullptr, &d_int, &d_dbl);
    f.stage(c);
    auto go = [&](auto kernel, auto tag) {
        using T = decltype(tag);
        const int grid = f.grid(c, kernel, lo::kDtThreads, smem, (n + lo::kDtThreads - 1) / lo::kDtThreads);
        c.mark();
        c.launch(1, [&] {
            kernel<<<grid, lo::kDtThreads, smem, c.s>>>((const T *)x->base, ld, k, n, ntrees, M, d_int + 3 * M, d_int, d_dbl,
                                                        d_int + M, d_int + 2 * M, d_dbl + M, C, forest_smem ? 1 : 0,
                                                        prob ? (double *)prob->base : nullptr,
                                                        raw ? (double *)raw->base : nullptr,
                                                        pred ? (double *)pred->base : nullptr,
                                                        y ? (const T *)y->base : nullptr, f.d_evl, f.neval, f.direct, f.conf,
                                                        hist_smem ? 1 : 0, f.bad.word);
        });
        c.mark();
    };
    if (x->dtype == LO_F32) {
        if (f.eval) go(lo::k_rf_predict<float, true>, 0.0f); else go(lo::k_rf_predict<float, false>, 0.0f);
    } else {
        if (f.eval) go(lo::k_rf_predict<double, true>, 0.0); else go(lo::k_rf_predict<double, false>, 0.0);
    }
    return f.finish(c, k, info, timing);
}

}  // extern "C"

#include "group.inc"
#include "csv.inc"

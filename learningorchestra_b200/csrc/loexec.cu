// loexec.cu — host side of libloexec.so: the C ABI declared in include/loexec.h.
//
// Nothing here computes on the CPU: every entry point either moves bytes or launches the
// sm_90a kernels in kernels.cuh.  There is no fallback path; without a Hopper device
// lo_init() fails and nothing else is callable.
#include "loexec.h"
#include "kernels.cuh"

#include <cub/device/device_scan.cuh>

#include <algorithm>
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
    std::atomic<bool> use_tma{false};   // LOEXEC_TMA=1 or lo_set_tma(): stage slabs through smem with cp.async.bulk
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

template <typename K>
int allow_smem_tma(K kernel) {
    LO_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lo::kTmaSmemBytes));
    return LO_OK;
}

int configure_kernels() {
    LO_TRY(allow_smem_tma(lo::k_project_cast_hist_tma<0, true, true>));
    LO_TRY(allow_smem_tma(lo::k_project_cast_hist_tma<1, true, true>));
    LO_TRY(allow_smem_tma(lo::k_project_cast_hist_tma<2, true, true>));
    LO_TRY(allow_smem_tma(lo::k_project_cast_hist_tma<1, false, false>));
    LO_TRY(allow_smem_tma(lo::k_project_cast_hist_tma<2, false, false>));
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
    bool fast = HIST;     // the TMA kernel's divide
    for (int j = 0; HIST && j < P.k; ++j) fast = fast && fastdiv_ok(P.w[j]);
    // LOEXEC_TMA=1: stage the slabs through shared memory with the bulk-copy engine (A/B variant, DESIGN §3.8).
    // Only full tiles; the ragged last tile of each column (and unaligned / slow-divide / group cases) keep the LDG kernel.
    if (ctx->use_tma.load(std::memory_order_relaxed) && aligned && fast == HIST && in->nrows >= lo::kTileRows && G.mode == 0) {
        const unsigned full_tiles = (unsigned)(in->nrows / lo::kTileRows);
        const unsigned long long tblocks = (unsigned long long)full_tiles * (unsigned)P.k;
        if (tblocks > 0x7fffffffull) return fail(LO_ERR_INVALID, "table too large for one launch (%llu tiles)", tblocks);
        lo::k_project_cast_hist_tma<OUT, HIST, HIST><<<(unsigned)tblocks, lo::kThreads + 32, lo::kTmaSmemBytes, s>>>(
            in->base, in->pitch, out_base, out_pitch, in->nrows, full_tiles, counts, P);
        LO_CUDA(launched(ctx, 1));
        const int64_t done = (int64_t)full_tiles * lo::kTileRows;
        if (done == in->nrows) return LO_OK;
        // the remaining rows of every column: one ragged tile each, through the regular kernel on a row-offset view
        const char *ib = in->base + done * 8;
        char *ob = out ? out->base + done * (int64_t)dtype_size(out->dtype) + (int64_t)out_col0 * out->pitch : nullptr;
        if (edges) lo::k_project_cast_hist<OUT, HIST, true, true><<<(unsigned)P.k, lo::kThreads, smem, s>>>(
                       ib, in->pitch, ob, out_pitch, in->nrows - done, 1u, counts, edges, P, kNoGroup);
        else       lo::k_project_cast_hist<OUT, HIST, true, false><<<(unsigned)P.k, lo::kThreads, smem, s>>>(
                       ib, in->pitch, ob, out_pitch, in->nrows - done, 1u, counts, edges, P, kNoGroup);
        LO_CUDA(launched(ctx, 1));
        if (et) LO_TRY(edge_used(et, s));
        return LO_OK;
    }
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

int project_cast_hist_impl(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                           lo_table *out, const lo_hist_spec *spec, uint64_t *counts_dev, cudaStream_t s,
                           const lo::GroupStep *group = nullptr) {
    if (!in) return fail(LO_ERR_INVALID, "input table is NULL");
    if (in->dtype != LO_F64) return fail(LO_ERR_INVALID, "input table must be LO_F64 (got dtype %d)", in->dtype);
    LO_TRY(check_cols(in, col_idx, k));
    int out_mode = 0;
    if (out) {
        if (out->dtype == LO_F32) out_mode = 1;
        else if (out->dtype == LO_F64) out_mode = 2;
        else return fail(LO_ERR_INVALID, "output table must be LO_F32 or LO_F64 (got dtype %d)", out->dtype);
        if (out->nrows != in->nrows) return fail(LO_ERR_INVALID, "output rows %lld != input rows %lld",
                                                  (long long)out->nrows, (long long)in->nrows);
        if (out->ncols < k) return fail(LO_ERR_INVALID, "output has %d columns, need %d", out->ncols, k);
        if (out->device != in->device) return fail(LO_ERR_INVALID, "tables live on different devices");
    }
    if (!out && !spec) return fail(LO_ERR_INVALID, "nothing to do: no output table and no histogram spec");
    std::vector<float> w;
    if (spec) {
        if (!counts_dev) return fail(LO_ERR_INVALID, "counts_dev is NULL");
        w.resize(k);
        LO_TRY(check_spec(spec, k, w.data()));
    }
    if (group && (!spec || k > lo::kMaxColsF64))
        return fail(LO_ERR_INVALID, "a group step needs a histogram spec and k <= %d (got %d)", lo::kMaxColsF64, k);
    if (in->nrows == 0 && !group) return LO_OK;
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

int hist_u8_impl(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                 uint64_t *counts_dev, cudaStream_t s, const lo::GroupStep *group = nullptr) {
    if (!in) return fail(LO_ERR_INVALID, "input table is NULL");
    if (in->dtype != LO_U8) return fail(LO_ERR_INVALID, "input table must be LO_U8 (got dtype %d)", in->dtype);
    LO_TRY(check_cols(in, col_idx, k));
    if (!counts_dev && !group) return fail(LO_ERR_INVALID, "counts_dev is NULL");
    if (group && k > lo::kMaxColsU8) return fail(LO_ERR_INVALID, "a group step takes k <= %d byte columns (got %d)", lo::kMaxColsU8, k);
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

    HostCall(lo_ctx *c, const char *call) : ctx(c), name(call), s(c->stream), launches0(c->launches.load()) {}
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
        run([&] {
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
    if (const char *e = getenv("LOEXEC_TMA")) ctx->use_tma.store(e[0] == '1');
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

int lo_set_tma(lo_ctx *ctx, int enabled) {
    if (!ctx) return fail(LO_ERR_INVALID, "ctx is NULL");
    ctx->use_tma.store(enabled != 0, std::memory_order_relaxed);
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

// The rest of lo_value_counts_*_host once the input is on the device.  count_and_compact(keys, counts, slots, out,
// out_n) launches the two kernels of the hash group-by: count into a table of `slots` slots (keys all ones, counts
// zero), then compact the groups into out[0 .. out_n) (keys) and out[out_n .. 2 out_n) (counts), at most `capacity`
// of them, and their number into out[2 out_n].  The first min(groups, capacity) of them are copied out.
template <typename CountAndCompact>
int value_counts_tail(HostCall &c, int64_t n, void *keys_out, uint64_t *counts_out, int64_t capacity, int64_t *ndistinct,
                      lo_host_timing *timing, CountAndCompact count_and_compact) {
    unsigned long long slots = 1024;
    while (slots < 2ull * (unsigned long long)n) slots <<= 1;
    const size_t out_n = (size_t)std::max<int64_t>(capacity, 1);
    unsigned long long *d_keys = nullptr, *d_counts = nullptr, *d_out = nullptr;
    c.alloc(&d_keys, slots * 8);
    c.alloc(&d_counts, slots * 8);
    c.alloc(&d_out, (2 * out_n + 1) * 8);
    c.mark();
    c.memset(d_keys, 0xFF, slots * 8);
    c.memset(d_counts, 0, slots * 8);
    c.memset(d_out + 2 * out_n, 0, 8);
    c.launch(2, [&] { count_and_compact(d_keys, d_counts, slots, d_out, out_n); });
    c.mark();
    unsigned long long nd = 0;
    c.to_host(&nd, d_out + 2 * out_n, 8);
    c.sync();
    const size_t take = (size_t)std::min<unsigned long long>(nd, (unsigned long long)capacity);
    c.to_host(keys_out, d_out, take * 8);
    c.to_host(counts_out, d_out + out_n, take * 8);
    LO_TRY(c.finish(timing));
    *ndistinct = (int64_t)nd;
    if ((int64_t)nd > capacity)
        return fail(LO_ERR_INVALID, "%llu distinct keys do not fit the caller's capacity %lld", nd, (long long)capacity);
    return LO_OK;
}

}  // namespace

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
    if (n < 0 || capacity < 0) return fail(LO_ERR_INVALID, "negative size");
    if (!ndistinct) return fail(LO_ERR_INVALID, "ndistinct is NULL");
    *ndistinct = 0;
    if (n == 0) return LO_OK;
    if (!values || (capacity > 0 && (!keys_out || !counts_out))) return fail(LO_ERR_INVALID, "NULL argument");
    HostCall c(ctx, "value_counts_f64");
    double *d_val = nullptr;
    c.alloc(&d_val, (size_t)n * 8);
    c.to_dev(d_val, values, (size_t)n * 8);
    return value_counts_tail(c, n, keys_out, counts_out, capacity, ndistinct, timing,
        [&](unsigned long long *keys, unsigned long long *counts, unsigned long long slots, unsigned long long *out, size_t out_n) {
            const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8);
            lo::k_hash_count_f64<<<grid, 256, 0, c.s>>>(d_val, n, keys, counts, slots - 1);
            lo::k_hash_compact<<<ctx->sm_count * 8, 256, 0, c.s>>>(keys, counts, slots, out, out + out_n,
                                                                    (unsigned long long)capacity, out + 2 * out_n);
        });
}

// exact value counts of one TEXT column (cells = chars[offsets[i] .. offsets[i+1])): GPU hash group-by on the bytes.
// rep_rows_out[g] = row index of one member of group g (the caller reads the key from its own cell), counts_out[g].
int lo_value_counts_str_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n, int64_t *rep_rows_out,
                             uint64_t *counts_out, int64_t capacity, int64_t *ndistinct, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0 || capacity < 0) return fail(LO_ERR_INVALID, "negative size");
    if (n > 0x7fffffffll) return fail(LO_ERR_INVALID, "at most 2^31-1 rows per call");
    if (!ndistinct) return fail(LO_ERR_INVALID, "ndistinct is NULL");
    *ndistinct = 0;
    if (n == 0) return LO_OK;
    if (!offsets || (capacity > 0 && (!rep_rows_out || !counts_out))) return fail(LO_ERR_INVALID, "NULL argument");
    const int64_t nbytes = offsets[n] - offsets[0];
    if (offsets[0] != 0 || nbytes < 0 || (nbytes > 0 && !chars)) return fail(LO_ERR_INVALID, "offsets must start at 0 and be non-decreasing");
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i + 1] < offsets[i]) return fail(LO_ERR_INVALID, "offsets must be non-decreasing (row %lld)", (long long)i);
    HostCall c(ctx, "value_counts_str");
    uint8_t *d_chars = nullptr;
    long long *d_off = nullptr;
    c.alloc(&d_chars, (size_t)nbytes);
    c.alloc(&d_off, (size_t)(n + 1) * 8);
    c.to_dev(d_chars, chars, (size_t)nbytes);
    c.to_dev(d_off, offsets, (size_t)(n + 1) * 8);
    return value_counts_tail(c, n, rep_rows_out, counts_out, capacity, ndistinct, timing,
        [&](unsigned long long *slots_keys, unsigned long long *counts, unsigned long long slots, unsigned long long *out, size_t out_n) {
            const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8);
            lo::k_hash_count_str<<<grid, 256, 0, c.s>>>(d_chars, d_off, n, slots_keys, counts, slots - 1);
            lo::k_hash_compact_str<<<ctx->sm_count * 8, 256, 0, c.s>>>(slots_keys, counts, slots, (long long *)out, out + out_n,
                                                                        (unsigned long long)capacity, out + 2 * out_n);
        });
}

// text -> number for one column of cells (R-semantics "number" cast).  chars: all cells back to back;
// offsets[i] .. offsets[i+1] delimit cell i.  values[i] = the binary64 CPython's float() returns,
// status[i] in {0 float, 1 integer-valued, 2 empty string, 3 invalid (ValueError), 4 not decidable on device}.
int lo_parse_number_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n, double *values,
                         uint8_t *status, lo_host_timing *timing) {
    LO_TRY(check_ctx(ctx));
    if (n < 0) return fail(LO_ERR_INVALID, "n < 0");
    if (n == 0) return LO_OK;
    if (!offsets || !values || !status) return fail(LO_ERR_INVALID, "NULL argument");
    const int64_t nbytes = offsets[n] - offsets[0];
    if (nbytes < 0 || (nbytes > 0 && !chars)) return fail(LO_ERR_INVALID, "bad offsets / chars");
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i + 1] < offsets[i]) return fail(LO_ERR_INVALID, "offsets must be non-decreasing (row %lld)", (long long)i);
    HostCall c(ctx, "parse_number");
    uint8_t *d_chars = nullptr, *d_status = nullptr;
    long long *d_off = nullptr;
    unsigned long long *d_val = nullptr;
    c.alloc(&d_chars, (size_t)nbytes);
    c.alloc(&d_off, (size_t)(n + 1) * 8);
    c.alloc(&d_val, (size_t)n * 8);
    c.alloc(&d_status, (size_t)n);
    c.to_dev(d_chars, chars + offsets[0], (size_t)nbytes);
    std::vector<int64_t> rel;
    const int64_t *off_src = offsets;
    if (offsets[0] != 0) {
        rel.resize(n + 1);
        for (int64_t i = 0; i <= n; ++i) rel[i] = offsets[i] - offsets[0];
        off_src = rel.data();
    }
    c.to_dev(d_off, off_src, (size_t)(n + 1) * 8);
    c.mark();
    c.launch(1, [&] {
        const int grid = (int)std::min<int64_t>((n + 127) / 128, (int64_t)ctx->sm_count * 16);
        lo::k_parse_number<<<grid, 128, 0, c.s>>>(d_chars, d_off, n, d_val, d_status);
    });
    c.mark();
    c.to_host(values, d_val, (size_t)n * 8);
    c.to_host(status, d_status, (size_t)n);
    return c.finish(timing);
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

#include "group.inc"
#include "csv.inc"

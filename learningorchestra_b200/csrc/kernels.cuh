// kernels.cuh — sm_90a device code of libloexec: projection + cast + histogram.
//
// Replaces (reference paths under /root/reference/microservices):
//   projection_image/projection.py:38-43          column subset copy        -> K1
//   data_type_handler_image/data_type_update.py:40-43  per-value cast       -> K2 (B-semantics: fp64->fp32 RNE)
//   histogram_image/histogram.py:31-36            per-field value counting  -> K3/K4
//
// Design (see DESIGN.md §3):
//   * table = columnar slabs in HBM; a work tile is (projected column j, kTileRows rows), one tile per CTA
//     (the grid de-phases itself; a persistent variant runs its CTAs in lock step).
//   * k_project_cast_hist: every thread streams 32-byte vectors (two LDG.E.128 each) of its column slab with
//     L1::no_allocate / L2::evict_first through a 2 x 5-vector register pipeline, converts, and streams the
//     result out with st.cs.  k_project_cast_hist_tma is the same tile fed by cp.async.bulk + mbarriers
//     (opt-in).
//   * histogram = PRIVATE PER-THREAD BYTE COUNTERS in shared memory, laid out so that thread t only ever
//     touches bank (t % 32): word w of thread t lives at smem word w*kThreads + t.  Increment = plain
//     LDS.U8 / IADD / STS.U8 — no bank conflicts, and the cost is independent of the value distribution (a
//     constant column is as fast as a uniform one).  A thread handles <= 255 elements per tile so a byte never
//     wraps; the CTA then folds the 256 private histograms (LDS.128, packed 16-bit adds, a transposing warp
//     butterfly) and issues one RED.64 per non-empty bin.
//   * byte columns (K4, k_hist_u8_cols_lanes) and histograms of more than 256 bins (k_project_cast_hist_bins) drop
//     the byte fields: 32-bit counters in lane slots shared by the CTA's warps, bank = lane, the counter address one
//     PRMT (bytes) or one shift-add (bins) away from the value, ONE ATOMS per element, a CTA streams a long chunk of
//     its column and folds once.
//   * several GPUs (GroupStep): the bins go to the device's own matrix; the CTA finishing a column's last tile pushes
//     the column to the root GPU with system-scope RED.64 over NVLink, the last pusher arrives, the root's last CTA
//     moves the merged matrix out — merge, arrival and epilogue ride inside the one streaming launch per step.
//   * bin index = trunc(RN((x - lo) / w)): in the tile kernel from a table of exact bin edges (one FFMA estimate, one
//     LDS.128, one comparison; edge_counter_offset), elsewhere without a divide (hoisted reciprocal + two FMA
//     corrections; bin_index_f32) — both proven and exhaustively self-tested equal to the IEEE quotient.
//   * also here: k_parse_number (CPython float() on the GPU, parse_number.cuh), k_format_number_len / _write (its
//     inverse, CPython str(), format_number.cuh), k_hash_count_f64 / _str
//     (exact group-by), k_minmax_cast, the group's small kernels (push, big-matrix merge, barrier), generators, checksum.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "parse_number.cuh"
#include "format_number.cuh"

namespace lo {

constexpr int kThreads      = 256;                 // threads per CTA
constexpr int kVec          = 4;                   // f64 elements per 32-byte vector (two 16-byte loads)
constexpr int kBatch        = 4;                   // vector loads in flight per thread
constexpr int kBatches      = 15;
constexpr int kVecPerThread = kBatch * kBatches;   // 60
constexpr int kElemsPerThread = kVec * kVecPerThread;      // 240 <= 255 (byte counter bound)
constexpr int kTileRows     = kThreads * kElemsPerThread;  // 61440 rows per tile
constexpr int kHalf         = kThreads * kVec / 2;         // second pair of a thread's vector (ldg_split4_stream)
constexpr int kHistRows     = 64;                  // smem words per thread (256 bins / 4)
constexpr int kHistSmemBytes = (kHistRows * kThreads + 256) * 4;   // 66560 B -> 3 CTAs / SM

// software pipeline of the full-tile path: kPfBuf register buffers of kPfBatch 32-byte vectors;
// kPfBuf-1 batches are always in flight per thread while one is being converted / binned
#ifndef LO_PF_BATCH
#define LO_PF_BATCH 5
#endif
#ifndef LO_PF_NBUF
#define LO_PF_NBUF 2
#endif
#ifndef LO_MIN_CTAS
#define LO_MIN_CTAS 2
#endif
constexpr int kPfBatch   = LO_PF_BATCH;
constexpr int kPfBuf     = LO_PF_NBUF;
constexpr int kPfBatches = kVecPerThread / kPfBatch;
static_assert(kVecPerThread % kPfBatch == 0 && kPfBatches % kPfBuf == 0, "pipeline shape must tile the 60 vectors");

constexpr int kU8VecBytes      = 16;
constexpr int kU8HostChunkRows = 61440;   // row granularity of the *_host byte pipeline's chunks

constexpr int kMaxColsF64   = 128;   // projected columns per launch (by-value kernel parameter)
constexpr int kMaxColsU8    = 1024;

struct ColsF64 {
    int32_t k;
    int32_t nbins;
    int32_t col[kMaxColsF64];
    float   lo[kMaxColsF64];
    float   hi[kMaxColsF64];
    float   w[kMaxColsF64];
};

struct ColsU8 {
    int32_t k;
    int32_t col[kMaxColsU8];
};

// One step of the multi-GPU histogram merge, executed INSIDE the streaming kernel (loexec.cu: lo_group_*).
// Every device accumulates into its own `local` matrix; the CTA that finishes the last tile of a column pushes
// that column's bins into the root GPU's `shared` matrix (system-scope RED.64 over NVLink / peer mapping), the CTA
// that pushes the last column release-adds the root's `arrived` counter, and on the root that same CTA waits for
// all W arrivals, moves the merged matrix to `result` (and to every peer's with bcast), re-zeroes `shared` and
// release-adds each peer's `clean` counter.  No separate flag / memset / epilogue launches: one launch per step.
constexpr int kMaxPeers = 15;
struct GroupStep {
    int mode;                          // 0: no group (plain accumulate into counts);  1: merge as described
    int is_root, npeers, epilogue_in_kernel;
    int overlap, pad_;                 // 1: launched with programmatic stream serialization: let the NEXT launch's CTAs
                                       //    take the SMs this one's tail leaves idle (LO_GROUP_INDEPENDENT)
    unsigned long long *gen;           // steps of this parity that are COMPLETE on this device: pushed, and on the root
                                       // also merged out (the root's own next push into `shared` must wait for that)
    unsigned long long gen_target;     // flush only once *gen >= gen_target (the step two launches back is done)
    unsigned long long *epi_seq;       // root: number of finished epilogues; epilogues run in step order even when
    unsigned long long step;           // their launches overlap, so `result` always ends up holding the LAST step
    unsigned long long *local;         // this device's accumulate matrix (zero at entry, left zero at exit)
    unsigned long long *shared;        // root's merge matrix of this step's parity (peer-mapped on the others)
    unsigned long long *arrived;       // root's arrival counter of this parity
    const unsigned long long *clean;   // this device's "root has re-zeroed shared" counter (nullptr on the root)
    unsigned long long clean_target;   // push only once *clean >= clean_target
    unsigned int *col_ticket;          // [k] tiles finished per column (self-resetting)
    unsigned int *done_ticket;         // columns pushed (self-resetting)
    unsigned long long arrive_target;  // root: W * (step / 2 + 1)
    unsigned long long *result;        // root: merged matrix of the finished step
    unsigned long long timeout_ns;     // bound on every wait; a lost peer raises *timed_out instead of hanging the GPU
    unsigned long long *timed_out;
    unsigned long long *peer_clean[kMaxPeers];    // root: the peers' clean counters
    unsigned long long *peer_result[kMaxPeers];   // root: the peers' result matrices (bcast), else nullptr
};

// ---------------------------------------------------------------------------------------------
// streaming memory ops
// ---------------------------------------------------------------------------------------------
// sm_90 loads and stores at most 16 bytes per thread.  A thread's four f64 of a CTA-wide block are therefore two pairs:
// {p[0], p[1]} and {p[half], p[half + 1]} with p = block + 2 * tid and half = 2 * threads, so each instruction of a warp
// covers 512 contiguous bytes (the layout the TMA kernel reads from its staging ring).  On sm_90 the L2 evict-first
// priority of 128-bit loads is an L2::cache_hint policy operand.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void ldg_split4_stream(const double *p, long long half, double (&v)[4]) {
    const uint64_t pol = l2_evict_first_policy();
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
                 : "=d"(v[0]), "=d"(v[1]) : "l"(p), "l"(pol));
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
                 : "=d"(v[2]), "=d"(v[3]) : "l"(p + half), "l"(pol));
}
__device__ __forceinline__ double ldg64_stream(const double *p) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ldg128_stream(const uint8_t *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ldg8_stream(const uint8_t *p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
// the stores matching ldg_split4_stream: {a, b} at p, {c, d} at p + half
__device__ __forceinline__ void stg_split4_stream(float *p, long long half, float a, float b, float c, float d) {
    asm volatile("st.global.cs.v2.f32 [%0], {%1,%2};" :: "l"(p), "f"(a), "f"(b) : "memory");
    asm volatile("st.global.cs.v2.f32 [%0], {%1,%2};" :: "l"(p + half), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void stg_split4_stream(double *p, long long half, const double (&v)[4]) {
    asm volatile("st.global.cs.v2.f64 [%0], {%1,%2};" :: "l"(p), "d"(v[0]), "d"(v[1]) : "memory");
    asm volatile("st.global.cs.v2.f64 [%0], {%1,%2};" :: "l"(p + half), "d"(v[2]), "d"(v[3]) : "memory");
}

// ---------------------------------------------------------------------------------------------
// element semantics (the CPU twins are oracle/bsem.c and oracle/bsem_numpy.py)
// ---------------------------------------------------------------------------------------------
// fp64 -> fp32 round-to-nearest-even; every NaN becomes the canonical quiet NaN 0x7fc00000.
__device__ __forceinline__ float cast_f64_f32(double x) {
    float f = __double2float_rn(x);
    return (f != f) ? __int_as_float(0x7fc00000) : f;
}

// byte offset of bin b inside a thread's private histogram (before OR-ing in 4*tid):
// word row (b >> 2) at stride kThreads words, byte (b & 3).  For kThreads == 256 the row
// offset is (b & 0xFC) << 8, so offset = (b * 0x101) & 0xFC03 and never overlaps 4*tid (bits 2..9).
static_assert(kThreads == 256, "private histogram addressing assumes 256 threads");
__device__ __forceinline__ uint32_t bin_byte_offset(uint32_t b) { return (b * 0x101u) & 0xFC03u; }

__device__ __forceinline__ void bump(uint8_t *priv /* smem + 4*tid */, uint32_t b) {
    uint8_t *p = priv + bin_byte_offset(b);
    *p = (uint8_t)(*p + 1);
}

// fixed-width binning of the CAST value (SURVEY.md §8c): fp32 RN subtract, fp32 RN divide,
// truncate, close the last bin.  NaN and out-of-range values are skipped (bin index < 0).
//
// FASTDIV = false: the divide is the compiler's IEEE __fdiv_rn (MUFU.RCP + Newton + FCHK slow path).
// FASTDIV = true : the same correctly-rounded quotient without the XU op and without the branch,
//   using the reciprocal r = RN(1/w) computed once per CTA:
//       q0 = RN(d*r); q1 = RN(q0 + (d - w*q0)*r); q2 = RN(q1 + (d - w*q1)*r)      (remainders exact in FMA)
//   q2 == RN(d/w) whenever d >= w/2 (Markstein's theorem; the one exception, a divisor whose
//   significand is all ones, and exponents that could under/overflow an intermediate are excluded by
//   the host, which then launches the FASTDIV = false variant — see fastdiv_ok() in loexec.cu and
//   DESIGN.md §3.3).  For d < w/2 every q stays below 1, so the truncated bin is 0 either way.
//   The truncation is an FADD.RZ against 2^23 (integer part lands in the low significand bits)
//   instead of an F2I, which would be another XU-pipe op.
struct BinParams {
    float lo, hi, w, r;
    int   last;
};

template <bool FASTDIV>
__device__ __forceinline__ int bin_index_f32(float f, const BinParams &B) {
    if (!(f >= B.lo && f <= B.hi)) return -1;
    const float d = __fsub_rn(f, B.lo);
    int i;
    if (FASTDIV) {
        float q = __fmul_rn(d, B.r);
        q = __fmaf_rn(__fmaf_rn(-B.w, q, d), B.r, q);
        q = __fmaf_rn(__fmaf_rn(-B.w, q, d), B.r, q);
        i = __float_as_int(__fadd_rz(q, 8388608.0f)) - 0x4B000000;   // trunc(q), 0 <= q < 2^23
    } else {
        i = __float2int_rz(__fdiv_rn(d, B.w));
    }
    return min(i, B.last);
}

template <bool FASTDIV>
__device__ __forceinline__ void bin_f32(uint8_t *priv, float f, const BinParams &B) {
    int i = bin_index_f32<FASTDIV>(f, B);
    if (i >= 0) bump(priv, (uint32_t)i);
}

// Four increments with their shared-memory latencies overlapped: all four counters are read
// before any is written, so equal bins must be merged by hand — element i adds 1 + (number of
// earlier elements in the same bin) and the stores go out in order, the last one carrying the
// total.  Skipped elements (bin < 0) never compare equal to a valid bin and touch no memory.
__device__ __forceinline__ void bump4(uint8_t *priv, int b0, int b1, int b2, int b3) {
    uint8_t *p0 = priv + bin_byte_offset((uint32_t)b0), *p1 = priv + bin_byte_offset((uint32_t)b1);
    uint8_t *p2 = priv + bin_byte_offset((uint32_t)b2), *p3 = priv + bin_byte_offset((uint32_t)b3);
    const bool v0 = b0 >= 0, v1 = b1 >= 0, v2 = b2 >= 0, v3 = b3 >= 0;
    uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
    if (v0) c0 = *p0;
    if (v1) c1 = *p1;
    if (v2) c2 = *p2;
    if (v3) c3 = *p3;
    c0 += 1;
    c1 += 1 + (b1 == b0);
    c2 += 1 + (b2 == b0) + (b2 == b1);
    c3 += 1 + (b3 == b0) + (b3 == b1) + (b3 == b2);
    if (v0) *p0 = (uint8_t)c0;
    if (v1) *p1 = (uint8_t)c1;
    if (v2) *p2 = (uint8_t)c2;
    if (v3) *p3 = (uint8_t)c3;
}

// Binning from a bin-edge table (EDGES kernels, DESIGN.md §3.2.1).  bin_index_f32<false> is a monotone step function of the
// fp32 value on [lo, hi], so it is fixed by its edges E[i] = the smallest fp32 f in [lo, hi] with bin(f) >= i.  The host
// computes them exactly (hist_edges in loexec.cu) and passes E[0] = lo, E[1 .. nbins-1], E[nbins] = nextup(hi) per column.
// Per element:
//     t  = sat(RN(RN(f - lo) * r * 2^-9 + 2^-10)) * 2^9,  r = RN(1/w)          (one FADD, one FFMA.SAT)
//     i0 = trunc(t)  in [0, 512]                         (FADD.RZ against 2^14: the integer part lands in the low bits)
//     counter = f >= E[i0] ? counter(i0) : counter(i0 - 1)          (one LDS.128 of the table entry, FSETP, SEL)
// For f in [lo, hi], |t - 0.5 - RN(RN(f - lo)/w)| <= (3 nbins + 4) 2^-24 < 0.5 whenever r and r 2^-9 are normal
// (2^-100 <= w <= 2^100, edges_ok), so i0 is bin(f) or bin(f) + 1 and the one comparison picks the right one.  Below lo
// (t < 1 or saturated to 0: i0 = 0, f < E[0] = lo), above hi (i0 >= nbins, f >= E[nbins] or E[i0 > nbins] = +inf) and
// NaN (saturates to 0, fails every comparison) land on a per-thread trash counter instead of a bin, so the increment
// needs no predicate.
constexpr int      kEdgeSlots     = 513;                         // table entries, i0 = 0 .. 512
constexpr uint32_t kTrashOffset   = kHistRows * kThreads * 4;    // byte offset (before 4*tid) of the trash counter: a
                                                                 // word of the fold's scratch row, bank = tid % 32
constexpr int      kEdgeSmemBytes = kHistSmemBytes + kEdgeSlots * 16;

// entry i0: {E[i0] (+inf past nbins), counter offset of bin i0, of bin i0 - 1} with out-of-range bins -> trash
__device__ __forceinline__ void load_edge_table(uint4 *tab, const float *__restrict__ E, int nbins) {
    for (int i = threadIdx.x; i < kEdgeSlots; i += blockDim.x) {
        const float e = i <= nbins ? E[i] : __int_as_float(0x7f800000);
        const uint32_t off0  = i < nbins ? bin_byte_offset((uint32_t)i) : kTrashOffset;
        const uint32_t offm1 = (i >= 1 && i <= nbins) ? bin_byte_offset((uint32_t)(i - 1)) : kTrashOffset;
        tab[i] = make_uint4(__float_as_uint(e), off0, offm1, 0u);
    }
}

struct EdgeParams {
    float    lo, rs;     // rs = RN(1/w) * 2^-9
    uint32_t tab_bits;   // shared-window address of the table minus 16 * 0x46800000 (mod 2^32): entry i0 of the
                         // FADD.RZ result with bit pattern 0x46800000 + i0 is at tab_bits + 16 * bits, one LEA
};

__device__ __forceinline__ EdgeParams edge_params(float lo, float w, const uint4 *tab) {
    // through a shuffle: ptxas cannot split the value back into window base + constant, which would cost an extra
    // VIADD per element instead of one register operand of the LEA
    const uint32_t base = __shfl_sync(0xffffffffu, (uint32_t)__cvta_generic_to_shared(tab) - 16u * 0x46800000u, 0);
    return {lo, __frcp_rn(w) * 0x1p-9f, base};
}

// byte offset (before 4*tid) of f's counter: its bin's, or the trash counter
__device__ __forceinline__ uint32_t edge_counter_offset(float f, const EdgeParams &E) {
    const float t = __saturatef(__fmaf_rn(__fsub_rn(f, E.lo), E.rs, 0x1p-10f));
    const uint32_t bits = __float_as_uint(__fadd_rz(t, 0x1p14f));                  // 2^14 + i0 * 2^-9
    uint32_t e, off0, offm1, pad;
    // the table is written before the barrier that precedes the streaming loop and is read-only afterwards
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(e), "=r"(off0), "=r"(offm1), "=r"(pad) : "r"(E.tab_bits + 16u * bits));
    asm volatile("" :: "r"(pad));      // the entry's fourth word is padding
    return f >= __uint_as_float(e) ? off0 : offm1;
}

// one increment, read-modify-write in program order: consecutive increments of one thread may hit the same counter
__device__ __forceinline__ void bump_edge(uint8_t *priv, float f, const EdgeParams &E) {
    uint8_t *p = priv + edge_counter_offset(f, E);
    *p = (uint8_t)(*p + 1);
}

// ---------------------------------------------------------------------------------------------
// CTA-wide fold of the private byte histograms -> RED.64 into counts[]
// ---------------------------------------------------------------------------------------------
// per-thread form (no barrier): each thread clears exactly the words it will count in
__device__ __forceinline__ void zero_private_own(uint32_t *smem, int rows) {
    for (int w = 0; w < rows; ++w) smem[w * kThreads + (threadIdx.x & (kThreads - 1))] = 0u;
}

// rows x kThreads words, 16 bytes per store; a thread zeroes OTHER threads' counters too, hence the barrier
__device__ __forceinline__ void zero_private(uint32_t *smem, int rows) {
    uint4 *p = reinterpret_cast<uint4 *>(smem);
    const int n = rows * (kThreads / 4);
    for (int i = threadIdx.x; i < n; i += kThreads) p[i] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
}

// Each private byte is <= 255 and a row holds kThreads = 256 words.  Warp `wp` owns rows wp, wp + 8, ..., wp + 56.
// Per row a lane reads 8 words with two LDS.128 and sums them into two packed 16-bit pairs (even bytes / odd bytes,
// <= 8 * 255 = 2040 each); the 16 packed registers of the warp's 8 rows are then reduced over the 32 lanes by a
// TRANSPOSING butterfly — at every step a lane hands half of its registers to its partner and keeps the other half
// (8 + 4 + 2 + 1 + 1 = 16 shuffles instead of 16 x 5; sums stay <= 65 280: no overflow) — and lane L ends up with
// the total of register (L >> 1) & 15.  Then one RED.64 per non-empty bin into counts[].
__device__ __forceinline__ void fold_and_flush(uint32_t *smem, int rows, int nbins,
                                               unsigned long long *counts /* this column's bins */) {
    static_assert(kThreads / 32 == 8 && kHistRows == 64, "fold assumes 8 warps x 8 rows");
    uint32_t *folded = smem + kHistRows * kThreads;   // 256 words
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    uint32_t r[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int w = warp + 8 * i;
        uint32_t even = 0u, odd = 0u;
        if (w < rows) {                                  // warp-uniform
            const uint4 a = *reinterpret_cast<const uint4 *>(smem + w * kThreads + 4 * lane);
            const uint4 b = *reinterpret_cast<const uint4 *>(smem + w * kThreads + 128 + 4 * lane);
            const uint32_t x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                even += x[q] & 0x00FF00FFu;
                odd  += __byte_perm(x[q], 0u, 0x4341u);       // bytes 1 and 3 moved down: (x >> 8) & 0x00FF00FF in one op
            }
        }
        r[2 * i] = even;
        r[2 * i + 1] = odd;
    }
    // one step per power of two; `half` is a compile-time constant in every step, so r[] stays in registers
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const int half = 8 >> s, bit = 16 >> s;
        const bool upper = (lane & bit) != 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (i < half) {
                const uint32_t send = upper ? r[i] : r[i + half];
                const uint32_t keep = upper ? r[i + half] : r[i];
                r[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
            }
        }
    }
    const uint32_t total = r[0] + __shfl_xor_sync(0xffffffffu, r[0], 1);
    if ((lane & 1) == 0) {
        const int idx = (lane >> 1) & 15;                // which of the 16 registers this lane reduced
        const int w = warp + 8 * (idx >> 1), parity = idx & 1;
        if (w < rows) {
            folded[4 * w + parity]     = total & 0xFFFFu;    // even reg: bins 4w, 4w+2 ; odd reg: bins 4w+1, 4w+3
            folded[4 * w + 2 + parity] = total >> 16;
        }
    }
    __syncthreads();
    if ((int)threadIdx.x < nbins) {
        uint32_t c = folded[threadIdx.x];
        // fire-and-forget reduction (RED, not an ATOM whose return value would have to come back before the CTA retires)
        if (c) asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(counts + threadIdx.x), "l"((unsigned long long)c) : "memory");
    }
}

// ---------------------------------------------------------------------------------------------
// multi-GPU merge, in-kernel (GroupStep).  Memory-model notes: the per-tile REDs into `local` are relaxed, gpu scope;
// bar.sync + thread 0's fence + its ticket atomic publish them to whichever CTA takes the column's last ticket
// (the threadFenceReduction pattern).  That CTA's pushes are system-scope REDs; bar.sync + fence.sys + the
// done-ticket atomic order them before the release-add on `arrived` issued by the CTA that takes the last done ticket
// (causality order is transitive over these synchronizes-with edges), and the root acquires `arrived` at system scope.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_relaxed_gpu(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_sys_add(unsigned long long *p, unsigned long long v) {
    asm volatile("red.release.sys.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// spin until *flag >= target; gives up after timeout_ns and raises *timed_out (returns false)
__device__ __forceinline__ bool wait_flag_ge(const unsigned long long *flag, unsigned long long target,
                                             unsigned long long timeout_ns, unsigned long long *timed_out) {
    if (ld_acquire_sys(flag) >= target) return true;
    const unsigned long long t0 = globaltimer_ns();
    for (;;) {
        if (ld_acquire_sys(flag) >= target) return true;
        if (globaltimer_ns() - t0 > timeout_ns) { atomicAdd(timed_out, 1ull); return false; }
        __nanosleep(64);
    }
}

// root, one thread: epilogues of overlapped launches take their turn in step order
__device__ __forceinline__ void epilogue_turn_wait(const GroupStep &G) {
    unsigned long long v;
    const unsigned long long t0 = globaltimer_ns();
    for (;;) {
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(G.epi_seq) : "memory");
        if (v >= G.step) return;
        if (globaltimer_ns() - t0 > G.timeout_ns) { atomicAdd(G.timed_out, 1ull); return; }
        __nanosleep(64);
    }
}
// root, one thread, after the epilogue: this parity may be reused by the launch after next, the next epilogue may run
__device__ __forceinline__ void epilogue_turn_done(const GroupStep &G) {
    __threadfence();
    asm volatile("red.release.gpu.global.add.u64 [%0], %1;" :: "l"(G.gen), "l"(1ull) : "memory");
    asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(G.epi_seq), "l"(G.step + 1ull) : "memory");
}

// root: all W devices have pushed -> move the merged matrix out, re-zero it, tell the peers.  One CTA (any size).
__device__ __forceinline__ void group_root_epilogue(const GroupStep &G, int n, int first, int stride, bool signal) {
    for (int i = first; i < n; i += stride) {
        // the peers' REDs were performed by this GPU's L2: read them there
        const unsigned long long c = ld_relaxed_sys(G.shared + i);
        G.result[i] = c;
        for (int p = 0; p < G.npeers; ++p)
            if (G.peer_result[p]) G.peer_result[p][i] = c;
        G.shared[i] = 0ull;
    }
    if (signal) {
        __syncthreads();
        __threadfence_system();
        if ((int)threadIdx.x < G.npeers) red_release_sys_add(G.peer_clean[threadIdx.x], 1ull);
    }
}

// Overlapped launches (GroupStep.overlap): before a CTA touches this parity's accumulate matrix or tickets, the step
// two launches back (same parity) must have finished pushing.  By the time a CTA has streamed its tile this is
// virtually always true already; the wait only matters for formal safety.  All of that step's CTAs are resident (the
// launch in between could not have started otherwise), so waiting here cannot starve them.
__device__ __forceinline__ void group_wait_generation(const GroupStep &G) {
    if (G.gen_target == 0ull) return;
    if (threadIdx.x == 0) {
        unsigned long long v;
        const unsigned long long t0 = globaltimer_ns();
        for (;;) {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(G.gen) : "memory");
            if (v >= G.gen_target) break;
            if (globaltimer_ns() - t0 > G.timeout_ns) { atomicAdd(G.timed_out, 1ull); break; }
            __nanosleep(64);
        }
    }
    __syncthreads();
}

// Called by every thread of a CTA after its tile's REDs into G.local were issued.  j: projected column, nb: its bins,
// k: columns of this launch.  Uses one word of shared memory (`sflag`, any smem word the caller no longer needs).
__device__ __forceinline__ void group_finish_column(const GroupStep &G, unsigned j, int nb, int k, unsigned tiles_per_col,
                                                    volatile uint32_t *sflag) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        *sflag = (atomicAdd(G.col_ticket + j, 1u) == tiles_per_col - 1u) ? 1u : 0u;
    }
    __syncthreads();
    if (*sflag == 0u) return;
    // last tile of column j on this device: every tile's REDs into local[j][*] are visible after this fence
    __threadfence();
    if (threadIdx.x == 0) {
        G.col_ticket[j] = 0u;
        if (G.clean) wait_flag_ge(G.clean, G.clean_target, G.timeout_ns, G.timed_out);   // root re-zeroed `shared`?
    }
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {
        unsigned long long *src = G.local + (long long)j * nb + b;
        const unsigned long long c = ld_relaxed_gpu(src);
        if (c) {
            // the owner's L2 performs the reduction
            asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" :: "l"(G.shared + (long long)j * nb + b), "l"(c) : "memory");
            *src = 0ull;                                               // local matrix is clean for the next step
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const bool last = atomicAdd(G.done_ticket, 1u) == (unsigned)k - 1u;
        if (last) {
            *G.done_ticket = 0u;
            __threadfence_system();
            red_release_sys_add(G.arrived, 1ull);
            // not the root: this parity's accumulate matrix and tickets are clean again, the launch after next may
            // flush into them.  The root says so only after its epilogue: its own next push goes into `shared` too.
            if (!G.is_root) asm volatile("red.release.gpu.global.add.u64 [%0], %1;" :: "l"(G.gen), "l"(1ull) : "memory");
        }
        *sflag = (last && G.is_root) ? 2u : 0u;
        if (*sflag == 2u) {
            epilogue_turn_wait(G);
            if (!wait_flag_ge(G.arrived, G.arrive_target, G.timeout_ns, G.timed_out)) *sflag = 3u;
        }
    }
    __syncthreads();
    if (*sflag == 2u) group_root_epilogue(G, k * nb, threadIdx.x, blockDim.x, true);
    else if (*sflag == 3u && (int)threadIdx.x < G.npeers) red_release_sys_add(G.peer_clean[threadIdx.x], 1ull);
    if (*sflag >= 2u) {
        __syncthreads();
        if (threadIdx.x == 0) epilogue_turn_done(G);
    }
}

// ---------------------------------------------------------------------------------------------
// K1+K2+K3: fused projection + cast + histogram over f64 column slabs
//   OUT: 0 = no projected output (histogram only), 1 = f32 (cast), 2 = f64 (copy)
//   HIST: accumulate per-column fixed-width histogram of the cast value
//   ALIGNED: column slabs (in and out) are 32-byte aligned -> 128-bit loads, 64/128-bit stores
//   EDGES: bin from the edge table `edges` (k x (nbins + 1) floats, edge_counter_offset); otherwise the IEEE divide
// grid.x = k * tiles_per_col ; tile index fastest along rows
// ---------------------------------------------------------------------------------------------
template <int OUT, bool HIST, bool ALIGNED, bool EDGES>
__global__ void __launch_bounds__(kThreads, LO_MIN_CTAS)
k_project_cast_hist(const char *__restrict__ in_base, long long in_pitch,
                    char *__restrict__ out_base, long long out_pitch,
                    long long nrows, unsigned tiles_per_col, unsigned long long *__restrict__ counts,
                    const float *__restrict__ edges, const __grid_constant__ ColsF64 P, const __grid_constant__ GroupStep G) {
    extern __shared__ uint32_t smem[];
    // overlapped steps: the next launch may start filling SMs as soon as every CTA of this one is resident
    if (G.overlap) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const unsigned j    = blockIdx.x / tiles_per_col;
    const unsigned tile = blockIdx.x - j * tiles_per_col;
    const long long r0  = (long long)tile * kTileRows;
    const long long n   = min((long long)kTileRows, nrows - r0);   // rows in this tile (> 0)

    const double *in = reinterpret_cast<const double *>(in_base + (long long)P.col[j] * in_pitch) + r0;
    float  *out32 = nullptr;
    double *out64 = nullptr;
    if (OUT == 1) out32 = reinterpret_cast<float *>(out_base + (long long)j * out_pitch) + r0;
    if (OUT == 2) out64 = reinterpret_cast<double *>(out_base + (long long)j * out_pitch) + r0;

    BinParams B = {0.f, 0.f, 1.f, 1.f, 0};
    int rows = 0;
    uint8_t *priv = reinterpret_cast<uint8_t *>(smem) + 4 * threadIdx.x;
    if (HIST) {
        B.lo = P.lo[j]; B.hi = P.hi[j]; B.w = P.w[j];
        B.r = __frcp_rn(B.w);
        B.last = P.nbins - 1;
        rows = (P.nbins + 3) >> 2;
    }
    EdgeParams E = {0.f, 0.f, 0u};
    if (HIST && EDGES) {
        uint4 *tab = reinterpret_cast<uint4 *>(reinterpret_cast<char *>(smem) + kHistSmemBytes);
        load_edge_table(tab, edges + (long long)j * (P.nbins + 1), P.nbins);   // zero_private's barrier publishes it
        E = edge_params(B.lo, B.w, tab);
    }

    if (ALIGNED && n == kTileRows) {
        // full tile (all but the last tile of a column): no bounds checks, register-pipelined loads.
        // (batch b, slot u) is the CTA-wide block (b*kPfBatch + u) of kThreads*kVec elements; the thread's four are
        // {2t, 2t+1} of its first half and of its second half (ldg_split4_stream)
        double v[kPfBuf][kPfBatch][4];
        const double *src = in + 2 * (long long)threadIdx.x;
#pragma unroll
        for (int pb = 0; pb < kPfBuf - 1; ++pb)
#pragma unroll
            for (int u = 0; u < kPfBatch; ++u)
                ldg_split4_stream(src + (long long)(pb * kPfBatch + u) * kThreads * kVec, kHalf, v[pb][u]);
        if (HIST) zero_private(smem, rows);        // the first batch's DRAM latency overlaps the clearing and its barrier
        // the addresses of a round of kPfBuf batches are fixed offsets from two pointers advanced once per round
        const long long t2 = 2 * (long long)threadIdx.x;
#pragma unroll 1
        for (int b0 = 0; b0 < kPfBatches; b0 += kPfBuf) {
            const double *rsrc = src + (long long)b0 * (kPfBatch * kThreads * kVec);
            float  *rout32 = (OUT == 1) ? out32 + t2 + (long long)b0 * (kPfBatch * kThreads * kVec) : nullptr;
            double *rout64 = (OUT == 2) ? out64 + t2 + (long long)b0 * (kPfBatch * kThreads * kVec) : nullptr;
#pragma unroll
            for (int s = 0; s < kPfBuf; ++s) {
                const int b  = b0 + s;                 // batch being processed, lives in buffer s
                const int nb = b + kPfBuf - 1;         // batch to fetch, into buffer (s + kPfBuf - 1) % kPfBuf
                if (nb < kPfBatches) {
#pragma unroll
                    for (int u = 0; u < kPfBatch; ++u)
                        ldg_split4_stream(rsrc + ((s + kPfBuf - 1) * kPfBatch + u) * kThreads * kVec, kHalf,
                                          v[(s + kPfBuf - 1) % kPfBuf][u]);
                }
#pragma unroll
                for (int u = 0; u < kPfBatch; ++u) {
                    const int e = (s * kPfBatch + u) * kThreads * kVec;    // from rout32 / rout64
                    float f0 = cast_f64_f32(v[s][u][0]), f1 = cast_f64_f32(v[s][u][1]);
                    float f2 = cast_f64_f32(v[s][u][2]), f3 = cast_f64_f32(v[s][u][3]);
                    if (OUT == 1) stg_split4_stream(rout32 + e, kHalf, f0, f1, f2, f3);
                    if (OUT == 2) stg_split4_stream(rout64 + e, kHalf, v[s][u]);
                    if (HIST && EDGES) {
                        bump_edge(priv, f0, E); bump_edge(priv, f1, E); bump_edge(priv, f2, E); bump_edge(priv, f3, E);
                    } else if (HIST) {
                        bump4(priv, bin_index_f32<false>(f0, B), bin_index_f32<false>(f1, B),
                              bin_index_f32<false>(f2, B), bin_index_f32<false>(f3, B));
                    }
                }
            }
        }
    } else if (ALIGNED) {
        if (HIST) zero_private(smem, rows);
#pragma unroll 1
        for (int b = 0; b < kBatches; ++b) {
            const long long e0 = (long long)b * kBatch * kThreads * kVec + 2 * threadIdx.x;   // first element of vector 0
            if (e0 >= n) break;
            double v[kBatch][4];
            if (e0 + (long long)(kBatch - 1) * kThreads * kVec + kHalf + 2 <= n) {
                // whole batch in range: all loads first (MLP), then convert/store/bin
#pragma unroll
                for (int u = 0; u < kBatch; ++u) ldg_split4_stream(in + e0 + (long long)u * kThreads * kVec, kHalf, v[u]);
#pragma unroll
                for (int u = 0; u < kBatch; ++u) {
                    const long long e = e0 + (long long)u * kThreads * kVec;
                    float f0 = cast_f64_f32(v[u][0]), f1 = cast_f64_f32(v[u][1]);
                    float f2 = cast_f64_f32(v[u][2]), f3 = cast_f64_f32(v[u][3]);
                    if (OUT == 1) stg_split4_stream(out32 + e, kHalf, f0, f1, f2, f3);
                    if (OUT == 2) stg_split4_stream(out64 + e, kHalf, v[u]);
                    if (HIST && EDGES) {
                        bump_edge(priv, f0, E); bump_edge(priv, f1, E); bump_edge(priv, f2, E); bump_edge(priv, f3, E);
                    } else if (HIST) {
                        bump4(priv, bin_index_f32<false>(f0, B), bin_index_f32<false>(f1, B),
                              bin_index_f32<false>(f2, B), bin_index_f32<false>(f3, B));
                    }
                }
            } else {
                // ragged end of the column: element-wise over the same four positions per vector
#pragma unroll 1
                for (int u = 0; u < kBatch; ++u) {
                    const long long e = e0 + (long long)u * kThreads * kVec;
#pragma unroll 1
                    for (int q = 0; q < kVec; ++q) {
                        const long long eq = e + (q & 1) + (q >> 1) * kHalf;
                        if (eq < n) {
                            double x = ldg64_stream(in + eq);
                            float  f = cast_f64_f32(x);
                            if (OUT == 1) out32[eq] = f;
                            if (OUT == 2) out64[eq] = x;
                            if (HIST && EDGES) bump_edge(priv, f, E);
                            else if (HIST) bin_f32<false>(priv, f, B);
                        }
                    }
                }
            }
        }
    } else {
        // unaligned slabs (wrapped foreign memory): scalar, lane-contiguous accesses
        if (HIST) zero_private(smem, rows);
#pragma unroll 1
        for (int i = 0; i < kElemsPerThread; ++i) {
            const long long e = (long long)i * kThreads + threadIdx.x;
            if (e >= n) break;
            double x = ldg64_stream(in + e);
            float  f = cast_f64_f32(x);
            if (OUT == 1) out32[e] = f;
            if (OUT == 2) out64[e] = x;
            if (HIST && EDGES) bump_edge(priv, f, E);
            else if (HIST) bin_f32<false>(priv, f, B);
        }
    }

    if (HIST) {
        if (G.mode == 0) {
            fold_and_flush(smem, rows, P.nbins, counts + (long long)j * P.nbins);
        } else {
            // multi-GPU merge riding on the flush: accumulate on this device, the column's last tile pushes to the root
            group_wait_generation(G);
            fold_and_flush(smem, rows, P.nbins, G.local + (long long)j * P.nbins);
            group_finish_column(G, j, P.nbins, P.k, tiles_per_col, smem);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K1+K2+K3 for histograms wider than the per-thread byte counters hold (256 < nbins <= LO_MAX_BINS): the optional
// ``bins`` key of the REST request is not capped at 256.  Same projection, cast and binning arithmetic; the counters
// are 32-bit words in shared memory, nbins x S lane slots (S = the largest power of two <= 32 with nbins * S <= 16 Ki
// words; slot = lane mod S, so S = 32 is conflict-free and smaller S spreads equal bins of one instruction over S
// words), one ATOMS per element; up to 56 Ki bins one slot per bin in 224 KiB (one CTA per SM); above that the increments go
// straight to the count matrix in L2 (RED.64: with that many bins two lanes rarely meet).  A CTA streams a chunk of one projected column, four 32-byte vectors in flight per thread, and folds once (32-bit
// counters: chunk_rows < 2^31).  HBM-bound like the 256-bin kernel: 12 B and one shared-memory atomic per element.
// grid.x = k * chunks_per_col
// ---------------------------------------------------------------------------------------------
constexpr int kWBThreads   = 512;
constexpr int kWBSmemWords = 16384;                                  // 64 KiB: two CTAs per SM
constexpr int kWBSmemWordsMax = 57344;                               // 224 KiB: one CTA per SM, one slot per bin
constexpr int kWBVecs      = 4;                                      // 32-byte vectors in flight per thread
constexpr int kWBRoundRows = kWBThreads * kVec * kWBVecs;            // rows per loop round

template <int OUT, bool FASTDIV>
__global__ void __launch_bounds__(kWBThreads, 2)
k_project_cast_hist_bins(const char *__restrict__ in_base, long long in_pitch, char *__restrict__ out_base, long long out_pitch,
                         long long nrows, unsigned chunks_per_col, long long chunk_rows, int slots_log2 /* < 0: no smem */,
                         int aligned, unsigned long long *__restrict__ counts,
                         const __grid_constant__ ColsF64 P, const __grid_constant__ GroupStep G) {
    extern __shared__ uint32_t smem[];
    if (G.overlap) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const unsigned j     = blockIdx.x / chunks_per_col;
    const unsigned chunk = blockIdx.x - j * chunks_per_col;
    const long long r0   = (long long)chunk * chunk_rows;
    const long long n    = min(chunk_rows, nrows - r0);
    const double *in = reinterpret_cast<const double *>(in_base + (long long)P.col[j] * in_pitch) + r0;
    float  *out32 = (OUT == 1) ? reinterpret_cast<float *>(out_base + (long long)j * out_pitch) + r0 : nullptr;
    double *out64 = (OUT == 2) ? reinterpret_cast<double *>(out_base + (long long)j * out_pitch) + r0 : nullptr;
    const int nb = P.nbins;
    BinParams B = {P.lo[j], P.hi[j], P.w[j], __frcp_rn(P.w[j]), nb - 1};
    unsigned long long *dst = (G.mode == 0 ? counts : G.local) + (long long)j * nb;
    const bool in_smem = slots_log2 >= 0;
    const int  sl = in_smem ? slots_log2 : 0;
    const uint32_t slot = threadIdx.x & ((1u << sl) - 1u);
    if (in_smem) {
        for (int i = threadIdx.x; i < (nb << sl); i += kWBThreads) smem[i] = 0u;
        __syncthreads();
    } else if (G.mode != 0) {
        group_wait_generation(G);                       // the increments land in G.local as they are issued
    }
    auto count = [&](float f) {
        const int i = bin_index_f32<FASTDIV>(f, B);
        if (i >= 0) {
            if (in_smem) atomicAdd(smem + ((uint32_t)i << sl) + slot, 1u);
            else asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(dst + i), "l"(1ull) : "memory");
        }
    };
    long long done = 0;
    if (aligned) {
        constexpr long long kWBHalf = kWBThreads * kVec / 2;
        const double *src = in + 2 * (long long)threadIdx.x;
#pragma unroll 1
        for (; done + kWBRoundRows <= n; done += kWBRoundRows) {
            double v[kWBVecs][4];
#pragma unroll
            for (int u = 0; u < kWBVecs; ++u) ldg_split4_stream(src + done + (long long)u * kWBThreads * kVec, kWBHalf, v[u]);
#pragma unroll
            for (int u = 0; u < kWBVecs; ++u) {
                const long long e = done + (long long)u * kWBThreads * kVec + 2 * threadIdx.x;
                const float f0 = cast_f64_f32(v[u][0]), f1 = cast_f64_f32(v[u][1]), f2 = cast_f64_f32(v[u][2]), f3 = cast_f64_f32(v[u][3]);
                if (OUT == 1) stg_split4_stream(out32 + e, kWBHalf, f0, f1, f2, f3);
                if (OUT == 2) stg_split4_stream(out64 + e, kWBHalf, v[u]);
                count(f0); count(f1); count(f2); count(f3);
            }
        }
    }
    // the rest of the chunk (all of it for unaligned slabs): element-wise, lane-contiguous
#pragma unroll 1
    for (long long e = done + threadIdx.x; e < n; e += kWBThreads) {
        const double x = ldg64_stream(in + e);
        const float  f = cast_f64_f32(x);
        if (OUT == 1) out32[e] = f;
        if (OUT == 2) out64[e] = x;
        count(f);
    }
    if (in_smem) {
        __syncthreads();
        if (G.mode != 0) group_wait_generation(G);
        const uint32_t S = 1u << sl;
        for (int b = threadIdx.x; b < nb; b += kWBThreads) {
            unsigned long long c = 0;
            for (uint32_t i = 0; i < S; ++i) c += smem[((uint32_t)b << sl) + ((i + threadIdx.x) & (S - 1u))];   // rotated: no bank conflicts
            if (c) asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(dst + b), "l"(c) : "memory");
        }
    }
    if (G.mode != 0) group_finish_column(G, j, nb, P.k, chunks_per_col, smem);
}

// ---------------------------------------------------------------------------------------------
// K1+K2+K3, TMA form (LOEXEC_TMA=1): the same tile, but the column slab is staged into shared memory by the
// bulk-copy engine (cp.async.bulk global -> shared, completion on an mbarrier) through a kTmaStages-deep ring
// driven by one producer thread; the 256 consumer threads read their 32 bytes from the ring instead of
// issuing the 128-bit loads themselves.  Built to answer "would TMA staging beat the register pipeline?" with a
// measurement (DESIGN.md §3.8); arithmetic, tile shape, private histograms and results are identical.
// Full, 32-byte-aligned tiles only — the host routes everything else to k_project_cast_hist.
// ---------------------------------------------------------------------------------------------
constexpr int kTmaStages     = 5;
constexpr int kTmaStageBytes = kThreads * kVec * 8;                    // 8 KiB = one 32-byte vector per consumer
constexpr int kTmaRounds     = kVecPerThread;                          // 60 rounds per tile
constexpr int kTmaSmemBytes  = kHistSmemBytes + kTmaStages * kTmaStageBytes + 2 * kTmaStages * 8;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "LO_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra LO_DONE_%=;\n\t"
        "bra LO_WAIT_%=;\n\t"
        "LO_DONE_%=:\n\t}"
        :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar) : "memory");
}

template <int OUT, bool HIST, bool FASTDIV>
__global__ void __launch_bounds__(kThreads + 32, 2)
k_project_cast_hist_tma(const char *__restrict__ in_base, long long in_pitch,
                        char *__restrict__ out_base, long long out_pitch,
                        long long nrows, unsigned tiles_per_col,
                        unsigned long long *__restrict__ counts,
                        const __grid_constant__ ColsF64 P) {
    extern __shared__ uint32_t smem[];
    uint8_t *ring = reinterpret_cast<uint8_t *>(smem) + kHistSmemBytes;                 // kTmaStages x 8 KiB
    const uint32_t bar_full  = smem_u32(ring + kTmaStages * kTmaStageBytes);            // kTmaStages x 8 B
    const uint32_t bar_empty = bar_full + kTmaStages * 8;
    const unsigned j    = blockIdx.x / tiles_per_col;
    const unsigned tile = blockIdx.x - j * tiles_per_col;
    const long long r0  = (long long)tile * kTileRows;            // host guarantees a full tile
    const double *in = reinterpret_cast<const double *>(in_base + (long long)P.col[j] * in_pitch) + r0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kTmaStages; ++s) {
            mbar_init(bar_full + 8 * s, 1);                    // the producer's expect_tx arrival
            mbar_init(bar_empty + 8 * s, kThreads / 32);       // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const bool producer = threadIdx.x >= kThreads;
    BinParams B = {0.f, 0.f, 1.f, 1.f, 0};
    int rows = 0;
    uint8_t *priv = reinterpret_cast<uint8_t *>(smem) + 4 * (threadIdx.x & (kThreads - 1));
    if (HIST && !producer) {
        B.lo = P.lo[j]; B.hi = P.hi[j]; B.w = P.w[j];
        B.r = __frcp_rn(B.w);
        B.last = P.nbins - 1;
        rows = (P.nbins + 3) >> 2;
        zero_private_own(smem, rows);
    }
    __syncthreads();

    if (producer) {
        if (threadIdx.x == kThreads) {                          // one elected thread drives the copy engine
#pragma unroll 1
            for (int r = 0; r < kTmaRounds; ++r) {
                const int s = r % kTmaStages;
                const uint32_t phase = (uint32_t)(r / kTmaStages) & 1u;
                mbar_wait(bar_empty + 8 * s, phase ^ 1u);       // slot free (passes at once on the first lap)
                mbar_expect_tx(bar_full + 8 * s, kTmaStageBytes);
                tma_load_1d(smem_u32(ring + s * kTmaStageBytes), in + (long long)r * (kThreads * kVec), kTmaStageBytes,
                            bar_full + 8 * s);
            }
        }
    } else {
        float  *out32 = (OUT == 1) ? reinterpret_cast<float *>(out_base + (long long)j * out_pitch) + r0 : nullptr;
        double *out64 = (OUT == 2) ? reinterpret_cast<double *>(out_base + (long long)j * out_pitch) + r0 : nullptr;
        const int lane = threadIdx.x & 31;
#ifndef LO_TMA_UNROLL
#define LO_TMA_UNROLL 1
#endif
        static_assert(kTmaRounds % LO_TMA_UNROLL == 0, "rounds per tile must be a multiple of the unroll");
#pragma unroll 1
        for (int r0u = 0; r0u < kTmaRounds; r0u += LO_TMA_UNROLL) {
            double2 a[LO_TMA_UNROLL], b[LO_TMA_UNROLL];
            // take LO_TMA_UNROLL stages at once: all their shared-memory reads are in flight together, the slots go
            // back to the copy engine before any arithmetic starts
#pragma unroll
            for (int u = 0; u < LO_TMA_UNROLL; ++u) {
                const int r = r0u + u, s = r % kTmaStages;
                mbar_wait(bar_full + 8 * s, (uint32_t)(r / kTmaStages) & 1u);
                // 16-byte accesses at 16-byte lane stride are bank-conflict free: a thread takes doubles
                // {2t, 2t+1} from the first half of the stage and {512+2t, 513+2t} from the second half
                a[u] = *reinterpret_cast<const double2 *>(ring + s * kTmaStageBytes + threadIdx.x * 16);
                b[u] = *reinterpret_cast<const double2 *>(ring + s * kTmaStageBytes + kTmaStageBytes / 2 + threadIdx.x * 16);
            }
            __syncwarp();
            if (lane == 0) {
#pragma unroll
                for (int u = 0; u < LO_TMA_UNROLL; ++u) mbar_arrive(bar_empty + 8 * ((r0u + u) % kTmaStages));
            }
#pragma unroll
            for (int u = 0; u < LO_TMA_UNROLL; ++u) {
                const long long e = (long long)(r0u + u) * (kThreads * kVec) + 2 * threadIdx.x;
                const float f0 = cast_f64_f32(a[u].x), f1 = cast_f64_f32(a[u].y), f2 = cast_f64_f32(b[u].x), f3 = cast_f64_f32(b[u].y);
                if (OUT == 1) {
                    asm volatile("st.global.cs.v2.f32 [%0], {%1,%2};" :: "l"(out32 + e), "f"(f0), "f"(f1) : "memory");
                    asm volatile("st.global.cs.v2.f32 [%0], {%1,%2};" :: "l"(out32 + e + 512), "f"(f2), "f"(f3) : "memory");
                }
                if (OUT == 2) {
                    asm volatile("st.global.cs.v2.f64 [%0], {%1,%2};" :: "l"(out64 + e), "d"(a[u].x), "d"(a[u].y) : "memory");
                    asm volatile("st.global.cs.v2.f64 [%0], {%1,%2};" :: "l"(out64 + e + 512), "d"(b[u].x), "d"(b[u].y) : "memory");
                }
                if (HIST)
                    bump4(priv, bin_index_f32<FASTDIV>(f0, B), bin_index_f32<FASTDIV>(f1, B),
                          bin_index_f32<FASTDIV>(f2, B), bin_index_f32<FASTDIV>(f3, B));
            }
        }
    }
    if (HIST) {
        // fold_and_flush is written for exactly kThreads threads; the producer warp only joins its barriers
        uint32_t *folded = smem + kHistRows * kThreads;
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        __syncthreads();
        if (!producer) {
            for (int w = warp; w < rows; w += kThreads / 32) {
                const uint32_t *row = smem + w * kThreads;
                uint32_t even = 0, odd = 0;
#pragma unroll
                for (int i = 0; i < kThreads / 32; ++i) {
                    uint32_t x = row[lane + 32 * i];
                    even += x & 0x00FF00FFu;
                    odd  += (x >> 8) & 0x00FF00FFu;
                }
#pragma unroll
                for (int sft = 16; sft > 0; sft >>= 1) {
                    even += __shfl_xor_sync(0xffffffffu, even, sft);
                    odd  += __shfl_xor_sync(0xffffffffu, odd, sft);
                }
                if (lane == 0) {
                    folded[4 * w + 0] = even & 0xFFFFu;
                    folded[4 * w + 1] = odd & 0xFFFFu;
                    folded[4 * w + 2] = even >> 16;
                    folded[4 * w + 3] = odd >> 16;
                }
            }
        }
        __syncthreads();
        if ((int)threadIdx.x < P.nbins) {
            const uint32_t c = folded[threadIdx.x];
            unsigned long long *dst = counts + (long long)j * P.nbins + threadIdx.x;
            if (c) atomicAdd(dst, (unsigned long long)c);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K4: per-column 256-bin value counts of byte columns; 32-bit counters in lane slots shared by all warps of the CTA.
// Per-thread byte counters (the f64 kernel's layout) are not bounded by the atomic unit here (conflict-free ATOMS with
// their operands ready retire fast enough) but by the arithmetic that turns a byte into (counter word, byte field):
// mask, PRMT, shift extraction, 1 << n.  This layout needs none of it.  The CTA keeps ONE histogram of 256 bins x 64
// slots of 32-bit counters (64 KiB): slot = lane + 32 * (warp & 1), counter of (bin b, slot s) at byte b * 256 + 4 * s.
//   * bank = (b * 64 + s) mod 32 = lane: every warp instruction is conflict-free, whatever the data;
//   * the address of a byte's counter is [4s | b | 0 | 0] byte by byte: ONE PRMT straight from the input word — no mask,
//     no field shift; the increment is the constant 1;
//   * warps of equal parity share counters through the atomics (different warps never collide inside one instruction);
//   * 32-bit counters do not wrap, so a CTA streams a long chunk of its column (up to 256 Ki rows) and folds once:
//     thread t sums the 64 slots of bin t (rotated start: conflict-free) and issues one RED.64.
// Per byte: one PRMT + one ATOMS.ADD (+ 1/4 of a LOP3 for the run test).
// ---------------------------------------------------------------------------------------------

// shared-window address at which a block's dynamic shared memory starts when the kernel has no static shared memory:
// the 1 KiB sm_90 reserves per block (lo_init checks the size).  The atomics carry it in their immediate offset; the
// kernel traps if it is wrong.  No return value: the shared-memory atomic is fire-and-forget.
#define LO_SMEM_WINDOW_BASE 1024
__device__ __forceinline__ void atoms_add_base(uint32_t offset, uint32_t v) {
    asm volatile("red.shared.add.u32 [%0+1024], %1;" :: "r"(offset), "r"(v) : "memory");
}
static_assert(LO_SMEM_WINDOW_BASE == 1024, "keep the immediate in atoms_add_base in sync");

constexpr int kU8LThreads   = 512;
constexpr int kU8LSmemBytes = 256 * 64 * 4;                       // 64 KiB
constexpr int kU8LRoundRows = kU8LThreads * 4 * kU8VecBytes;      // 32 768 rows per loop iteration (4 vectors per thread)

// ALIGNED = false: the slab's base or pitch is not a multiple of 16 bytes (a wrapped foreign table), so there are no
// 128-bit loads: every byte of the chunk is one 8-bit load and one atomic.
template <bool ALIGNED>
__global__ void __launch_bounds__(kU8LThreads, 3)
k_hist_u8_cols_lanes(const uint8_t *__restrict__ in_base, long long in_pitch, long long nrows,
                     unsigned chunks_per_col, long long chunk_rows, unsigned long long *__restrict__ counts,
                     const __grid_constant__ ColsU8 P, const __grid_constant__ GroupStep G) {
    extern __shared__ uint32_t smem[];
    if (G.overlap) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const unsigned j     = blockIdx.x / chunks_per_col;
    const unsigned chunk = blockIdx.x - j * chunks_per_col;
    const long long r0   = (long long)chunk * chunk_rows;
    const long long n    = min(chunk_rows, nrows - r0);
    const uint8_t *in    = in_base + (long long)P.col[j] * in_pitch + r0;
    if ((uint32_t)__cvta_generic_to_shared(smem) != LO_SMEM_WINDOW_BASE) __trap();     // immediate offset of the atomics
    const uint32_t slot4 = 4u * ((threadIdx.x & 31u) + 32u * ((threadIdx.x >> 5) & 1u));
    const uint8_t *src = in + (long long)threadIdx.x * kU8VecBytes;
    constexpr long long kStride = (long long)kU8LThreads * kU8VecBytes;        // bytes between a thread's vectors

    const long long rounds = ALIGNED ? n / kU8LRoundRows : 0;
    uint4 a[4], b[4];                                   // loads land in a[] while a copy in b[] is counted
    auto load_round = [&](uint4 (&d)[4], long long r) {
#pragma unroll
        for (int u = 0; u < 4; ++u) d[u] = ldg128_stream(src + r * kU8LRoundRows + u * kStride);
    };
    if (rounds > 0) load_round(a, 0);
    {   // clear the counters (overlaps the first loads' DRAM latency)
        uint4 *p = reinterpret_cast<uint4 *>(smem);
        for (int i = threadIdx.x; i < kU8LSmemBytes / 16; i += kU8LThreads) p[i] = make_uint4(0u, 0u, 0u, 0u);
        __syncthreads();
    }
    auto count_vec = [&](const uint4 &x) {
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            atoms_add_base(__byte_perm(w[q], slot4, 0x6504u), 1u);
            atoms_add_base(__byte_perm(w[q], slot4, 0x6514u), 1u);
            atoms_add_base(__byte_perm(w[q], slot4, 0x6524u), 1u);
            atoms_add_base(__byte_perm(w[q], slot4, 0x6534u), 1u);
        }
    };
    auto count_round = [&](const uint4 (&c)[4]) {
        // a warp whose 2 KiB are one value (constant columns: borders, flags, padding) issues one atomic per lane;
        // two compares reject mixed data before the full test is paid
        const uint32_t splat = __byte_perm(c[0].x, 0, 0x0000);
        if (__all_sync(0xffffffffu, (c[0].x == splat) & (c[3].w == splat))) {
            uint32_t diff = 0u;
#pragma unroll
            for (int u = 0; u < 4; ++u) diff |= (c[u].x ^ splat) | (c[u].y ^ splat) | (c[u].z ^ splat) | (c[u].w ^ splat);
            if (__all_sync(0xffffffffu, diff == 0u)) {
                atoms_add_base(((splat & 0xFFu) << 8) | slot4, 64u);
                return;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) count_vec(c[u]);
    };
#pragma unroll 1
    for (long long r = 0; r < rounds; ++r) {
#pragma unroll
        for (int u = 0; u < 4; ++u) b[u] = a[u];
        if (r + 1 < rounds) load_round(a, r + 1);
        count_round(b);
    }
    if (ALIGNED) {   // rest of the chunk (< one round): every whole vector requested before the first is counted, then single bytes
        const long long base = rounds * kU8LRoundRows;
        bool have[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            have[u] = base + (long long)threadIdx.x * kU8VecBytes + u * kStride + kU8VecBytes <= n;
            if (have[u]) a[u] = ldg128_stream(src + base + u * kStride);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (have[u]) count_vec(a[u]);
        const long long q = base + ((n - base) / kU8VecBytes) * kU8VecBytes + threadIdx.x;
        if (q < n) atoms_add_base((ldg8_stream(in + q) << 8) | slot4, 1u);
    } else {
#pragma unroll 1
        for (long long e = threadIdx.x; e < n; e += kU8LThreads) atoms_add_base((ldg8_stream(in + e) << 8) | slot4, 1u);
    }
    __syncthreads();
    if (G.mode != 0) group_wait_generation(G);
    if (threadIdx.x < 256) {
        const uint32_t *row = smem + threadIdx.x * 64;
        unsigned long long c = 0;
#pragma unroll 8
        for (int i = 0; i < 64; ++i) c += row[(threadIdx.x + i) & 63];      // rotated start: lanes hit distinct banks
        unsigned long long *dst = (G.mode == 0 ? counts : G.local) + (long long)j * 256 + threadIdx.x;
        if (c) asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(dst), "l"(c) : "memory");
    }
    if (G.mode != 0) group_finish_column(G, j, 256, P.k, chunks_per_col, smem);
}

// ---------------------------------------------------------------------------------------------
// synthetic tables (bench / parity inputs) — CPU twins: oracle/bsem.c, oracle/synth.py
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

constexpr int kSpecialPeriod = 1009;
constexpr int kNumSpecials   = 20;

__device__ __forceinline__ double special_value(int idx, double lo, double hi) {
    switch (idx) {
        case 0:  return 0.0;
        case 1:  return -0.0;
        case 2:  return 1e-40;                                  // fp32 subnormal
        case 3:  return 1e-46;                                  // underflows to +0
        case 4:  return -1e-46;                                 // underflows to -0
        case 5:  return 1e39;                                   // overflows to +inf
        case 6:  return -1e39;
        case 7:  return __longlong_as_double(0x7ff8000000000000ll);   // quiet NaN
        case 8:  return __longlong_as_double(0xfff4000000000001ll);   // negative signalling NaN with payload
        case 9:  return 1.0 + 5.9604644775390625e-08;           // 1 + 2^-24 : RNE tie -> 1.0
        case 10: return 1.0 + 1.7881393432617188e-07;           // 1 + 3*2^-24 : tie -> 1 + 2^-22
        case 11: return 16777217.0;                             // 2^24 + 1 : tie -> 2^24
        case 12: return 3.4028235677973366e38;                  // tie at FLT_MAX boundary -> +inf
        case 13: return hi;
        case 14: return lo;
        case 15: return __longlong_as_double(__double_as_longlong(hi) + (hi > 0 ? 1 : -1));   // next above hi (hi != 0)
        case 16: return __dadd_rn(hi, __dmul_rn(hi - lo, 9.5367431640625e-07));    // clearly above hi (no FMA)
        case 17: return __dsub_rn(lo, __dmul_rn(hi - lo, 9.5367431640625e-07));    // clearly below lo (no FMA)
        case 18: return __longlong_as_double(0x7ff0000000000000ll);   // +inf
        default: return __longlong_as_double(0xfff0000000000000ll);   // -inf
    }
}

__global__ void k_fill_f64(double *base, long long pitch_elems, long long nrows, int ncols,
                           int kind, uint64_t seed, long long row_offset, double lo, double hi) {
    const long long total = nrows * (long long)ncols;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int       c = (int)(i / nrows);
        const long long r = i - (long long)c * nrows;
        const uint64_t  g = (uint64_t)(row_offset + r);
        const uint64_t  u = splitmix64(seed ^ ((uint64_t)c << 40) ^ g);
        // separate RN multiply and add (no FMA) so numpy / C reproduce it bit for bit
        double x = __dadd_rn(lo, __dmul_rn(hi - lo, __dmul_rn((double)(u >> 11), 1.1102230246251565e-16)));
        if (kind >= 1 && (g % kSpecialPeriod) == (uint64_t)(c % kSpecialPeriod))
            x = special_value((int)((g / kSpecialPeriod + (uint64_t)c) % kNumSpecials), lo, hi);
        if (kind == 2 && c == 0) x = __dadd_rn(lo, __dmul_rn(hi - lo, 0.75));
        base[(long long)c * pitch_elems + r] = x;
    }
}

__global__ void k_fill_u8_mnist(uint8_t *base, long long pitch, long long nrows, int ncols,
                                uint64_t seed, long long row_offset) {
    const long long total = nrows * (long long)ncols;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int       c = (int)(i / nrows);
        const long long r = i - (long long)c * nrows;
        const uint64_t  u = splitmix64(seed ^ ((uint64_t)c << 40) ^ (uint64_t)(row_offset + r));
        const int py = (c % 784) / 28, px = (c % 784) % 28;
        uint8_t v = 0;
        if (py >= 4 && py < 24 && px >= 4 && px < 24 && (u & 0xFFu) >= 0x99u) v = (uint8_t)((u >> 8) & 0xFFu);
        base[(long long)c * pitch + r] = v;
    }
}

// ---------------------------------------------------------------------------------------------
// multi-GPU merge: the launches that are NOT the streaming kernel
// ---------------------------------------------------------------------------------------------
// Merge of a LARGE count matrix (config M: 784 x 256 counts = 1.5 MiB) as its own launch after a plain streaming
// kernel that accumulated into G.local: moving that much through one CTA (or paying a ticket + fence per streaming
// CTA — 13 k CTAs of ~10 us each for config M) costs more than a second launch.  grid <= SM count, so every CTA is
// resident and CTAs may wait on each other through global memory.  Phase 1: each CTA pushes its slice of the local
// matrix into the root's (system-scope RED.64) and re-zeroes it; the last one arrives.  Phase 2 (root): every CTA
// waits for the W arrivals itself, moves its slice of the merged matrix out and re-zeroes it; the last one tells
// the peers.
__global__ void __launch_bounds__(256)
k_group_merge_big(const __grid_constant__ GroupStep G, int n) {
    __shared__ int ok, last;
    const int first = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    if (threadIdx.x == 0 && G.clean) wait_flag_ge(G.clean, G.clean_target, G.timeout_ns, G.timed_out);
    __syncthreads();
    for (int i = first; i < n; i += stride) {
        const unsigned long long c = ld_relaxed_gpu(G.local + i);
        if (c) {
            asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" :: "l"(G.shared + i), "l"(c) : "memory");
            G.local[i] = 0ull;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        if (atomicAdd(G.done_ticket, 1u) == gridDim.x - 1u) {
            *G.done_ticket = 0u;
            __threadfence_system();
            red_release_sys_add(G.arrived, 1ull);
            if (!G.is_root) asm volatile("red.release.gpu.global.add.u64 [%0], %1;" :: "l"(G.gen), "l"(1ull) : "memory");
        }
        ok = G.is_root ? (wait_flag_ge(G.arrived, G.arrive_target, G.timeout_ns, G.timed_out) ? 1 : 0) : -1;
    }
    __syncthreads();
    if (ok < 0) return;                                   // not the root: done
    if (ok) group_root_epilogue(G, n, first, stride, false);
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        last = atomicAdd(G.col_ticket, 1u) == gridDim.x - 1u;
        if (last) { *G.col_ticket = 0u; __threadfence_system(); epilogue_turn_done(G); }
    }
    __syncthreads();
    if (last && (int)threadIdx.x < G.npeers) red_release_sys_add(G.peer_clean[threadIdx.x], 1ull);
}

// merge of a small per-device vector that some other kernel(s) already accumulated into G.local (the *_host
// pipelines, the min/max pre-pass): one CTA pushes it to the root, arrives, and on the root runs the epilogue.
//   op 0: every element is a sum.   op 1: min/max pre-pass layout, elements 3j, 3j+1 are maxima, 3j+2 a sum.
__global__ void __launch_bounds__(256)
k_group_push(const __grid_constant__ GroupStep G, int n, int op) {
    __shared__ int state;
    if (threadIdx.x == 0 && G.clean) wait_flag_ge(G.clean, G.clean_target, G.timeout_ns, G.timed_out);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long c = ld_relaxed_gpu(G.local + i);
        if (c) {
            if (op == 1 && (i % 3) != 2) atomicMax_system(G.shared + i, c);
            else                         atomicAdd_system(G.shared + i, c);
            G.local[i] = 0ull;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        red_release_sys_add(G.arrived, 1ull);
        if (!G.is_root) asm volatile("red.release.gpu.global.add.u64 [%0], %1;" :: "l"(G.gen), "l"(1ull) : "memory");
        state = G.is_root ? (wait_flag_ge(G.arrived, G.arrive_target, G.timeout_ns, G.timed_out) ? 2 : 3) : 0;
    }
    __syncthreads();
    if (state == 2) group_root_epilogue(G, n, threadIdx.x, blockDim.x, true);
    else if (state == 3 && (int)threadIdx.x < G.npeers) red_release_sys_add(G.peer_clean[threadIdx.x], 1ull);
    if (state >= 2) {
        __syncthreads();
        if (threadIdx.x == 0) epilogue_turn_done(G);
    }
}

// device-side barrier across the group: everybody release-adds the root's counter and spins on it (remote polling
// over NVLink for the non-root devices).  Used to start a timed region on all GPUs within a few microseconds.
__global__ void k_group_barrier(unsigned long long *root_counter, unsigned long long target, unsigned long long timeout_ns,
                                unsigned long long *timed_out) {
    __threadfence_system();
    red_release_sys_add(root_counter, 1ull);
    wait_flag_ge(root_counter, target, timeout_ns, timed_out);
}

// LO_MERGE_NCCL min/max pre-pass: result[0, n) holds the max-reduction, result[n, 2n) the sum-reduction of the same
// vector; element 3j+2 (the finite count) is meaningful in the sum, the others in the max
__global__ void k_minmax_compose(unsigned long long *result, int n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (i % 3 == 2) result[i] = result[n + i];
}

// a non-root device waits for the root's broadcast of step `target` (its clean counter doubles as "result ready")
__global__ void k_flag_wait(const unsigned long long *flag, unsigned long long target, unsigned long long timeout_ns,
                            unsigned long long *timed_out) {
    wait_flag_ge(flag, target, timeout_ns, timed_out);
}

// exact value counts of dictionary codes (R-semantics $group on arbitrary columns): RED.64 per element;
// counts[ncodes] collects out-of-range codes so the host can reject them
__global__ void k_count_codes_u32(const uint32_t *__restrict__ codes, long long n, uint32_t ncodes,
                                  unsigned long long *__restrict__ counts) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const uint32_t c = codes[i];
        atomicAdd(counts + (c < ncodes ? c : ncodes), 1ull);
    }
}

// per-column min / max / count of the finite cast values.  out[3*j+0] = max over ~ordered(x) (i.e. the
// min, stored complemented so that zero-filled memory is the identity), out[3*j+1] = max over ordered(x),
// out[3*j+2] = count;  ordered(bits) maps fp32 to uint32 monotonically.
__device__ __forceinline__ uint32_t ordered_u32(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void k_minmax_cast(const char *__restrict__ base, long long pitch, long long n,
                              unsigned long long *__restrict__ out) {
    const double *col = reinterpret_cast<const double *>(base + (long long)blockIdx.y * pitch);
    uint32_t mn = 0, mx = 0;
    unsigned long long cnt = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float f = cast_f64_f32(col[i]);
        if (f == f && fabsf(f) != __int_as_float(0x7f800000)) {
            const uint32_t o = ordered_u32(f);
            mn = max(mn, ~o);
            mx = max(mx, o);
            ++cnt;
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        mn = max(mn, __shfl_xor_sync(0xffffffffu, mn, s));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, s));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, s);
    }
    if ((threadIdx.x & 31) == 0 && cnt) {
        atomicMax(out + 3 * blockIdx.y + 0, (unsigned long long)mn);
        atomicMax(out + 3 * blockIdx.y + 1, (unsigned long long)mx);
        atomicAdd(out + 3 * blockIdx.y + 2, cnt);
    }
}

// ---------------------------------------------------------------------------------------------
// exact value counts of a numeric column without a host dictionary: GPU hash group-by
// ($group / $sum:1 of histogram_image/histogram.py:31-36 on number fields).  Keys are binary64 bit patterns
// canonicalised to MongoDB's grouping equality for numbers (-0.0 == 0.0, NaN == NaN); open addressing with
// linear probing in HBM, 64-bit CAS to claim a slot, RED.64 to count; equal keys inside a warp are merged
// first (match.any) so a two-valued column does not serialise on two L2 addresses.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;      // a NaN payload no canonical key can have

__device__ __forceinline__ unsigned long long canonical_key(double x) {
    if (x != x) return 0x7FF8000000000000ull;
    if (x == 0.0) return 0ull;
    return (unsigned long long)__double_as_longlong(x);
}

__global__ void k_hash_count_f64(const double *__restrict__ values, long long n, unsigned long long *__restrict__ keys,
                                 unsigned long long *__restrict__ counts, unsigned long long mask) {
    for (long long i0 = blockIdx.x * (long long)blockDim.x; i0 < n; i0 += (long long)gridDim.x * blockDim.x) {
        const long long i = i0 + threadIdx.x;
        const bool live = i < n;
        const unsigned active = __ballot_sync(0xffffffffu, live);
        if (!live) continue;
        const unsigned long long key = canonical_key(values[i]);
        const unsigned peers = __match_any_sync(active, key);
        if ((int)(threadIdx.x & 31) != __ffs(peers) - 1) continue;      // one lane per distinct key in the warp
        const unsigned long long add = (unsigned long long)__popc(peers);
        unsigned long long h = splitmix64(key) & mask;
        for (;;) {
            const unsigned long long old = atomicCAS(keys + h, kEmptyKey, key);
            if (old == kEmptyKey || old == key) { atomicAdd(counts + h, add); break; }
            h = (h + 1) & mask;
        }
    }
}

__global__ void k_hash_compact(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ counts,
                               unsigned long long slots, unsigned long long *__restrict__ out_keys,
                               unsigned long long *__restrict__ out_counts, unsigned long long capacity,
                               unsigned long long *__restrict__ n_out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < slots;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = keys[i];
        if (k != kEmptyKey) {
            const unsigned long long pos = atomicAdd(n_out, 1ull);
            if (pos < capacity) { out_keys[pos] = k; out_counts[pos] = counts[i]; }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// exact value counts of a TEXT column (cells packed as chars + offsets): GPU hash group-by on the bytes.
// A slot holds (33 bits of the cell's hash | 31-bit row index of the group's representative); a probing
// thread whose hash bits match compares its bytes with the representative's (the input is immutable), so the
// result is exact whatever the hash does.  Lanes of a warp with the same 64-bit hash are merged first
// (match.any), after verifying byte equality with the group leader.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ unsigned long long hash_bytes(const uint8_t *p, long long len) {
    unsigned long long h = 0xCBF29CE484222325ull ^ (unsigned long long)len;
    for (long long i = 0; i < len; ++i) h = (h ^ p[i]) * 0x100000001B3ull;     // FNV-1a
    return splitmix64(h);
}

__device__ __forceinline__ bool same_cell(const uint8_t *chars, const long long *offsets, long long a, long long b) {
    const long long a0 = offsets[a], b0 = offsets[b], la = offsets[a + 1] - a0;
    if (la != offsets[b + 1] - b0) return false;
    for (long long i = 0; i < la; ++i)
        if (chars[a0 + i] != chars[b0 + i]) return false;
    return true;
}

__global__ void k_hash_count_str(const uint8_t *__restrict__ chars, const long long *__restrict__ offsets, long long n,
                                 unsigned long long *__restrict__ slots, unsigned long long *__restrict__ counts,
                                 unsigned long long mask) {
    for (long long i0 = blockIdx.x * (long long)blockDim.x; i0 < n; i0 += (long long)gridDim.x * blockDim.x) {
        const long long i = i0 + threadIdx.x;
        const bool live = i < n;
        const unsigned active = __ballot_sync(0xffffffffu, live);
        if (!live) continue;
        const unsigned long long h = hash_bytes(chars + offsets[i], offsets[i + 1] - offsets[i]);
        const unsigned peers = __match_any_sync(active, h);
        const int leader = __ffs(peers) - 1;
        const long long leader_row = __shfl_sync(active, i, leader);
        const bool same = ((int)(threadIdx.x & 31) == leader) || same_cell(chars, offsets, i, leader_row);
        const unsigned eq = __ballot_sync(active, same);
        unsigned long long add;
        if ((int)(threadIdx.x & 31) == leader) add = (unsigned long long)__popc(peers & eq);
        else if (!same) add = 1ull;               // hash collision inside the warp: insert on its own
        else continue;                            // counted by the leader
        const unsigned long long tag = (h >> 31) << 31;                     // top 33 bits
        const unsigned long long mine = tag | (unsigned long long)i;        // i < 2^31
        unsigned long long s = splitmix64(h) & mask;
        for (;;) {
            unsigned long long cur = atomicCAS(slots + s, kEmptyKey, mine);
            if (cur == kEmptyKey) { atomicAdd(counts + s, add); break; }
            if ((cur >> 31) == (tag >> 31) && same_cell(chars, offsets, i, (long long)(cur & 0x7FFFFFFFull))) {
                atomicAdd(counts + s, add);
                break;
            }
            s = (s + 1) & mask;
        }
    }
}

__global__ void k_hash_compact_str(const unsigned long long *__restrict__ slots, const unsigned long long *__restrict__ counts,
                                   unsigned long long nslots, long long *__restrict__ out_rows,
                                   unsigned long long *__restrict__ out_counts, unsigned long long capacity,
                                   unsigned long long *__restrict__ n_out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nslots;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = slots[i];
        if (k != kEmptyKey) {
            const unsigned long long pos = atomicAdd(n_out, 1ull);
            if (pos < capacity) { out_rows[pos] = (long long)(k & 0x7FFFFFFFull); out_counts[pos] = counts[i]; }
        }
    }
}

// R-semantics cast "number" (data_type_update.py:40-43): one cell per thread, CPython float() grammar,
// correctly rounded binary64 (parse_number.cuh) + the is_integer() flag the adapter turns into int(v)
__global__ void k_parse_number(const uint8_t *__restrict__ chars, const long long *__restrict__ offsets, long long n,
                               unsigned long long *__restrict__ value_bits, uint8_t *__restrict__ status) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = offsets[i], e = offsets[i + 1];
        uint64_t bits = 0;
        const long long len = e - b;
        uint8_t st = (len < 0 || len > num::kMaxLen) ? (uint8_t)num::kUnsupported
                                                     : num::parse_number(chars + b, (int)len, bits);
        value_bits[i] = bits;
        status[i] = st;
    }
}

// R-semantics cast "string" (data_type_update.py:22-28): str(v) / None -> "" of one cell per thread
// (format_number.cuh).  Pass 1 writes each cell's length (the input of the offsets scan) and the first row whose status
// or value cannot be formatted; pass 2 writes each cell's text at its scanned offset.  Both run the same format_cell.
__global__ void k_format_number_len(const unsigned long long *__restrict__ value_bits, const uint8_t *__restrict__ status,
                                    long long n, long long *__restrict__ lengths, unsigned long long *__restrict__ first_bad) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int len = fmt::format_cell(value_bits[i], status[i], nullptr);
        if (len < 0) {
            atomicMin(first_bad, (unsigned long long)i);
            len = 0;
        }
        lengths[i] = len;
    }
}

__global__ void k_format_number_write(const unsigned long long *__restrict__ value_bits, const uint8_t *__restrict__ status,
                                      long long n, const long long *__restrict__ offsets, uint8_t *__restrict__ chars) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        fmt::format_cell(value_bits[i], status[i], chars + offsets[i]);
}

// exhaustive self-test: every one of the 2^32 fp32 bit patterns through both divide variants
__global__ void k_selftest_fastdiv(float lo, float hi, float w, int nbins, unsigned long long *mismatches) {
    BinParams B = {lo, hi, w, __frcp_rn(w), nbins - 1};
    unsigned long long bad = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < (1ull << 32);
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const float f = __uint_as_float((unsigned)i);
        bad += bin_index_f32<true>(f, B) != bin_index_f32<false>(f, B);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, s);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatches, bad);
}

// every fp32 bit pattern: the edge-table counter (edge_counter_offset, as the EDGES kernels use it) against the counter of
// the IEEE-divide bin, or the trash counter where that skips the value
__global__ void __launch_bounds__(256) k_selftest_edges(float lo, float hi, float w, int nbins, const float *edges,
                                                        unsigned long long *mismatches) {
    __shared__ uint4 tab[kEdgeSlots];
    load_edge_table(tab, edges, nbins);
    __syncthreads();
    const EdgeParams E = edge_params(lo, w, tab);
    const BinParams B = {lo, hi, w, __frcp_rn(w), nbins - 1};
    unsigned long long bad = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < (1ull << 32);
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const float f = __uint_as_float((unsigned)i);
        const int b = bin_index_f32<false>(f, B);
        bad += edge_counter_offset(f, E) != (b >= 0 ? bin_byte_offset((uint32_t)b) : kTrashOffset);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, s);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatches, bad);
}

template <typename T>
__global__ void k_checksum(const T *col, long long nrows, long long row_offset, unsigned long long *out) {
    unsigned long long acc = 0;
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < nrows;
         r += (long long)gridDim.x * blockDim.x) {
        unsigned long long bits;
        if (sizeof(T) == 8)      bits = (unsigned long long)reinterpret_cast<const unsigned long long *>(col)[r];
        else if (sizeof(T) == 4) bits = (unsigned long long)reinterpret_cast<const unsigned int *>(col)[r];
        else                     bits = (unsigned long long)reinterpret_cast<const unsigned char *>(col)[r];
        acc += bits * (2ull * (unsigned long long)(row_offset + r) + 1ull);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

}  // namespace lo

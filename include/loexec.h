/*
 * loexec.h — C ABI of libloexec.so, the H100-native (sm_90a) executor for
 * learningOrchestra's projection -> type-cast -> histogram hot path.
 *
 * The reference has no native boundary on this path: it crosses from Python
 * into py4j/JVM (Spark) and pymongo/mongod.  Each entry point below names the
 * reference call site whose work it replaces (paths relative to
 * /root/reference/microservices):
 *
 *   lo_project_cast*        projection_image/projection.py:35-46   (load/filter/select/write)
 *                           data_type_handler_image/data_type_update.py:30-43 (per-value cast)
 *   lo_project_cast_hist*   the two above fused with
 *                           histogram_image/histogram.py:28-42     ($group/$sum:1 per field)
 *   lo_hist_u8_cols*        histogram_image/histogram.py:31-36 on byte columns
 *                           ($group value counts == 256 unit-width bins)
 *   lo_table_*              database_api_image/database.py:124-151 (the table the path reads;
 *                           here: columnar slabs resident in HBM instead of Mongo documents)
 *
 * Conventions
 *   - every function returns LO_OK (0) or a negative LO_ERR_*; the message of
 *     the last failure on the calling thread is lo_last_error().
 *   - plain C types only.  `stream` arguments are a cudaStream_t passed as
 *     void* (NULL = the context's own stream).  Functions whose name ends in
 *     `_dev` are asynchronous on `stream` and touch only device memory;
 *     all others synchronise before returning.
 *   - the caller owns every host buffer; the library owns device allocations
 *     behind lo_table handles and never keeps a host pointer after return.
 *   - there is NO CPU fallback: without a usable CUDA device lo_init fails with
 *     LO_ERR_NO_DEVICE and nothing else can be called.
 *   - re-entrant: no mutable global state except the thread-local error string;
 *     concurrent calls on one lo_ctx are allowed when they use different streams.  No entry point
 *     synchronises the whole device: a call waits only for the stream it was given (or the context's own).
 *   - several GPUs: a lo_group (below) owns the peer mappings, the merge buffers and the optional NCCL
 *     communicator; lo_group_* calls take one table / stream per LOCAL member device.
 */
#ifndef LOEXEC_H
#define LOEXEC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LO_ABI_VERSION 3

#define LO_OK                    0
#define LO_ERR_INVALID          -1   /* bad argument (message says which)              */
#define LO_ERR_CUDA             -2   /* a CUDA runtime call failed                      */
#define LO_ERR_NOMEM            -3   /* device or pinned-host allocation failed         */
#define LO_ERR_NOT_IMPLEMENTED  -4
#define LO_ERR_NO_DEVICE        -5   /* no CUDA device / wrong architecture             */
#define LO_ERR_ALIGNMENT        -6   /* external device pointer not 32-byte aligned     */

/* element types of a columnar table */
#define LO_F64 1   /* IEEE binary64 */
#define LO_F32 2   /* IEEE binary32 */
#define LO_U8  3   /* unsigned byte */
#define LO_U32 4   /* dictionary codes (host entry points only) */

/* synthetic generators (oracle/bsem.c and oracle/bsem_numpy.py hold the bit-identical CPU twins) */
#define LO_SYNTH_UNIFORM   0  /* f64: lo + (hi-lo) * (splitmix64(...)>>11) * 2^-53            */
#define LO_SYNTH_EDGES     1  /* UNIFORM + special values where row % 1009 == col % 1009       */
#define LO_SYNTH_CONSTCOL  2  /* EDGES + column 0 constant (contention worst case)           */
#define LO_SYNTH_MNIST_U8  3  /* u8: 28x28 image columns, border 0, ~80 % zeros overall      */

#define LO_MAX_BINS 65536     /* bins per column of a binned histogram                         */
#define LO_TILE_BINS 256      /* up to here the fused tile kernel's per-thread byte counters;  */
                              /* above: the chunk kernel's 32-bit shared / L2 counters         */

typedef struct lo_ctx   lo_ctx;    /* one per (process, device) */
typedef struct lo_table lo_table;  /* columnar table: ncols slabs of nrows elements, one dtype */

/* Fixed-width histogram request (B-semantics, SURVEY.md §8c):
 *   for projected column j with range [lo[j], hi[j]] (fp32) and nbins bins, over the
 *   CAST fp32 value x:  skip NaN and x outside [lo,hi];  w = (hi-lo)/nbins (fp32 RN);
 *   i = (int)((x-lo)/w) (fp32 RN sub, fp32 RN div, truncate);  i = min(i, nbins-1).
 *   lo/hi are HOST arrays of k floats.  Counts are uint64, layout [k][nbins].
 *   nbins <= LO_TILE_BINS runs the fused tile kernel, larger nbins the chunk kernel (same arithmetic and results;
 *   DESIGN.md 3.4.1). */
typedef struct lo_hist_spec {
    int32_t      nbins;     /* 1..LO_MAX_BINS */
    int32_t      flags;     /* must be 0 */
    const float *lo;        /* k lower edges  */
    const float *hi;        /* k upper edges (closed) ; hi[j] > lo[j], both finite */
} lo_hist_spec;

/* per-call device timing filled by the *_host entry points (milliseconds) */
typedef struct lo_host_timing {
    double total_ms;   /* wall time inside the call                      */
    double h2d_bytes;  /* bytes copied host -> device                    */
    double d2h_bytes;  /* bytes copied device -> host                    */
    int64_t launches;  /* kernels launched                               */
    double kernel_ms;  /* device time of the call's kernels between two events on its stream (parser, formatter,
                          group-by); 0 for the chunked pipelines, whose kernels overlap their copies   */
} lo_host_timing;

/* ---- context ------------------------------------------------------------------------- */
int         lo_abi_version(void);
const char *lo_last_error(void);
int         lo_device_count(int *out);
int         lo_init(int device, lo_ctx **out);
int         lo_shutdown(lo_ctx *ctx);
int         lo_ctx_device(const lo_ctx *ctx, int *device, int *sm_count, size_t *hbm_bytes);
int         lo_sync(lo_ctx *ctx, void *stream);
/* choose how full tiles of the fused kernel are fed: 0 = register-pipelined LDG.E.256 (default), 1 = TMA bulk
 * copies into a shared-memory ring (cp.async.bulk + mbarrier).  Same results; also set by LOEXEC_TMA=1 at lo_init. */
int         lo_set_tma(lo_ctx *ctx, int enabled);
/* number of kernels this context has launched since lo_init (bench "gpu_launches") */
int         lo_launch_count(const lo_ctx *ctx, int64_t *out);

/* ---- pinned host memory (so *_host calls can overlap copies with kernels) ------------ */
int lo_host_alloc(lo_ctx *ctx, size_t bytes, void **out);
/* flags: LO_HOST_WRITE_COMBINED — for buffers the host only WRITES (staging inputs for the GPU): uncached on the CPU
 * side, no snooping on the PCIe read; CPU reads from such memory are very slow */
#define LO_HOST_WRITE_COMBINED 1
int lo_host_alloc_flags(lo_ctx *ctx, size_t bytes, int32_t flags, void **out);
int lo_host_free(lo_ctx *ctx, void *p);

/* ---- tables --------------------------------------------------------------------------- */
/* library-owned table: each column slab is 256-byte aligned (pitch rounded up) */
int lo_table_alloc(lo_ctx *ctx, int dtype, int64_t nrows, int32_t ncols, lo_table **out);
/* wrap caller-owned device memory (e.g. a torch tensor): column j starts at
 * base + j*pitch_bytes.  Not freed by lo_table_free. */
int lo_table_wrap(lo_ctx *ctx, int dtype, int64_t nrows, int32_t ncols,
                  void *base_dev, int64_t pitch_bytes, lo_table **out);
int lo_table_free(lo_ctx *ctx, lo_table *t);
int lo_table_info(const lo_table *t, int *dtype, int64_t *nrows, int32_t *ncols,
                  int64_t *pitch_bytes, void **base_dev);
/* host <-> device, one column slab (or a row range of it) at a time; synchronous */
int lo_table_upload_col(lo_ctx *ctx, lo_table *t, int32_t col, int64_t row0,
                        const void *host, int64_t nrows);
/* ordered after everything already enqueued on `stream` (NULL = the context's stream); waits for that stream only */
int lo_table_download_col(lo_ctx *ctx, const lo_table *t, int32_t col, int64_t row0,
                          void *host, int64_t nrows, void *stream);
/* fill every column on the device with the counter-based generator; row r of this table is
 * global row (row_offset + r), so any shard regenerates its own range. */
int lo_table_fill_synthetic_dev(lo_ctx *ctx, lo_table *t, int kind, uint64_t seed,
                                int64_t row_offset, double lo, double hi, void *stream);
/* position-weighted 64-bit checksum of one column slab's bit patterns:
 *   sum_r  bits(x[r]) * (2*(row_offset+r)+1)  mod 2^64   (bits zero-extended to 64) */
int lo_table_checksum(lo_ctx *ctx, const lo_table *t, int32_t col, int64_t row_offset,
                      uint64_t *out);

/* Exhaustive self-test of the binning arithmetic for one (lo, hi, nbins): runs all 2^32 fp32 bit
 * patterns through the branch-free divide the fast kernels use AND through the IEEE divide, and
 * returns how many bin indices differ (must be 0 whenever *fast_path_used == 1, i.e. whenever the
 * library would pick the fast kernels for this range; ranges that fail the safety conditions run
 * the IEEE-divide kernels instead). */
int lo_selftest_fastdiv(lo_ctx *ctx, float lo, float hi, int32_t nbins, int *fast_path_used,
                        uint64_t *mismatches);

/* Bin edges of the edge-table tile kernels (host only, no device needed): edges[0] = lo, edges[i] = the smallest fp32
 * value in [lo, hi] whose bin is >= i (the next value above hi when bins i.. are empty), edges[nbins] = the next fp32
 * value above hi.  edges: nbins + 1 floats. */
int lo_hist_edges(float lo, float hi, int32_t nbins, float *edges);

/* Every fp32 bit pattern through the edge-table binning of the tile kernels against the IEEE-divide bin (nbins <=
 * LO_TILE_BINS).  *edges_used: whether histograms with this range take the edge-table kernels. */
int lo_selftest_edges(lo_ctx *ctx, float lo, float hi, int32_t nbins, int *edges_used, uint64_t *mismatches);

/* The context's cache of device edge tables: tables held now (at most 8, least recently used retired first), their
 * bytes, and how many tile-kernel launches so far binned with the IEEE divide instead (bin widths outside
 * [2^-100, 2^100]).  Any pointer may be NULL. */
int lo_edge_tables_info(lo_ctx *ctx, int32_t *tables, uint64_t *bytes, int64_t *divide_launches);

/* ---- the hot path, device-resident ------------------------------------------------------ */
/* out[j][r] = cast(in[col_idx[j]][r]) for j < k.  in: LO_F64.  out: LO_F32 (fp64->fp32 RNE,
 * NaN -> 0x7fc00000) or LO_F64 (plain copy).  out->ncols >= k, out->nrows == in->nrows. */
int lo_project_cast_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                        lo_table *out, void *stream);
/* fused: projection + cast + per-column histogram of the cast value.  out may be NULL
 * (histogram only).  counts_dev: device uint64[k*nbins], ACCUMULATED into (caller zeroes,
 * e.g. with lo_counts_zero_dev) so shards / chunks add up. */
int lo_project_cast_hist_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                             lo_table *out, const lo_hist_spec *spec, uint64_t *counts_dev,
                             void *stream);
/* per-column 256-bin value counts of LO_U8 columns; counts_dev: uint64[k*256], accumulated */
int lo_hist_u8_cols_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                        uint64_t *counts_dev, void *stream);
/* range pre-pass on RESIDENT columns: out_dev = device uint64[3*k] (lo_counts_alloc), zeroed by the call;
 * download it (lo_counts_download) and decode with lo_minmax_decode (host-only helper). */
int lo_minmax_cast_dev(lo_ctx *ctx, const lo_table *in, const int32_t *col_idx, int32_t k,
                       uint64_t *out_dev, void *stream);
int lo_minmax_decode(const uint64_t *raw, int32_t k, float *mins, float *maxs, uint64_t *nfinite);
/* device scratch for counts */
int lo_counts_alloc(lo_ctx *ctx, int64_t n, uint64_t **out_dev);
int lo_counts_free(lo_ctx *ctx, uint64_t *counts_dev);
int lo_counts_zero_dev(lo_ctx *ctx, uint64_t *counts_dev, int64_t n, void *stream);
int lo_counts_download(lo_ctx *ctx, const uint64_t *counts_dev, int64_t n, uint64_t *host,
                       void *stream);

/* ---- the hot path, host buffers in / host buffers out (what the plugin calls) ----------- */
/* in_cols[j]  : host pointer to the nrows doubles of projected column j (already selected by
 *               the caller: the document->column gather is the adapter's job)
 * out_cols[j] : host pointer receiving nrows floats, or out_cols == NULL for histogram only
 * spec        : NULL for projection+cast only
 * counts      : host uint64[k*nbins], overwritten
 * Rows are streamed through the device in chunks on three streams (H2D / kernel / D2H);
 * copies overlap kernels when the host buffers are pinned (lo_host_alloc). */
int lo_project_cast_hist_host(lo_ctx *ctx, const double *const *in_cols, int64_t nrows, int32_t k,
                              float *const *out_cols, const lo_hist_spec *spec, uint64_t *counts,
                              lo_host_timing *timing);
/* in_cols[j]: host pointer to nrows bytes; counts: host uint64[k*256], overwritten */
int lo_hist_u8_cols_host(lo_ctx *ctx, const uint8_t *const *in_cols, int64_t nrows, int32_t k,
                         uint64_t *counts, lo_host_timing *timing);

/* ---- several GPUs: row-range shards, one merged count matrix ------------------------------------------
 * The reference has no multi-device path (one mongod pipeline per field, histogram_image/histogram.py:31-36; three
 * single-core Spark executors, projection_image/server.py:58-60).  Here rows are range-sharded over the GPUs of one
 * box and the per-GPU partial histograms are merged INSIDE the streaming kernel: every device accumulates its own
 * matrix, the CTA that finishes a column's last tile pushes that column's bins into the root device's matrix with
 * system-scope RED.64 over NVLink, the last pusher release-adds an arrival counter, and the root's last CTA moves the
 * merged matrix out, re-zeroes and signals the peers — one kernel launch per device per step, no separate collective
 * (LO_MERGE_PEER).  LO_MERGE_NCCL is the conventional form: local matrix + one ncclAllReduce(uint64, sum) on the
 * same stream, through the libnccl.so.2 found at run time (dlopen; the library does not link against NCCL).
 *
 * Two ways to form a group:
 *   - lo_group_create_local: ONE process drives several devices (what a single microservice process does on an
 *     8-GPU box); peer access is enabled directly.
 *   - lo_group_rank_begin / lo_group_rank_connect: one process per device (torchrun-style).  As with
 *     ncclGetUniqueId / ncclCommInitRank the library produces an opaque blob per rank, the launcher's own
 *     out-of-band channel gathers the W blobs, and every rank connects with all of them (CUDA IPC inside).
 * All members must issue the same sequence of lo_group_* calls.  Member 0 / rank 0 is the root. */
typedef struct lo_group lo_group;
#define LO_GROUP_BLOB_BYTES 512
#define LO_GROUP_MAX_DEVICES 16
#define LO_GROUP_MAX_COUNTS  262144   /* entries of the largest merged matrix (1024 byte columns x 256) */
#define LO_MERGE_AUTO 0   /* peer-memory merge when every pair of devices has peer access, else NCCL */
#define LO_MERGE_PEER 1
#define LO_MERGE_NCCL 2
#define LO_GROUP_BCAST 1  /* call flag: every member receives the merged matrix (all-reduce); default: root only */
#define LO_GROUP_INDEPENDENT 2 /* call flag (lo_group_*_dev): this step reads nothing the PREVIOUS group step on the same
                                * streams wrote, so its CTAs may start while that step's last wave is still draining
                                * (programmatic dependent launch; the steps use alternating accumulate matrices).  Other
                                * work on the stream — and a step without the flag — still waits for full completion. */

int lo_group_create_local(lo_ctx *const *ctxs, int32_t n, int32_t merge, lo_group **out);
int lo_group_rank_begin(lo_ctx *ctx, int32_t rank, int32_t world, int32_t merge, lo_group **out,
                        void *blob /* LO_GROUP_BLOB_BYTES, filled */);
int lo_group_rank_connect(lo_group *g, const void *blobs /* world * LO_GROUP_BLOB_BYTES, rank order */);
int lo_group_destroy(lo_group *g);
/* world size, members driven by this process, the merge actually in use (LO_MERGE_PEER / LO_MERGE_NCCL) */
int lo_group_info(const lo_group *g, int32_t *world, int32_t *nlocal, int32_t *merge);
/* rows [begin, end) of a `total_rows` table owned by member `index`; interior cuts are multiples of 32 rows */
int lo_group_shard(const lo_group *g, int64_t total_rows, int32_t index, int64_t *begin, int64_t *end);

/* The hot path over the group.  in[i] / out[i] / streams[i]: the shard, output table (or out == NULL) and stream
 * (or streams == NULL: each context's own) of LOCAL member i.  Asynchronous.  The merged k x nbins matrix of the
 * step lands in the group's result buffer on the root (on every member with LO_GROUP_BCAST or LO_MERGE_NCCL);
 * read it with lo_group_result.  k <= 128 (f64) / 1024 (u8) per call. */
int lo_group_project_cast_hist_dev(lo_group *g, const lo_table *const *in, const int32_t *col_idx, int32_t k,
                                   lo_table *const *out, const lo_hist_spec *spec, int32_t flags,
                                   void *const *streams);
int lo_group_hist_u8_cols_dev(lo_group *g, const lo_table *const *in, const int32_t *col_idx, int32_t k,
                              int32_t flags, void *const *streams);
/* range pre-pass over all shards (SURVEY.md §2.1 C2): merged per-column min / max / finite count of the cast values;
 * read with lo_group_result(n = 3*k) and decode with lo_minmax_decode.  Always delivered to every member. */
int lo_group_minmax_cast_dev(lo_group *g, const lo_table *const *in, const int32_t *col_idx, int32_t k,
                             void *const *streams);
/* host buffers in / out, rows of THIS process only: with a local group the library cuts [0, nrows) into one row range
 * per member and drives one H2D / kernel / D2H pipeline per device (a host thread each); with a rank group every
 * rank passes its own shard.  counts: merged k x nbins matrix (root / member 0; every rank with LO_GROUP_BCAST). */
int lo_group_project_cast_hist_host(lo_group *g, const double *const *in_cols, int64_t nrows, int32_t k,
                                    float *const *out_cols, const lo_hist_spec *spec, uint64_t *counts,
                                    int32_t flags, lo_host_timing *timing);
int lo_group_hist_u8_cols_host(lo_group *g, const uint8_t *const *in_cols, int64_t nrows, int32_t k,
                               uint64_t *counts, int32_t flags, lo_host_timing *timing);
/* waits for the last step on local member `member` and copies the first n entries of its result buffer.
 * LO_ERR_INVALID when that member holds no result (non-root without LO_GROUP_BCAST / NCCL). */
int lo_group_result(lo_group *g, int32_t member, int64_t n, uint64_t *host);
/* device pointer of a local member's result buffer (valid until lo_group_destroy; contents: the last step) */
int lo_group_result_dev(lo_group *g, int32_t member, uint64_t **dev_ptr);
/* device-side barrier over all members on the given streams (a few microseconds of skew instead of a host barrier's
 * tens): every stream continues once all W devices have reached it.  Peer merge only. */
int lo_group_barrier_dev(lo_group *g, void *const *streams);
/* number of bounded device-side waits that gave up (a lost or wedged peer) since the group was formed; must be 0 */
int lo_group_timeouts(lo_group *g, uint64_t *out);

/* pin the CALLING thread to the CPUs local to the context's GPU (PCI device's NUMA node, from sysfs): pinned host
 * buffers allocated and first touched afterwards land on the memory next to the GPU's PCIe root. */
int lo_ctx_bind_numa(lo_ctx *ctx, int32_t *node_out, int32_t *ncpus_out);

/* Exact value counts of one dictionary-encoded column (R-semantics `$group`/`$sum:1`,
 * histogram_image/histogram.py:31-36, for columns with more than 256 distinct keys):
 * counts[c] = number of rows whose code is c; counts: host uint64[ncodes], overwritten.
 * A code >= ncodes fails with LO_ERR_INVALID. */
int lo_value_counts_u32_host(lo_ctx *ctx, const uint32_t *codes, int64_t nrows, uint32_t ncodes,
                             uint64_t *counts, lo_host_timing *timing);
/* Exact value counts of one NUMERIC column without a host dictionary (GPU hash group-by): keys are
 * compared with MongoDB's `$group` equality for numbers (-0.0 == 0.0 -> key +0.0, every NaN -> one NaN key).
 * keys_out / counts_out: host arrays of `capacity` entries, filled in unspecified order (as `$group`);
 * *ndistinct = number of groups.  More groups than capacity -> LO_ERR_INVALID (ndistinct still set). */
int lo_value_counts_f64_host(lo_ctx *ctx, const double *values, int64_t n, double *keys_out,
                             uint64_t *counts_out, int64_t capacity, int64_t *ndistinct,
                             lo_host_timing *timing);

/* The same for one TEXT column: cell i = chars[offsets[i] .. offsets[i+1]) (offsets[0] == 0, n < 2^31).  Keys are
 * compared byte for byte on the device (exact whatever the hash does).  rep_rows_out[g] = row index of one member
 * of group g — the caller reads the key from its own cell — and counts_out[g] its size; order unspecified. */
int lo_value_counts_str_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n,
                             int64_t *rep_rows_out, uint64_t *counts_out, int64_t capacity,
                             int64_t *ndistinct, lo_host_timing *timing);

/* Text -> number for one column of cells: the reference's REAL cast, `float(document[field])` followed by
 * `is_integer()` (data_type_handler_image/data_type_update.py:40-43), for every cell at once on the GPU.
 * chars holds all cells back to back, cell i = chars[offsets[i] .. offsets[i+1]).  values[i] receives exactly
 * the binary64 CPython's float() returns (correctly rounded; grammar incl. '_', inf, nan, whitespace).
 * status[i]: LO_NUM_FLOAT 0 | LO_NUM_INTEGER 1 (integer valued: store int(v)) | LO_NUM_EMPTY 2 ("" -> None) |
 * LO_NUM_INVALID 3 (float() raises ValueError) | LO_NUM_UNSUPPORTED 4 (cell > 1 MiB, or a byte >= 0x80: the caller
 * passes the ASCII text float(str) itself parses after mapping Unicode digits / whitespace — a code-point property
 * lookup the Python packer does, columnar.ascii_number_text). */
#define LO_NUM_FLOAT 0
#define LO_NUM_INTEGER 1
#define LO_NUM_EMPTY 2
#define LO_NUM_INVALID 3
#define LO_NUM_UNSUPPORTED 4
int lo_parse_number_host(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, int64_t n,
                         double *values, uint8_t *status, lo_host_timing *timing);

/* Number -> text for one column: the reference's "string" cast, str(v) / None -> "" (data_type_handler_image/
 * data_type_update.py:22-28), for every cell at once on the GPU.  The inverse of lo_parse_number_host.
 * status[i] uses the LO_NUM_* codes above: FLOAT -> repr(float) (shortest round-trip digits, CPython's notation),
 * INTEGER -> str(int) (values[i] finite and integral; every digit of the exact value), EMPTY -> "".  Any other status,
 * or an INTEGER cell that is not finite and integral -> LO_ERR_INVALID, the message names the first such row.
 * offsets: host int64[n+1], always written, offsets[0] == 0; cell i is chars[offsets[i] .. offsets[i+1]) (the layout of
 * an Arrow large_string array).  chars: written when chars_capacity >= offsets[n]; chars == NULL with
 * chars_capacity == 0 asks for the sizes only; a non-NULL buffer that is too small -> LO_ERR_INVALID (offsets still
 * written).  One cell is at most LO_FORMAT_MAX_CELL bytes (a FLOAT cell at most 24). */
#define LO_FORMAT_MAX_CELL 310
int lo_format_number_host(lo_ctx *ctx, const double *values, const uint8_t *status, int64_t n,
                          int64_t *offsets, uint8_t *chars, int64_t chars_capacity, lo_host_timing *timing);

/* Per-column min and max of the CAST fp32 values over finite entries (NaN / +-inf ignored): the
 * range pre-pass for a histogram request that carries no range (SURVEY.md §2.1 C2).
 * mins / maxs: host float[k]; nfinite: host uint64[k] (0 -> min = max = 0). */
int lo_minmax_cast_host(lo_ctx *ctx, const double *const *in_cols, int64_t nrows, int32_t k,
                        float *mins, float *maxs, uint64_t *nfinite, lo_host_timing *timing);

/* CSV text -> text columns: the reference's upload reader, csv.reader(codecs.iterdecode(response.iter_lines(),
 * "utf-8"), delimiter=",", quotechar='"') followed by __treat_row (database_api_image/database.py:110-137), tokenised on
 * the GPU.  Lines end at every run of '\r' / '\n' (blank lines vanish, a line break inside quotes is dropped); fields
 * follow CPython's _csv reader with the default dialect; a field holds at most 131072 code points; UTF-8 is decoded
 * strictly line by line; NUL is rejected (Python 3.7's _csv).  Record 0 is the header and fixes ncols; a data record
 * with more fields keeps the first ncols, one with fewer fails.
 *
 * lo_csv_read_host copies the body to the device, tokenises it and keeps the columns of every record before the first
 * failing one on the device.  info->records = header + kept data rows (0 when the header itself fails or the body has
 * no record); info->fail_record = the failing record (-1: none), info->fail_kind = why, info->fail_pos = the byte
 * offset the failure was raised at (line start for LO_CSV_BAD_UTF8 / LO_CSV_UNSUPPORTED; -1 for LO_CSV_SHORT_ROW and
 * LO_CSV_EMPTY).  The device needs about the body, 0.5 bytes per body byte of scratch, 8 bytes per kept cell and the
 * text; more than is free -> LO_ERR_NOMEM naming the size.
 * lo_csv_columns_host: offsets host int64[ncols][records + 1] (column c's cell r = chars[offsets[c][r] ..
 * offsets[c][r+1]), absolute in ONE column-major chars buffer: the buffers of Arrow large_string arrays) and chars
 * (info->chars bytes; chars_capacity smaller -> LO_ERR_INVALID).  lo_csv_free releases the handle (NULL is fine). */
#define LO_CSV_OK           0
#define LO_CSV_SHORT_ROW    1   /* a data record has fewer fields than the header (IndexError in __treat_row)     */
#define LO_CSV_FIELD_LIMIT  2   /* a field of more than 131072 code points (_csv.Error)                          */
#define LO_CSV_BAD_UTF8     3   /* a line is not valid UTF-8 (UnicodeDecodeError)                                */
#define LO_CSV_NUL          4   /* a line contains NUL (_csv.Error in Python 3.7)                                */
#define LO_CSV_UNSUPPORTED  5   /* a line ends inside a UTF-8 sequence: the decoder would join it with the next   */
#define LO_CSV_EMPTY        6   /* no record at all (StopIteration reading the header)                           */
typedef struct lo_csv lo_csv;
typedef struct lo_csv_info {
    int64_t records;       /* header + kept data rows */
    int64_t ncols;
    int64_t chars;         /* bytes of text of all kept cells */
    int64_t fail_record;
    int32_t fail_kind;     /* LO_CSV_* */
    int32_t pad;
    int64_t fail_pos;
} lo_csv_info;
int lo_csv_read_host(lo_ctx *ctx, const uint8_t *body, int64_t nbytes, lo_csv **out, lo_csv_info *info,
                     lo_host_timing *timing);
int lo_csv_columns_host(lo_csv *h, int64_t *offsets, uint8_t *chars, int64_t chars_capacity, lo_host_timing *timing);
int lo_csv_free(lo_csv *h);

/* The same reader on a body fed in pieces, with device memory bounded by a window instead of the body.
 *
 * lo_csv_stream_open: window_bytes = the window's starting capacity W (0 -> LO_CSV_STREAM_WINDOW).
 * lo_csv_stream_push: hands the stream `n` more bytes of the body; last = 1 says they end it (n may be 0).  Pieces may
 *   be of any size and cut anywhere (inside "\r\n", a UTF-8 sequence, a "" pair, a quoted multi-line field, a record):
 *   the result does not depend on the cuts.  The stream copies what fits into its window [tail of the last window |
 *   new bytes]; when the window is full, or holds the body's last byte, it reads the window up to one past the last
 *   byte that ended a record (all of it at the end of the body) and keeps the rest as the next window's tail.  A push
 *   reads at most one window: win->consumed says how many of the n bytes it took, and the caller pushes the others
 *   again (with the same `last`).  win->records records were read (win->first_record = the absolute index of the
 *   first; record 0 is the header) with win->ncols columns and win->chars bytes of text; lo_csv_stream_columns copies
 *   them out in lo_csv_columns_host's layout (offsets int64[ncols][records + 1], absolute in the window's chars), and
 *   must be called before the next push, which releases them.
 *   A full window in which no record ends doubles its capacity; only a record the device cannot hold fails, with
 *   LO_ERR_NOMEM naming its size.
 *   *info is the body so far as lo_csv_read_host reports it: once win->done, it equals lo_csv_read_host's info on the
 *   whole body (records, ncols, chars summed over the windows; fail_record and fail_pos absolute in the body).  The
 *   stream is done after the last byte, or after the first failing record: the rows before it have been delivered,
 *   and later pushes take their bytes and do nothing.  Any other error (LO_ERR_NOMEM, LO_ERR_CUDA) ends the stream:
 *   later pushes fail with LO_ERR_INVALID.
 * Device memory: with W the window's capacity (window_bytes, doubled while a record does not fit in it), the stream
 *   holds at most 2W (the window and its tail buffer) + 0.47W (segment scratch) + CUB temporary storage + the columns
 *   of one window: 8 bytes per kept cell + 8 (ncols + 1) + at most W of text; a cell takes at least half a byte of
 *   the window, so in no case more than 19.5W + CUB storage + 8 (ncols + 1).  It does not grow with the body.
 *   win->peak_device_bytes reports the most the stream has held so far.
 * lo_csv_stream_free releases the stream (NULL is fine).  The calls follow the single-pass rules: no device-wide
 * synchronisation, scratch from the stream-ordered pool, the first error reported, lo_host_timing filled per call. */
#define LO_CSV_STREAM_WINDOW (64ll << 20)
typedef struct lo_csv_stream lo_csv_stream;
typedef struct lo_csv_window {
    int64_t consumed;            /* bytes of this push taken by the stream */
    int64_t records;             /* records read by this push (their columns: lo_csv_stream_columns) */
    int64_t first_record;        /* absolute index of the first of them */
    int64_t ncols;
    int64_t chars;               /* their bytes of text */
    int64_t peak_device_bytes;   /* the most device memory the stream has held so far */
    int32_t done;                /* 1: the body is read, or a record failed */
    int32_t pad;
} lo_csv_window;
int lo_csv_stream_open(lo_ctx *ctx, int64_t window_bytes, lo_csv_stream **out);
int lo_csv_stream_push(lo_csv_stream *st, const uint8_t *bytes, int64_t n, int32_t last, lo_csv_window *win,
                       lo_csv_info *info, lo_host_timing *timing);
int lo_csv_stream_columns(lo_csv_stream *st, int64_t *offsets, uint8_t *chars, int64_t chars_capacity,
                          lo_host_timing *timing);
int lo_csv_stream_free(lo_csv_stream *st);

#ifdef __cplusplus
}
#endif
#endif /* LOEXEC_H */

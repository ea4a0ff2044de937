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

#define LO_ABI_VERSION 7

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
#define LO_I32 5   /* dictionary codes of a text column (lo_text_codes): read by lo_assemble_rows only, refused elsewhere */

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
/* device -> device: column src_col of src into column dst_col of dst, both on ctx's device, same dtype and rows
 * (else LO_ERR_INVALID); on the context's stream, waited for */
int lo_table_copy_col(lo_ctx *ctx, const lo_table *src, int32_t src_col, lo_table *dst, int32_t dst_col);
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
 * read it with lo_group_result.  k <= 128 (f64) / 1024 (u8) per call, and k * nbins <= LO_GROUP_MAX_COUNTS: the
 * group's matrices hold that many counts, so the f64 entry points (_dev and _host) return LO_ERR_INVALID for a larger
 * step before launching anything; split its columns over several steps. */
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
/* The same on rows [0, nrows) of column `col` of a device table (LO_F64), e.g. a dataset's slab kept in HBM for
 * repeated `$group` requests: nothing crosses PCIe but the groups (h2d_bytes 0), two kernel launches.  A null stored as
 * NaN in the slab counts under the NaN key: the caller, which knows its nulls, separates them from real NaNs.
 * LO_ERR_INVALID before anything is enqueued for a NULL table, a table that is not LO_F64 or lives on another
 * context's device, `col` outside [0, ncols), or NULL outputs with capacity > 0.  Not `_dev`: it synchronises and
 * writes host arrays.  Both calls run one binary64 group-by kernel: warp-merged keys are staged in a per-CTA
 * shared-memory table before the global one (16-byte loads when the column is 16-byte aligned, as every slab of
 * lo_table_alloc is). */
int lo_value_counts_f64_table(lo_ctx *ctx, const lo_table *t, int32_t col, double *keys_out,
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

/* The same parse written straight into a device table: cell i (i < n) goes to row row0 + i of column `col` of `out`
 * (LO_F64) as the bits float() returns; a null cell and "" store the canonical NaN (0x7ff8000000000000), which the
 * histogram and min/max kernels skip.  chars / offsets are host buffers laid out as for lo_parse_number_host; offsets[0]
 * need not be 0 (a sliced Arrow array), only chars[offsets[0] .. offsets[n]) is copied.  A cell whose offsets leave that
 * range counts as unsupported.  validity: NULL (every cell present), or one of
 *   mask   — n host bytes, 0 = cell i is null;
 *   bitmap — an Arrow validity bitmap, bit (bit_offset + i), least significant bit first, 0 = cell i is null
 * (Arrow does not promise that a null slot is empty: its bytes are never parsed).  Instead of a status per row the call
 * fills *summary: the first invalid row (float() raises ValueError) and the first unsupported row (cell over 1 MiB or a
 * byte >= 0x80), -1 when there is none, relative to the call's first cell; the null + empty cells; and whether every
 * other cell is integer valued (the resident column's "int" kind).  Rows of invalid / unsupported cells hold
 * unspecified values: the caller fails the request. */
typedef struct lo_validity {
    const uint8_t *mask;
    const uint8_t *bitmap;
    int64_t bit_offset;
} lo_validity;
typedef struct lo_parse_summary {
    int64_t first_invalid;
    int64_t first_unsupported;
    int64_t nulls;
    int32_t all_integer;
    int32_t pad;
} lo_parse_summary;
int lo_parse_number_to_table(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, const lo_validity *validity,
                             int64_t n, lo_table *out, int32_t col, int64_t row0, lo_parse_summary *summary,
                             lo_host_timing *timing);

/* One text column resident in HBM, for `$group` requests that come back to the same dataset: the cells cross PCIe once.
 * lo_text_upload takes what lo_parse_number_to_table takes — offsets[0] need not be 0 (only chars[offsets[0] ..
 * offsets[n]) is copied, the device offsets are rebased to 0), validity NULL / mask / bitmap with any bit_offset — and
 * n < 2^31.  It checks free device memory first: too little -> LO_ERR_NOMEM naming the size.  lo_text_info: cells,
 * bytes of text, null cells, device bytes held (any pointer may be NULL).  lo_text_free: NULL is fine.
 * lo_value_counts_text: lo_value_counts_str_host's contract (rep_rows_out / counts_out / capacity / *ndistinct, more
 * groups than capacity -> LO_ERR_INVALID with *ndistinct set) on the resident column: no cell crosses PCIe
 * (h2d_bytes 0), null rows are not counted, representative rows index the whole column, nulls included.  Not `_dev`: it
 * synchronises and writes host arrays.
 * The text group-by kernel stages keys in a per-CTA shared-memory table of LO_TEXT_STAGE_SLOTS slots before the global
 * one, with at most 8 CTAs per SM: a column with more than LO_TEXT_STAGE_SLOTS distinct cells per CTA overflows it,
 * those keys go straight to the global table, and after a few such spills the CTA stops probing its stage. */
#define LO_TEXT_STAGE_SLOTS 512
typedef struct lo_text lo_text;
int lo_text_upload(lo_ctx *ctx, const uint8_t *chars, const int64_t *offsets, const lo_validity *validity,
                   int64_t n, lo_text **out, lo_host_timing *timing);
int lo_text_info(const lo_text *t, int64_t *n, int64_t *nbytes, int64_t *nulls, size_t *device_bytes);
int lo_text_free(lo_ctx *ctx, lo_text *t);
int lo_value_counts_text(lo_ctx *ctx, const lo_text *t, int64_t *rep_rows_out, uint64_t *counts_out,
                         int64_t capacity, int64_t *ndistinct, lo_host_timing *timing);

/* lo_value_counts_text of one text column cut into nshards row-range shards, each a lo_text on any context (several
 * may share one): shards[i] holds the column's rows [row0[i], row0[i] + n_i), disjoint and in row order.  Each shard is
 * counted on its own context's device and stream; its groups are packed into a key column there (cells, global rows,
 * counts), copied to root's device with cudaMemcpyPeerAsync (peer access need not be enabled) and merged there by a
 * second hash pass over the distinct keys only, with 64-bit counts.  The contract is lo_value_counts_text's, with
 * rep_rows_out holding GLOBAL rows (row0[i] + the shard's row); nshards == 1 is lo_value_counts_text plus row0[0].
 * Refused with LO_ERR_INVALID before anything is launched: a NULL root, shards, row0 or shard; nshards outside
 * [1, LO_GROUP_MAX_DEVICES]; a negative, decreasing or overlapping row0; NULL outputs with capacity > 0.  The merge
 * keeps a 31-bit key index: more than 2^31-1 groups summed over the shards -> LO_ERR_INVALID.
 * Launches: 5 on the context of every shard with a non-null cell (count, compact, key lengths, scan, key gather) and
 * 3 on root (merge, compact, global rows).  timing: total_ms is the whole call, kernel_ms the root's merge (between two
 * events on root's stream), launches those on root's context during the call, h2d_bytes 0 and d2h_bytes the groups
 * read back.  The bytes that cross between devices are in neither byte count. */
int lo_value_counts_text_shards(lo_ctx *root, const lo_text *const *shards, const int64_t *row0, int32_t nshards,
                                int64_t *rep_rows_out, uint64_t *counts_out, int64_t capacity, int64_t *ndistinct,
                                lo_host_timing *timing);

/* Dictionary codes of one resident text column, for a GPU consumer that indexes words itself (a model's categorical
 * inputs).  Row i of column `col` of `out` (LO_I32, nrows == the text's n, on the text's device) receives -1 for a null
 * row, else the code of its cell: the distinct non-null cells are numbered 0, 1, ... in the order of their FIRST ROWS
 * (the order of Arrow's dictionary_encode).  Cells compare byte for byte; "" is a cell, not a null.
 * first_rows_out[c] = the first row of code c (ascending): the dictionary is the cells at those rows.  capacity /
 * *ndistinct as in lo_value_counts_text: more distinct cells than capacity -> LO_ERR_INVALID with *ndistinct set and the
 * first `capacity` first rows copied (the codes are written all the same).  Codes do not depend on the hash table's
 * layout, nor on how the column is cut into shards.
 * Refused with LO_ERR_INVALID before anything is launched: a NULL text or out, text made on another context, `out` not
 * LO_I32 or of other rows than the text or on another device, `col` outside [0, ncols), a negative capacity, a NULL
 * ndistinct, a NULL first_rows_out with capacity > 0.
 * Launches: 6 (count, slot pass, compact, radix sort, rank, remap) when a cell is not null, else none (the column is set
 * to -1).  timing: kernel_ms the call's kernels (between events on the context's stream, the group count read between
 * them left out), h2d_bytes 0, d2h_bytes the group count and the first rows read back. */
int lo_text_codes(lo_ctx *ctx, const lo_text *t, lo_table *out, int32_t col, int64_t *first_rows_out,
                  int64_t capacity, int64_t *ndistinct, lo_host_timing *timing);
/* lo_text_codes of one text column cut into nshards row-range shards, laid out as for lo_value_counts_text_shards:
 * shards[i] holds rows [row0[i], row0[i] + n_i), and its codes land in column `col` of out[i], a table on shards[i]'s
 * device.  first_rows_out holds GLOBAL rows; codes and first rows equal lo_text_codes' on the whole column for any cut.
 * Each shard numbers its own cells on its device and packs its distinct cells with their first global rows (the key
 * column of lo_value_counts_text_shards); the keys are copied to root's device, merged there by the lowest first row
 * of each cell and ordered, and each shard copies its keys' codes back and remaps its rows.
 * Refused with LO_ERR_INVALID before anything is launched: a NULL root, shards, row0, out, shard or out[i]; nshards
 * outside [1, LO_GROUP_MAX_DEVICES]; a negative, decreasing or overlapping row0; out[i] failing lo_text_codes' checks
 * against shards[i]; a negative capacity, NULL ndistinct, NULL first_rows_out with capacity > 0.  More than 2^31-1
 * distinct cells summed over the shards -> LO_ERR_INVALID before the root merges.
 * Launches: 8 on the context of every shard with a non-null cell (count, slot pass, compact, key lengths, scan, key
 * gather, rank, remap), none on a shard without one, and 5 on root (merge, compact, radix sort, rank, key remap).
 * timing: total_ms the whole call, kernel_ms the root's merge and ordering, launches those on root's context during the
 * call, h2d_bytes 0, d2h_bytes the group count and first rows read back on root. */
int lo_text_codes_shards(lo_ctx *root, const lo_text *const *shards, const int64_t *row0, int32_t nshards,
                         lo_table *const *out, int32_t col, int64_t *first_rows_out, int64_t capacity,
                         int64_t *ndistinct, lo_host_timing *timing);

/* The feature matrix of a model's training step: Spark 2.4's VectorAssembler(inputCols, outputCol="features") plus its
 * "label" column (builder_image/builder.py:99-134), from k source columns in HBM into one row-major matrix, on the GPU.
 * Source j is column src_col[j] of src[j], an LO_F64 slab (NaN is invalid: a null or a real NaN) or an LO_I32 column of
 * dictionary codes (lo_text_codes; -1 is invalid).  The tables may differ; all live on ctx's device with the same nrows
 * n.  Row i of x (x's column 0, row stride ld >= k elements) is [value(j, i) for j < k]; y[i] (optional, with label /
 * label_col: one more source) is the label's value.  x and y are both LO_F32 (fp64->fp32 RNE, NaN -> 0x7fc00000, codes
 * int->fp32 RNE) or both LO_F64 (exact).  An invalid cell, by mode:
 *   LO_INVALID_ERROR — the call fails with LO_ERR_INVALID; info->bad_row / bad_col name the lowest invalid row and its
 *                      lowest invalid source in that row (k: the label); x and y hold nothing to read;
 *   LO_INVALID_SKIP  — rows with an invalid cell in any source or the label are left out; the kept rows stay in order;
 *   LO_INVALID_KEEP  — written as NaN of the output dtype (a -1 code too; an f64 NaN keeps its bits in LO_F64).
 * info->nkept = the rows written to x and y; kept_rows (host int64[n] or NULL) receives their source rows in output order.
 * x must hold n * ld elements in column 0, y n (the rows skip leaves out stay unwritten).
 * Refused with LO_ERR_INVALID before anything is enqueued: NULL src, src_col, x or info; k outside [1, 2097120]; ld < k; a
 * NULL source, a source that is not LO_F64 / LO_I32, on another device, with src_col outside [0, ncols) or rows other
 * than src[0]'s (the label likewise); an unknown mode; x not LO_F32 / LO_F64 or on another device or too small; y
 * without a label or a label without y; y of another dtype than x, on another device or too small.
 * Launches: none when n == 0; 1 (ERROR, KEEP: the write pass); 3 (SKIP: validity pass, scan of the tiles' kept counts,
 * write pass).  Bytes moved: ERROR / KEEP read every source once and write n rows; SKIP reads every source twice and
 * writes the kept rows (DESIGN.md §3.6.1).  timing: kernel_ms the call's kernels, d2h_bytes the kept rows and the counts
 * read back, h2d_bytes the k source descriptors. */
#define LO_INVALID_ERROR 0
#define LO_INVALID_SKIP  1
#define LO_INVALID_KEEP  2
typedef struct lo_assemble_info {
    int64_t nkept;
    int64_t bad_row;     /* LO_INVALID_ERROR: the lowest row holding an invalid cell, else -1 */
    int32_t bad_col;     /* its lowest invalid source (k: the label), else -1 */
    int32_t pad;
} lo_assemble_info;
int lo_assemble_rows(lo_ctx *ctx, const lo_table *const *src, const int32_t *src_col, int32_t k, const lo_table *label,
                     int32_t label_col, int32_t mode, lo_table *x, int64_t ld, lo_table *y, int64_t *kept_rows,
                     lo_assemble_info *info, lo_host_timing *timing);

/* Spark 2.4's multinomial NaiveBayes (ml.classification.NaiveBayes with smoothing, no weightCol, no thresholds;
 * builder_image/builder.py:55-61's "NB") over a feature matrix of lo_assemble_rows: x holds n rows of k features
 * (column 0, row stride ld >= k elements), y their labels, both LO_F32 or both LO_F64 on ctx's device; every value is
 * widened to f64 exactly.  Classes are label values, ascending; C = their number.  DESIGN.md §3.6.2.
 *
 * lo_nb_labels: the distinct values of y[0 .. n), ascending, into labels_out (host double[capacity]); -0.0 is 0.0.  The
 * f64 hash group-by of lo_value_counts_f64_table (an LO_F32 y is widened on the way in).  *nlabels = their number; more
 * than capacity fails with LO_ERR_INVALID after *nlabels is set, and so does a NaN label (*nlabels set, labels_out
 * unwritten).  Launches: none when n == 0; 2 (LO_F64) or 3 (LO_F32: the widening).  Bytes: y read once (LO_F32: read,
 * written as f64 and read again).  timing: d2h_bytes the groups read back.
 *
 * lo_nb_fit: counts_out[c] (host int64[C]) = the rows whose label is classes[c]; sums_out[c * k + j] (host double[C * k])
 * = the f64 sum of x[i][j] over those rows, reduced in a fixed order without floating-point atomics: the same input gives
 * the same bits on every run, and exact partial sums (integer-valued features below 2^53) give the exact sum.  No sum
 * is a sequential run of more than 256 adds (a tree above that), so |sum - exact| <= 1e-13 * sum.  Every
 * feature must be >= 0.0 (Spark's requireNonnegativeValues: NaN fails it, +inf passes); else the call fails with
 * LO_ERR_INVALID and info->bad_row / bad_col name the lowest such row and its lowest such column.  A label that is none
 * of classes fails the same way with bad_col = k.  classes: nclasses values, strictly ascending, not NaN.
 * Launches: none when n == 0; per window of rows whose CTAs' C x k partials fit 256 MiB, one k_nb_sums (one read of x
 * and y) and the k_nb_reduce levels of its partials (32 to 1 each); then the levels over the windows' sums.  timing:
 * h2d_bytes the classes, d2h_bytes the sums, counts and the error word.
 *
 * lo_nb_predict: the model (pi host double[C], theta host double[C * k], row-major) applied to every row:
 *   raw_c = (sum_j theta[c * k + j] * x_j, from 0.0 in ascending j) + pi[c], every product and add rounded on its own
 *   (F2J dgemv, no FMA); then Spark's raw2probabilityInPlace: m the left-fold max, e_c = exp(raw_c - m), summed in c
 *   order, p_c = e_c / sum; prediction = Vector.argmax(p) (index 0, then a later index only when strictly greater) as
 *   the f64 class INDEX.
 * Transform (confusion_out NULL): prob (LO_F64, n * C elements, row-major) and pred (LO_F64, n) are written, and raw
 * (LO_F64, n * C, or NULL) receives the raw values; y and eval_labels must be NULL.  Evaluate (confusion_out a host
 * int64[neval * C]): nothing per row is written (prob, raw and pred must be NULL); confusion_out[a * C + p] = the rows
 * whose label is eval_labels[a] (neval values, strictly ascending, not NaN) and whose prediction is p.  A label that is
 * none of eval_labels fails with LO_ERR_INVALID, info->bad_row its lowest row, bad_col = k.
 * Launches: none when n == 0; 1 (k_nb_predict).  Bytes: x read once; transform writes n * 8 * (C + 1) (+ n * 8 * C with
 * raw); evaluate reads y once more and writes nothing per row.  timing: h2d_bytes the model (and labels), d2h_bytes the
 * confusion counts and the error word.
 *
 * Refused with LO_ERR_INVALID before anything is enqueued (all three, as they apply): a NULL x, y, classes, model,
 * output or info; x or y not LO_F32 / LO_F64, of different dtypes or on another device; k < 1; ld < k; n < 0; x holding
 * fewer than n * ld elements, y fewer than n; C or neval outside [1, LO_NB_MAX_CLASSES]; C * k > LO_NB_MAX_THETA;
 * classes or eval_labels not strictly ascending or holding NaN; an output table of the wrong dtype, device or size;
 * the transform / evaluate arguments mixed. */
#define LO_NB_MAX_CLASSES 1024
#define LO_NB_MAX_THETA   16384   /* C * k: theta in f64 in 128 KiB of shared memory */
typedef struct lo_nb_info {
    int64_t bad_row;     /* the lowest row holding a refused value, else -1 */
    int32_t bad_col;     /* its lowest refused feature column (k: the label), else -1 */
    int32_t pad;
} lo_nb_info;
int lo_nb_labels(lo_ctx *ctx, const lo_table *y, int64_t n, double *labels_out, int64_t capacity, int64_t *nlabels,
                 lo_host_timing *timing);
int lo_nb_fit(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, const lo_table *y, int64_t n, const double *classes,
              int32_t nclasses, double *sums_out, int64_t *counts_out, lo_nb_info *info, lo_host_timing *timing);
int lo_nb_predict(lo_ctx *ctx, const lo_table *x, int64_t ld, int32_t k, int64_t n, const double *pi, const double *theta,
                  int32_t nclasses, lo_table *prob, lo_table *raw, lo_table *pred, const lo_table *y,
                  const double *eval_labels, int32_t neval, int64_t *confusion_out, lo_nb_info *info,
                  lo_host_timing *timing);

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

/* The two casts of a stored column between resident objects, so that a column already in HBM converts there.
 *
 * lo_parse_text_to_table: lo_parse_number_to_table (same kernel, same summary, same canonical NaN for null and "") with
 * the resident text column `src` as the input: its device chars, offsets and validity are read in place, no cell
 * crosses PCIe (h2d_bytes 0).  Cell i goes to row i of column `col` of `out`.  Refused with LO_ERR_INVALID before
 * anything is launched: a NULL src / out / summary, src made on another context, `out` not LO_F64 or on another
 * device, `col` outside [0, ncols), src->n != out's rows.
 *
 * lo_format_table_to_text: lo_format_number_host of column `col` of the f64 table `in` into a NEW resident text column
 * *out (no nulls: an empty cell is "").  Cell i's status is LO_NUM_EMPTY where `valid` says 0, else LO_NUM_INTEGER
 * where `is_int` says 1, else LO_NUM_FLOAT; each is a lo_validity (mask or Arrow bitmap as for lo_text_upload; NULL:
 * every cell valid / no cell integer), and only its bytes cross PCIe.  lo_format_number_host's rules hold: an is_int
 * cell that is not finite and integral -> LO_ERR_INVALID naming the first such row (nothing is made), a cell takes at
 * most LO_FORMAT_MAX_CELL bytes.  The table must have fewer than 2^31 rows (a text column's limit).
 *
 * lo_text_download: a resident text column back into host Arrow large_string buffers: offsets int64[n + 1] from 0 and
 * the chars (chars_capacity at least the text's bytes, lo_text_info's nbytes; else LO_ERR_INVALID).  The validity is
 * not copied: lo_text_info says how many cells are null. */
int lo_parse_text_to_table(lo_ctx *ctx, const lo_text *src, lo_table *out, int32_t col, lo_parse_summary *summary,
                           lo_host_timing *timing);
int lo_format_table_to_text(lo_ctx *ctx, const lo_table *in, int32_t col, const lo_validity *valid,
                            const lo_validity *is_int, lo_text **out, lo_host_timing *timing);
int lo_text_download(lo_ctx *ctx, const lo_text *t, int64_t *offsets, uint8_t *chars, int64_t chars_capacity,
                     lo_host_timing *timing);

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

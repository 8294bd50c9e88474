/*
 * bydb_gpu.h -- C ABI of libbydbgpu.so: the H100-native (sm_90a) measure scan -> filter -> aggregate path.
 *
 * This is the drop-in boundary a cgo binding in BanyanDB would bind (see INTEGRATION.md).  It
 * replaces, for one query, the reference's HOT LOOPS 1-3 (SURVEY.md section 3.1):
 *
 *   bydb_part_register  <- banyand/measure/part.go:312-375 (mustOpenFilePart) +
 *                          part_iter.go:184-208 (readPrimaryBlock -> blockMetadata cache)
 *   bydb_part_release   <- banyand/measure/part.go:282-299 (partWrapper.decRef -> close)
 *   bydb_scan_agg       <- banyand/measure/query.go:594-639 (searchBlocks) +
 *                          query_batch.go:64-238 (PullBatch / loadCursorsForBatch / mergeBatch) +
 *                          block.go:793-870 (blockCursor.loadData) +
 *                          pkg/query/vectorized/measure/aggregation.go:193-334 (BatchAggregation) +
 *                          pkg/query/vectorized/measure/top.go:145-214 (BatchTop)
 *   bydb_scan_partials / bydb_reduce_finalize
 *                       <- pkg/query/logical/measure/measure_plan_aggregation.go:67-124
 *                          (emitPartial map phase / reduceAccumulator.Combine)
 *
 * Rules: C linkage, plain pointers and sizes; no pointer passed in is retained after the call
 * returns (cgo rule); every function is thread-safe; functions return 0 or a negative errno-style
 * code and never abort; bydb_last_error() returns a thread-local message.  There is NO CPU fallback
 * behind this ABI: pages the device path cannot decode make the call fail with BYDB_ENOTSUP so the
 * caller can route the query to its own CPU path outside this library.
 */
#ifndef BYDB_GPU_H
#define BYDB_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BYDB_OK 0
#define BYDB_ENOENT (-2)    /* unknown part handle / missing file            */
#define BYDB_EIO (-5)       /* CUDA runtime failure                          */
#define BYDB_ENOMEM (-12)   /* HBM budget exceeded / allocation failure      */
#define BYDB_EINVAL (-22)   /* malformed argument or corrupt part            */
#define BYDB_ENOTSUP (-95)  /* encoding not handled on the device path       */

/* value types, pkg/pb/v1/value.go:39-47 */
#define BYDB_VT_STR 1
#define BYDB_VT_INT64 2
#define BYDB_VT_FLOAT64 3
#define BYDB_VT_BINARY 4

/* aggregation functions, api/proto/banyandb/model/v1/common.proto:75-80 */
#define BYDB_AGG_MEAN 1
#define BYDB_AGG_MAX 2
#define BYDB_AGG_MIN 3
#define BYDB_AGG_COUNT 4
#define BYDB_AGG_SUM 5

/* row-predicate operators on a stored tag column */
#define BYDB_OP_EQ 1
#define BYDB_OP_NE 2
#define BYDB_OP_LT 3
#define BYDB_OP_LE 4
#define BYDB_OP_GT 5
#define BYDB_OP_GE 6

typedef struct bydb_ctx bydb_ctx; /* owns one device, its streams and the HBM part cache */
typedef uint64_t bydb_part_h;

typedef struct {
    int32_t device;            /* CUDA device ordinal                                    */
    int32_t warps_per_sm;      /* scan workers per SM; 0 = default (16)                  */
    uint64_t hbm_budget_bytes; /* cap on resident part bytes; 0 = no cap                 */
    uint32_t flags;            /* BYDB_CFG_*                                             */
    uint32_t reserved;
} bydb_cfg;
#define BYDB_CFG_HOST_INDEX 1u /* bydb_part_register: parse the block index (meta.bin / primary.bin / *.tfm) on the host instead of
                                  with the device kernels (the default; both build the same directory -- the host parser is what
                                  the cold host-buffer paths use, where one frame's latency matters more than throughput) */
#define BYDB_CFG_NO_DENSE_PAGES 2u /* bydb_part_register: keep every page as the part stores it.  By default the narrow delta field
                                     pages that the all-rows SUM / COUNT / MEAN scan reads (varints of <= 3 bytes, values spanning
                                     <= 32 bits) also get a bit-plane form in HBM when that form is smaller; results are the same
                                     bit for bit, the scan reads fewer bytes, the part holds more (bydb_part_dense_pages) */

/* One file image of a part (banyand/measure/part.go:40-55).  name is one of "meta.bin",
 * "primary.bin", "timestamps.bin", "fv.bin", "<family>.tf", "<family>.tfm". */
typedef struct {
    const char *name;
    const uint8_t *data;
    uint64_t len;
} bydb_file;

typedef struct {
    uint32_t n_files;
    const bydb_file *files;
} bydb_part_files;

typedef struct {
    const char *family;   /* tag family name                                   */
    const char *tag;      /* tag name                                          */
    int32_t op;           /* BYDB_OP_*                                         */
    int32_t value_type;   /* BYDB_VT_STR / BYDB_VT_BINARY / BYDB_VT_INT64      */
    const uint8_t *lit;   /* literal bytes for STR/BINARY                      */
    uint64_t lit_len;
    int64_t lit_i64;      /* literal for INT64                                 */
} bydb_pred;

typedef struct {
    const char *field; /* field name (model.MeasureAgg input)       */
    int32_t func;      /* BYDB_AGG_*                                */
    int32_t reserved;
} bydb_agg;

/* bydb_query.flags */
#define BYDB_Q_HOST_ZERO_COPY 1u /* bydb_scan_agg_host only: the file images are in pinned, device-mapped host memory,
                                    16-byte aligned, with >= 64 readable bytes after each buffer; the kernels then read
                                    only the pages the query touches, in place over PCIe (no staging copy) */

#define BYDB_Q_ROW_PATH_TYPES 2u /* result typing of the reference's ROW path (a14 / a15): every aggregate, COUNT included, is typed
                                    like its field -- countFunc[N] is N-typed (pkg/query/aggregation/function.go:78-93,
                                    measure_plan_aggregation.go:152-175), so the count over a float64 field comes back as a float64.
                                    Default (flag clear) is the vectorized path's typing: COUNT is int64 (aggregation.go:425-430) */

/* One query = selected series (+ their dense group ids) x parts x predicates x aggregations.
 * Mirrors model.MeasureQueryOptions (pkg/query/model/model.go:75-88) after series resolution:
 * series_ids is what searchSeriesList returned (ascending, query.go:601), series_group is the
 * GroupBy key of each series densified by the caller in first-appearance order (entity / indexed
 * tags live in the series index, not in the part: SURVEY.md F3). */
typedef struct {
    uint32_t n_parts;
    const bydb_part_h *parts;
    uint64_t n_series;
    const uint64_t *series_ids;   /* ascending, unique                                   */
    const int32_t *series_group;  /* [n_series] dense group id; NULL = one group (scalar) */
    int32_t n_groups;             /* ignored when series_group is NULL                    */
    int32_t reserved0;
    int64_t tmin, tmax;           /* inclusive (pkg/timestamp/range.go:143)               */
    uint32_t n_preds;
    const bydb_pred *preds;       /* conjunction                                          */
    uint32_t n_aggs;
    const bydb_agg *aggs;
    int32_t top_n;                /* 0 = no Top                                           */
    int32_t top_agg;              /* index into aggs                                      */
    int32_t top_desc;             /* 1 = largest first                                    */
    uint32_t flags;               /* BYDB_Q_*                                             */
} bydb_query;

typedef struct {
    uint64_t rows_scanned;    /* rows of every selected block (before time trim)            */
    uint64_t rows_matched;    /* rows folded into an aggregate                               */
    uint64_t blocks_scanned;
    uint64_t page_bytes;      /* encoded page bytes the scan kernel consumed                 */
    uint64_t h2d_bytes;       /* host->device bytes moved by this call (a replayed prepared query: 0) */
    uint64_t d2h_bytes;       /* device->host bytes moved by this call                       */
    double scan_kernel_ms;    /* CUDA-event time of the scan kernel on the call's stream     */
    double device_ms;         /* CUDA-event time of all kernels of the call                  */
    uint32_t kernel_launches; /* kernels launched by this call                               */
    uint32_t blocks_slow_lane; /* blocks the fast lane handed to the general decoder          */
    uint32_t slow_lane_reasons; /* OR of: 1 irregular timestamps, 2 int64 tag page, 4<<c field c needs the general decoder */
    uint32_t blocks_express_lane; /* blocks the express lane (all-rows SUM / COUNT / MEAN of plain delta pages) finished */
} bydb_stats;

/* Dense result table; arrays are owned by the library until bydb_result_free.
 * Rows are groups in group-id order (groups that never appeared are omitted), or rank order when
 * top_n > 0.  Column a has type is_float[a]: COUNT is always int64, everything else follows the
 * field type (pkg/query/vectorized/measure/aggregation.go:425-430). */
typedef struct {
    int32_t n_rows;
    int32_t n_aggs;
    const int32_t *group_id;  /* [n_rows]            */
    const int64_t *rows;      /* [n_rows]            */
    const uint8_t *is_float;  /* [n_aggs]            */
    const int64_t *val_i64;   /* [n_rows * n_aggs]   */
    const double *val_f64;    /* [n_rows * n_aggs]   */
    bydb_stats stats;
    void *owner;              /* private             */
} bydb_result;

int bydb_init(const bydb_cfg *cfg, bydb_ctx **out);
void bydb_shutdown(bydb_ctx *ctx);

/* Upload an immutable part into HBM and build its block directory.  Idempotent per part_id.  Unless the context was made with
 * BYDB_CFG_NO_DENSE_PAGES, the part also holds the dense form of its narrow delta field pages: about 2.8 GB more for bench.py's
 * 1e9-datapoint part (21.8 GB of reference pages and directory), charged to the part like everything else it holds. */
int bydb_part_register(bydb_ctx *ctx, uint64_t part_id, const bydb_part_files *files, bydb_part_h *out);
int bydb_part_release(bydb_ctx *ctx, bydb_part_h part);
/* resident bytes / block / row counts of a registered part */
int bydb_part_info(bydb_ctx *ctx, bydb_part_h part, uint64_t *hbm_bytes, uint64_t *n_blocks, uint64_t *n_rows);
/* Fallback pages of a registered part -- EncodeTypePlain numeric pages (null cells, floats that are not short
 * decimals; banyand/measure/column.go:147-153,203-208) and zstd-compressed string blocks (pkg/encoding/bytes.go:
 * 291-304): `unpacked` were rewritten into scan-friendly pages in HBM when the part was registered, `left` could
 * not be (a query that touches one of those returns BYDB_ENOTSUP). */
int bydb_part_fallback_pages(bydb_ctx *ctx, bydb_part_h part, uint64_t *unpacked, uint64_t *left);
/* Dense pages of a registered part (BYDB_CFG_NO_DENSE_PAGES): `pages` field pages got a bit-plane form at registration, held in
 * `bytes` of HBM beside the part's own pages (included in bydb_part_info's hbm_bytes). */
int bydb_part_dense_pages(bydb_ctx *ctx, bydb_part_h part, uint64_t *pages, uint64_t *bytes);
/* Diagnostics: copies the part's DEVICE block directory (the DevBlock[64 B] / DevCol[16 B] records the scan kernels read,
 * csrc/part_dir.hpp) into caller buffers; either pointer may be NULL to only query the counts.  Tests compare the directory the
 * device index kernels build with the host parser's. */
int bydb_part_directory(bydb_ctx *ctx, bydb_part_h part, void *blocks_out, uint64_t blocks_cap_bytes, void *cols_out, uint64_t cols_cap_bytes,
                        uint64_t *n_blocks, uint64_t *n_cols);

/* Scan -> filter -> aggregate over parts already resident in HBM. */
int bydb_scan_agg(bydb_ctx *ctx, const bydb_query *q, bydb_result *out);

/* Group-by on a STORED tag: the key changes from row to row inside a series (a12; the vectorized path's BatchAggregation with
 * a non-entity key column, pkg/query/vectorized/measure/aggregation.go:193-254).  A row belongs to the group
 * (series_group of its series, value of the key tag in that row); groups come back in insertion order -- the scan order is
 * series by series (ascending series id), by time inside a series -- or in rank order when top_n > 0 (ties: the group
 * inserted first, top.go:62-76).  A nil cell and "" are the same key (groupby.go:226-254 encodes a string / bytes key as
 * length + raw bytes).  value_type declares the key tag's type, from the schema the caller holds (as bydb_pred.value_type):
 *   0, BYDB_VT_STR or BYDB_VT_BINARY: a string / binary tag stored with the dictionary encoding (<= 256 distinct values per
 *     block, pkg/encoding/dictionary.go); a block that fell back to the plain bytes block makes the call return
 *     BYDB_ENOTSUP, a value longer than 64 bytes BYDB_ENOTSUP, a tag stored as int64 BYDB_EINVAL.
 *   BYDB_VT_INT64: an int64 tag.  A key value is 8 bytes of little-endian two's complement (the reference's key bytes), so
 *     key_off advances in steps of 8; a nil cell, or a block without the column, is the key 0 (the column's zero value,
 *     typed_column.go:49-53).  A tag stored as a string gives BYDB_EINVAL, a numeric fallback page that admission left
 *     packed BYDB_ENOTSUP.
 *   any other value: BYDB_EINVAL.
 * n_keys counts the distinct values over ALL rows of the selected blocks (series in the query, time span meeting the
 * range), before the time trim and the predicates.  More than max_values of them give BYDB_ENOMEM (the reference's
 * aggregation memory budget).  Device side: one pass collects the distinct values, then ONE SCAN PASS PER VALUE (the key as
 * an extra predicate) fills that value's slice of a composite partial table; stats count every pass.  A group-key query
 * takes at most 7 predicates of its own.  Its prepared form is bydb_query_prepare_keyed (below); not over parts that overlap
 * in time; its map-phase form (the rows a data node answers with) is bydb_scan_partials_keyed, its multi-GPU forms are
 * bydb_scan_reduce_keyed and bydb_scan_reduce_keyed_partials (below). */
typedef struct {
    const char *family;    /* tag family of the key tag                                      */
    const char *tag;       /* tag name                                                       */
    uint32_t max_values;   /* distinct key values accepted over the whole query; 0 = 64, at most 256 */
    uint32_t value_type;   /* 0 / BYDB_VT_STR / BYDB_VT_BINARY (string key) or BYDB_VT_INT64 */
} bydb_group_key;

typedef struct {
    bydb_result base;          /* rows as in bydb_result; base.group_id[r] = series_group of row r       */
    const int32_t *key_id;     /* [base.n_rows] key value of row r: index into the table below           */
    int32_t n_keys;            /* distinct key values found in the selected blocks (some may have no row) */
    int32_t reserved;
    const uint32_t *key_off;   /* [n_keys + 1] value k is key_bytes[key_off[k] .. key_off[k+1])          */
    const uint8_t *key_bytes;
    void *owner;               /* private                                                                 */
} bydb_keyed_result;

int bydb_scan_agg_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_keyed_result *out);
void bydb_keyed_result_free(bydb_ctx *ctx, bydb_keyed_result *r);

/* Write side (SURVEY 8 f4): numeric field pages encoded ON THE DEVICE, byte for byte what banyand/measure/column.go:113-234
 * (encodeInt64Column / encodeFloat64Column -> pkg/encoding/int_list.go:27-53, float.go:30-124) writes into fv.bin for a block:
 * [encode type][decimal exponent, float64 only][first value][zig-zag varint body].  The building block of a device-side merger
 * (decoded blocks in, pages out).  A float64 block that needs the reference's general shortest-digits search, holds NaN / Inf or
 * overflows on the common exponent is not encoded here: needs_cpu[b] = 1 and its page is empty -- the CPU writer (which owns the
 * EncodeTypePlain fallback page) takes it.  Columns with null cells are not accepted (they always take the fallback page). */
typedef struct {
    int32_t value_type;          /* BYDB_VT_INT64 / BYDB_VT_FLOAT64                                  */
    uint32_t n_blocks;
    const uint32_t *block_rows;  /* [n_blocks] rows of each block (>= 1)                              */
    const void *values;          /* HOST memory: int64_t / double values, the blocks back to back     */
} bydb_encode_input;

typedef struct {
    uint32_t n_blocks;
    uint32_t reserved;
    const uint64_t *page_off;    /* [n_blocks + 1] page b = bytes[page_off[b] .. page_off[b+1])       */
    const uint8_t *bytes;
    const uint8_t *needs_cpu;    /* [n_blocks]                                                        */
    uint64_t n_cpu_blocks;
    double device_ms;            /* CUDA-event time of the two kernels (encode + gather)              */
    void *owner;                 /* private                                                           */
} bydb_encoded_pages;

int bydb_encode_pages(bydb_ctx *ctx, const bydb_encode_input *in, bydb_encoded_pages *out);
void bydb_encoded_pages_free(bydb_ctx *ctx, bydb_encoded_pages *r);

/* Same, but the parts come as HOST file images: they are uploaded, scanned and dropped inside the
 * call (the end-to-end path of a cold query).  q->parts / q->n_parts are ignored. */
int bydb_scan_agg_host(bydb_ctx *ctx, uint32_t n_parts, const bydb_part_files *parts, const bydb_query *q, bydb_result *out);

void bydb_result_free(bydb_ctx *ctx, bydb_result *r);

/* Prepared queries.  A query that is executed many times (dashboard refresh, alert rule) is copied and planned once;
 * from its third execution on, the whole step -- block selection, scan, reduce, finalisation, row
 * selection, read-back -- is replayed as ONE captured CUDA graph: one launch and one synchronisation per call instead of
 * ~20 runtime calls.  Every execution still scans the parts (nothing is cached but the launch sequence).  Results and
 * errors are those of bydb_scan_agg; stats.scan_kernel_ms is 0 on replays (per-kernel events do not exist inside a
 * graph), stats.device_ms is the whole graph.  Queries whose parts overlap in time (version dedup needs a host
 * decision) transparently keep the ordinary path.  One execution at a time per prepared query; different prepared
 * queries run concurrently.  The parts named by the query must stay registered while it exists.
 * A replay is nine graph nodes: a reset kernel, block selection, the three scan lanes, the two reduce kernels, finalisation +
 * row selection, and ONE device-to-host copy that carries the result rows and the step's status and counters.  Its stats say so:
 * kernel_launches = the plain call's + 1 (the reset kernel), h2d_bytes = 0 (the series list went up when the step was captured),
 * d2h_bytes = the size of that one copy (the plain call's two copies together).
 * Device memory a captured query keeps until bydb_query_release, or until one of its handles stops naming the part it was
 * captured with (then the next execution captures again); it is not charged to hbm_budget_bytes.  With NS series, G groups,
 * F distinct fields, A aggregations, P parts, NB blocks in those parts and R = min(top_n, G) or G result rows, each term rounded
 * up to 256 B:
 *   the partial table (bydb_partials_layout.total_bytes: 56*G*F + 8*G + 8*F)
 *   + 12*NS + 4*(G+1) + NB*(36 + 32*F) + NS*(32*F + 8) + 4*NS*P (left out above 16 Mi entries)     the scan's lists and partials
 *   + G*(16*A + 9) + 16 + A + R*(12 + 16*A)                                                        finalisation and result rows
 *   + 512                                                                                          the zero page and its read-back image.
 * bench.py's query (NS 10,000, G 1,000, F 1, A 2, P 1, NB 130,000, R 100) keeps 9.5 MB. */
typedef struct bydb_prepared bydb_prepared;
int bydb_query_prepare(bydb_ctx *ctx, const bydb_query *q, bydb_prepared **out);
int bydb_scan_agg_prepared(bydb_ctx *ctx, bydb_prepared *pq, bydb_result *out);
void bydb_query_release(bydb_ctx *ctx, bydb_prepared *pq);

/* Prepared group-by on a stored tag: bydb_scan_agg_keyed for a query executed many times (a dashboard panel grouped by a stored
 * tag).  bydb_query_prepare_keyed checks the arguments as bydb_scan_agg_keyed does (same codes) and copies the query and the key.
 * Every execution returns what bydb_scan_agg_keyed returns for the same arguments at that moment: code and device-error text
 * (the block a max_values error names is the one whose value went over the cap first, which varies between plain calls too),
 * key table, rows, values bit for bit, and the counters (rows_scanned, rows_matched, page_bytes, blocks_scanned, blocks_slow_lane,
 * slow_lane_reasons, blocks_express_lane) summed over the passes.  Free each result with bydb_keyed_result_free.
 * Schedule: the first execution runs the plain keyed path; the second discovers the key values once and captures the step -- the
 * V passes, the insertion order, finalisation and the mapping of rows to (series group, key value) -- as ONE CUDA graph; later
 * executions replay it, with the key table found at the capture.  Discovery is a function of what the handles name, so the graph
 * is dropped, and discovery and the capture run again, when a handle stops naming the part object it was captured with; a handle
 * that names no part any more fails with BYDB_ENOENT.  A query whose discovery fails (above max_values, a plain key page, a
 * 65-byte value, a key of the wrong type), whose parts overlap in time, or whose state cannot be allocated or captured, keeps
 * the plain keyed path for good.  V = 0 (no block selected) needs no graph: no rows, no keys, zero stats.
 * Stats of a replay: h2d_bytes = 0; scan_kernel_ms = 0 and device_ms = the whole graph (as bydb_scan_agg_prepared);
 * kernel_launches = the plain call's (discovery's two kernels give way to the step's reset kernel and the row-mapping kernel);
 * d2h_bytes = the size of its ONE copy: with A aggregations and R = min(top_n, V*G) or V*G result rows, each term rounded up to
 * 256 B,
 *   256 + A + 4*R + 8*R + 8*R*A + 8*R*A      the result rows (the finalisation's read-back over V*G groups)
 *   + 8*R                                   the (series group, key value) of each row
 *   + 256*V                                 each pass's zero page (counters and device error).
 * Device memory a captured keyed query keeps until bydb_query_release_keyed, or until the graph is dropped; it is not charged to
 * hbm_budget_bytes.  With GP = V*G composite groups, F fields, NS series, P parts and NB blocks in them, each term rounded up to
 * 256 B:
 *   2 * (56*GP*F + 8*GP + 8*F)                                                       the composite table and its permuted copy
 *   + 8*V*F + 8*V*NS + 4*V*NS                                                        the passes' column types, Kts, Krow
 *   + 4*NS*V + 4*GP + 4*GP + 16                                                      the insertion order (slots, first series, perm)
 *   + 256 + 12*NS + 4*(G+1) + NB*(40 + 32*F) + NS*(32*F + 8) + 4*NS*P (left out above 16 Mi entries)   one scan scratch, shared by the passes
 *   + GP*(16*A + 9) + 16 + A + R*(12 + 16*A)                                          finalisation over GP groups and the result rows
 *   + 8*R + 256*V                                                                    the row mapping and the passes' zero pages.
 * One execution at a time per handle; different handles, keyed or plain, run concurrently. */
typedef struct bydb_prepared_keyed bydb_prepared_keyed;
int bydb_query_prepare_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_prepared_keyed **out);
int bydb_scan_agg_keyed_prepared(bydb_ctx *ctx, bydb_prepared_keyed *pq, bydb_keyed_result *out);
void bydb_query_release_keyed(bydb_ctx *ctx, bydb_prepared_keyed *pq);

/* ---- multi-GPU map/reduce: per-rank partial tables, one collective, one finalize ----
 * Layout of a partial table for (n_groups G, n_fields F = distinct aggregated fields):
 *   double  sum_f64[G*F]; double max_f64[G*F]; double negmin_f64[G*F];
 *   int64   sum_i64[G*F]; int64 cnt[G*F]; int64 rows[G]; int64 max_i64[G*F]; int64 negmin_i64[G*F];
 * so that ONE all-reduce(SUM) over [sum_f64] + [sum_i64,cnt,rows] and one all-reduce(MAX) over the
 * max/negmin halves combine ranks (min is carried as max of the negation; int64 negation of
 * INT64_MIN is handled by carrying ~x instead of -x).  bydb_partials_layout reports the byte
 * offsets so the caller can issue the collectives on sub-ranges.  A caller that merges tables with its own
 * all-reduce(MAX) over n_max_i64 cannot see a field stored as int64 on one rank and float64 on another;
 * bydb_partials_combine reports that type mix (BYDB_EINVAL at bydb_reduce_finalize / bydb_partials_rows). */
typedef struct {
    uint64_t total_bytes;
    uint64_t off_sum_f64, off_max_f64;   /* [sum_f64] , [max_f64 | negmin_f64]                 */
    uint64_t off_sum_i64, off_max_i64;   /* [sum_i64 | cnt | rows] , [max_i64 | notmin_i64]    */
    uint64_t n_sum_f64, n_max_f64, n_sum_i64, n_max_i64; /* element counts of the four ranges */
} bydb_partials_layout_t;

int bydb_partials_layout(const bydb_query *q, bydb_partials_layout_t *out);
/* Run the scan and leave the partial table in caller-provided DEVICE memory (e.g. a torch tensor),
 * enqueued on `stream` (a cudaStream_t passed as void*; NULL = the CUDA legacy default stream, for this call
 * and for bydb_partials_combine / bydb_reduce_finalize alike, so consecutive calls are always ordered).
 * stats != NULL: the call waits for the scan, fills *stats and reports device-side failures itself.
 * stats == NULL: ASYNCHRONOUS -- the call returns once the work is enqueued, so the collective that ships the
 * table can be enqueued right behind it with no host round trip; a device-side failure (corrupt page, ...) then
 * travels inside the table and is returned by bydb_reduce_finalize on whichever rank finalises. */
int bydb_scan_partials(bydb_ctx *ctx, const bydb_query *q, void *d_partials, uint64_t bytes, void *stream, bydb_stats *stats);
/* Combine n_tables partial tables laid out back to back in DEVICE memory (e.g. the output of ONE all-gather of the
 * per-rank tables) into the first one, in rank order: sums add, max ranges take the maximum.  Deterministic. */
int bydb_partials_combine(bydb_ctx *ctx, const bydb_query *q, void *d_tables, uint32_t n_tables, uint64_t bytes_each, void *stream);
/* Finalize a (reduced) partial table: MEAN finalisation, output typing, Top-N; copies the result to host. */
int bydb_reduce_finalize(bydb_ctx *ctx, const bydb_query *q, const void *d_partials, uint64_t bytes, void *stream, bydb_result *out);

/* Map-phase rows in the reference's wire shape (a18 / f3): what a data node answers when the liaison asks for partials
 * (InternalQueryRequest.agg_return_partial -> mapAccumulator.Result with emitPartial, measure_plan_aggregation.go:67-84;
 * aggregation.PartialToFieldValues, pkg/query/aggregation/aggregation.go:128-145).  One row per group that appeared; aggregate a
 * carries Partial.Value -- SUM: the sum, COUNT: the count, MAX / MIN: the extreme (the N-typed sentinel when no value was
 * folded, aggregation.go:169-191), MEAN: the SUM -- and, for MEAN only, Partial.Count, which the Go side ships as the extra
 * field "__agg_count".  Everything is typed like the FIELD (the row path is N-typed: the count over a float64 field is a
 * float64; function.go:20-236).  The liaison's reduceAccumulator.Combine consumes exactly these pairs. */
typedef struct {
    int32_t n_rows;
    int32_t n_aggs;
    const int32_t *group_id;  /* [n_rows]                                             */
    const uint8_t *is_float;  /* [n_aggs] N of aggregate a = its field's type         */
    const int64_t *val_i64;   /* [n_rows * n_aggs] Partial.Value when !is_float[a]    */
    const double *val_f64;    /* [n_rows * n_aggs] Partial.Value when  is_float[a]    */
    const int64_t *cnt_i64;   /* [n_rows * n_aggs] Partial.Count (MEAN only, else 0)  */
    const double *cnt_f64;
    void *owner;              /* private                                              */
} bydb_partial_rows;
int bydb_partials_rows(bydb_ctx *ctx, const bydb_query *q, const void *d_partials, uint64_t bytes, void *stream, bydb_partial_rows *out);
void bydb_partial_rows_free(bydb_ctx *ctx, bydb_partial_rows *r);

/* Map-phase rows of a group-by on a STORED tag: what a data node answers when the liaison pushes a bydb_scan_agg_keyed query
 * down with agg_return_partial (measure_plan_distributed.go:277; the liaison then drops replicas by (shard, group-by key) and
 * folds the rows with reduceAccumulator.Combine).
 *   - Rows: one per composite group (series group, key value) with rows > 0, in the insertion order bydb_scan_agg_keyed gives
 *     (measure_plan_groupby.go:127-158).  base.group_id[r] is the series group of row r, key_id[r] its key value.
 *   - Values: per aggregate exactly what bydb_partials_rows gives for a plain group -- SUM the sum, COUNT the count, MEAN the sum
 *     with Partial.Count (MEAN only), MAX / MIN the extreme, the N-typed sentinel for a group that met only nulls, 0 for one that
 *     never met the column; everything typed like the field.
 *   - Keys: as in bydb_keyed_result (a string key's bytes, nil -> ""; an int64 key's 8 little-endian bytes, nil -> 0).
 *   - Validation, refusals, caps and device errors: those of bydb_scan_agg_keyed, with the same codes.  top_n / top_agg /
 *     top_desc do not change the rows (as bydb_partials_rows ignores them).
 *   - Stats: every pass counted, as bydb_scan_agg_keyed.  The composite table never crosses PCIe: with cap = max_values (0 -> 64),
 *     V key values found, F distinct aggregated fields and A aggregations,
 *       d2h_bytes = 256 + align256(64 * cap) + align256(4 * cap)   the discovery read-back
 *                 + 256 * V                                       each pass's status / counter page
 *                 + 8 + 8 * F                                     the control word (present rows, column types + status)
 *                 + n_rows * (8 + 16 * A)                         the rows
 *     (V = 0: the first term only).  The root of bydb_scan_reduce_keyed_partials adds the union's read-back, the same size as the
 *     discovery's, and takes no pass term for the union. */
typedef struct {
    bydb_partial_rows base;    /* rows as bydb_partials_rows: base.group_id[r] = series_group of row r, Partial.Value / .Count  */
    const int32_t *key_id;     /* [base.n_rows] index into the key table                                                     */
    int32_t n_keys;            /* as bydb_keyed_result.n_keys                                                                */
    int32_t reserved;
    const uint32_t *key_off;   /* [n_keys + 1]                                                                               */
    const uint8_t *key_bytes;
    bydb_stats stats;          /* every pass counted, as bydb_scan_agg_keyed                                                 */
    void *owner;               /* private                                                                                    */
} bydb_keyed_partial_rows;

int bydb_scan_partials_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_keyed_partial_rows *out);
void bydb_keyed_partial_rows_free(bydb_ctx *ctx, bydb_keyed_partial_rows *r);

/* Group-by on a stored tag in ONE scan pass, for up to 65,536 key values (bydb_scan_agg_keyed runs one pass per value).
 *   - Answer: that of bydb_scan_agg_keyed / bydb_scan_partials_keyed, with the same definitions: a composite group is (series
 *     group, key value); rows are the composite groups with rows > 0 in insertion order (series by series in ascending id, then
 *     by time; a group is inserted at its first row that survives the time range and the predicates); with Top-N, rank order,
 *     ties to the group inserted first.  A nil cell and "" are one string key; for an int64 key a nil cell and a block without
 *     the column are the key 0.  MEAN quirks, output typing, BYDB_Q_ROW_PATH_TYPES, met-column and the empty-fold sentinels as
 *     there.  The partial form follows partial_words' wire rule and ignores top_n.  n_keys counts the distinct values of the
 *     selected blocks before the time trim and the predicates; the key table holds all of them, in no promised order.
 *   - Caps and refusals: max_values 0 means 64, 1..65,536 are accepted, above gives BYDB_EINVAL; more distinct values than
 *     max_values gives BYDB_ENOMEM.  A string key must be a dictionary page (a plain page, or a value longer than 64 bytes:
 *     BYDB_ENOTSUP).  An int64 key takes every page kind bydb_scan_agg_keyed takes; a block whose key column holds more than 256
 *     distinct values gives BYDB_ENOTSUP, the message naming the block.  A key of the wrong type gives BYDB_EINVAL, parts that
 *     overlap in time BYDB_ENOTSUP.  Up to 8 predicates (the key takes no predicate slot); block size and Top-N as bydb_scan_agg.
 *   - Numbers: counts, int64 values and min / max bit-exact; float sums within 1e-9 x (sum of |x| over the group's values) +
 *     1e-9 x |reference| of the reference, and bit-identical from call to call (the records of a group are folded in scan order
 *     by a fixed tree), though not necessarily bit-identical with bydb_scan_agg_keyed, whose passes fold zero partials for the
 *     blocks without the value.  A decimal page's block sum is exact in the integer domain and rounded once, where the reference
 *     adds the page's doubles in row order, so no bound relative to the reference alone holds where values cancel: 0.1, 0.2 and
 *     -0.3 in one block sum to 0 here and to 5.55e-17 there.  bydb_scan_agg_keyed and the express lane of bydb_scan_agg sum
 *     decimal pages the same way and give the same 0.
 *   - Stats (one pass): rows_scanned, blocks_scanned and rows_matched are what bydb_scan_agg reports for the same query without
 *     the key; page_bytes counts every page read once (the key page included).  With cap = max_values, V key values found,
 *     R = sum over the selected blocks of the block's distinct key values, C the composite groups with rows > 0, F distinct
 *     fields, A aggregations, NS series, NB blocks of the parts, pow2(x) the least power of two >= x:
 *       d2h_bytes = 32 + V * (64 + 4) (string key) or 32 + V * 8 (int64 key)    the discovery read-back (V = 0: 32 only)
 *                 + 256 + 8                                                     the scan's status / counter page, C
 *                 + the finalisation read-back of bydb_scan_agg over C groups   (bydb_scan_agg_keyed_wide)
 *                   or 8 + 8 * F + C * (8 + 16 * A)                             (bydb_scan_partials_keyed_wide: control word, rows)
 *                 + 8 * C                                                       each composite group's (series group, key value)
 *     (C = 0: the first two terms only)
 *     and the device scratch of one call is, up to 256-byte alignment of each region,
 *       12 * NS + 12 * S + 68 * cap + 8 * NB   with S = pow2(max(2 * cap, 1024))                            discovery
 *     + 256 + R * (16 + 32 * F) + 12 * pow2(max(2 * R, 1024)) + 8 * R + 12 * pow2(max(R, 2048))              scan and order
 *     + 8 * (C * (7 * F + 1) + F) + 12 * C                                                                    the composite table
 *     + the finalisation's scratch over C groups (or the row image, 8 + 8 * F + C * (8 + 16 * A)).
 *     Nothing of size G * V is allocated. */
int bydb_scan_agg_keyed_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_keyed_result *out);
int bydb_scan_partials_keyed_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_keyed_partial_rows *out);

/* Group-by on a TUPLE of 2..4 stored tags in one scan pass ("latency by endpoint and status code"): the reference's computeKey
 * concatenates one key component per GroupBy tag (aggregation.go:328-337, groupby.go:226-254), so two rows share a group only when
 * every component is equal.  One stored key is bydb_scan_agg_keyed_wide; this is its answer with the key tuple in place of the key.
 *   - Answer: that of bydb_scan_agg_keyed_wide / bydb_scan_partials_keyed_wide word for word, with a composite group = (series
 *     group, key tuple): rows in insertion order or Top-N rank order (ties to the group inserted first), MEAN quirks,
 *     BYDB_Q_ROW_PATH_TYPES, sentinels, the partial form's wire rule, the float bound and call-to-call bit identity as there.  Each
 *     component follows the one-key rules: a string nil is "", an int64 nil or a block without the column is 0.  String and int64
 *     tags mix freely.
 *   - Keys: one table per tag.  Tag t's values are entries key_base[t] .. key_base[t+1]-1 (entry e is key_bytes[key_off[e] ..
 *     key_off[e+1]), a string's bytes or an int64's 8 little-endian bytes), in no promised order; tag t of row r is entry
 *     key_id[r * n_tags + t].  n_tuples counts the distinct tuples over all rows of the selected blocks, before the time trim and
 *     the predicates (some may have no row), and key_base[t+1] - key_base[t] counts tag t's distinct values on the same terms.
 *   - Refusals: n_keys outside 2..4, the same (family, tag) twice, a key whose own max_values is not 0, max_values above 65,536,
 *     or a key failing bydb_scan_agg_keyed_wide's checks: BYDB_EINVAL.  More distinct tuples than max_values (0 = 64): BYDB_ENOMEM,
 *     even when every tag alone is under it.  A block holding more than 256 distinct tuples: BYDB_ENOTSUP, the message naming the
 *     block (the block-local index is one byte).  Per tag the one-key rules and codes hold: a plain string page or a 65-byte value
 *     BYDB_ENOTSUP, a wrong type BYDB_EINVAL, an int64 column with more than 256 values in a block BYDB_ENOTSUP.  Parts that
 *     overlap in time: BYDB_ENOTSUP.  Up to 8 predicates; the keys take no predicate slot.
 *   - Stats (one pass): rows_scanned, rows_matched and blocks_scanned are those of bydb_scan_agg for the same query without keys;
 *     page_bytes counts every page read once (every key page included).  With K tags, V_t tag t's distinct values, T = n_tuples,
 *     R = sum over the selected blocks of the block's distinct tuples, C the composite groups with rows > 0, F fields, A
 *     aggregations, NB blocks of the parts:
 *       kernel_launches = (K + 1) * ((NB > 0) + 1) + 3          discovery: a value kernel and a numbering kernel per table, the scan of R
 *                         (R = 0: that only), then what bydb_scan_agg_keyed_wide launches after its discovery for the same R and C
 *       d2h_bytes = 32 * (K + 1) + sum_t V_t * (64 + 4 for a string tag, 8 for an int64 tag) + 8 * T     the discovery read-back
 *                 + 256 + 8                                                     the scan's status / counter page, C
 *                 + the finalisation read-back of bydb_scan_agg over C groups   (bydb_scan_agg_keys_wide)
 *                   or 8 + 8 * F + C * (8 + 16 * A)                             (bydb_scan_partials_keys_wide: control word, rows)
 *                 + 8 * C                                                       each composite group's (series group, tuple)
 *     (R = 0: the first term only), and the device scratch of one call is, with cap = max_values and S = pow2(max(2 * cap, 1024)),
 *     up to 256-byte alignment of each region,
 *       12 * NS + K * (12 * S + 68 * cap) + 12 * S + 8 * cap + 8 * NB                                     discovery
 *     + then bydb_scan_agg_keyed_wide's scan, order, composite table and finalisation terms for this R and C.
 * Free the answers with bydb_keys_result_free / bydb_keys_partial_rows_free.  The prepared form is bydb_query_prepare_keys_wide,
 * the multi-GPU form bydb_scan_reduce_keys_wide; there is no host-image form. */
typedef struct {
    uint32_t n_keys;              /* 2..4 stored GroupBy tags, in the request's GroupBy order                               */
    uint32_t max_values;          /* distinct key TUPLES accepted over the query; 0 = 64, at most 65,536                    */
    const bydb_group_key *keys;   /* [n_keys] family, tag, value_type as bydb_group_key; each .max_values must be 0         */
} bydb_group_keys;

typedef struct {
    bydb_result base;             /* rows as in bydb_result; base.group_id[r] = series_group of row r                       */
    uint32_t n_tags;              /* = n_keys                                                                                */
    int32_t n_tuples;             /* distinct key tuples in the selected blocks (some may have no row)                      */
    const int32_t *key_id;        /* [base.n_rows * n_tags]: tag t of row r is entry key_id[r * n_tags + t]                 */
    const int32_t *key_base;      /* [n_tags + 1]: tag t's values are entries key_base[t] .. key_base[t+1]-1                */
    const uint32_t *key_off;      /* [key_base[n_tags] + 1]: entry e is key_bytes[key_off[e] .. key_off[e+1])               */
    const uint8_t *key_bytes;
    void *owner;                  /* private                                                                                 */
} bydb_keys_result;

typedef struct {
    bydb_partial_rows base;       /* rows as bydb_partials_rows: base.group_id[r] = series_group of row r                   */
    uint32_t n_tags;              /* as bydb_keys_result                                                                     */
    int32_t n_tuples;
    const int32_t *key_id;
    const int32_t *key_base;
    const uint32_t *key_off;
    const uint8_t *key_bytes;
    bydb_stats stats;             /* as bydb_keys_result.base.stats                                                          */
    void *owner;                  /* private                                                                                 */
} bydb_keys_partial_rows;

int bydb_scan_agg_keys_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_keys *keys, bydb_keys_result *out);
int bydb_scan_partials_keys_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_keys *keys, bydb_keys_partial_rows *out);
void bydb_keys_result_free(bydb_ctx *ctx, bydb_keys_result *r);
void bydb_keys_partial_rows_free(bydb_ctx *ctx, bydb_keys_partial_rows *r);

/* Prepared wide group-by on a stored tag: bydb_scan_agg_keyed_wide for a query executed many times (a dashboard panel grouped by
 * endpoint, instance or status code).  The handle is a bydb_prepared_keyed: bydb_scan_agg_keyed_prepared,
 * bydb_scan_partials_keyed_prepared and bydb_query_release_keyed take it, and on it answer what bydb_scan_agg_keyed_wide /
 * bydb_scan_partials_keyed_wide answer at that moment: code and device-error text, rows in the same order, each row's series group
 * and key bytes, values bit for bit, n_keys, and the counters (rows_scanned, rows_matched, page_bytes, blocks_scanned, ...).
 *   - Arguments: checked at prepare as the wide call checks them, in its order and with its codes (max_values 0 means 64,
 *     1..65,536 accepted, above BYDB_EINVAL; up to 8 predicates, the key takes no slot; the key's type).  A refusal that depends
 *     on the data (above max_values: BYDB_ENOMEM; a block with more than 256 values, a plain string key page or a 65-byte value,
 *     parts that overlap in time: BYDB_ENOTSUP) comes at every execution as the unprepared call gives it, and the handle keeps the
 *     unprepared path for good.
 *   - Schedule: the first execution runs the unprepared wide path; the second runs its discovery, scan and order once to learn
 *     the key table, R and C (functions of the parts the handles name and of the query), captures the step -- a reset kernel,
 *     the scan, the order, the fold into C composite groups, the form's tail and its read-back -- as ONE CUDA graph, and answers
 *     from its first replay; later executions replay it, with the key table found at the capture (the same on every replay).
 *     Part lifecycle, one step per handle of the form last asked for, one execution at a time per handle: as the keyed prepared
 *     forms above.  V = 0 (no block selected) needs no graph: no rows, no keys, zero stats.  C = 0 captures and answers no rows.
 *   - Stats of a replay: h2d_bytes = 0; scan_kernel_ms = 0 and device_ms = the whole graph; with NB blocks in the parts, R
 *     records, C present composite groups, F fields, A aggregations, N = pow2(max(R, 2048)) and align256(x) = x rounded up to 256,
 *       kernel_launches = 1 (reset) + (NB > 0) (scan) + 8 + sum over s = 4096..N (s a power of two) of (log2(s) - 10)  (order)
 *                         + (C > 0) * (1 (fold) + the finalisation's launches over C groups, or 2: rows and copy kernels),
 *         i.e. the unprepared call's with discovery's five launches given way to the reset kernel (partial form: plus the copy
 *         kernel; C = 0: less the fold);
 *       d2h_bytes = finalised: the finalisation's read-back over C groups + 256 + 8*C   (rows, zero page, pairs: ONE copy)
 *                   partial:   align256(8*C) + 256 + (8 + 8*F) + n_rows*(8 + 16*A)   (pairs, zero page, control word, rows)
 *                   C = 0:     256                                                   (the zero page).
 *   - Device memory a captured step keeps until bydb_query_release_keyed, or until the step is dropped; it is not charged to
 *     hbm_budget_bytes.  With cap = max_values, NS series, S = pow2(max(2*cap, 1024)), M = pow2(max(2*R, 1024)), each term
 *     rounded up to 256 B:
 *       12*NS + 12*S + 68*cap + 8*NB + 32 + 4*(NB/1024 + 1)                             discovery's outputs (a copy)
 *       + 56*C*F + 8*C + 8*F + 4*C                                                      the table of C groups, perm
 *       + 256 + 12*M + 8 + R*(16 + 32*F) + 8*R + 12*N + 4*N/1024                        scan and order
 *       + (finalised) the finalisation's scratch over C groups + 256 + 8*C,  or  (partial) 8*C + (8 + 8*F) + C*(8 + 16*A)
 *     (C = 0: no finalisation or row image).  The handle's page-locked staging holds the read-back. */
int bydb_query_prepare_keyed_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_prepared_keyed **out);

/* Prepared group-by on a TUPLE of 2..4 stored tags: bydb_scan_agg_keys_wide for a query executed many times (a dashboard panel or an
 * alert rule grouped by endpoint and status code).  The handle is a bydb_prepared_keyed that bydb_scan_agg_keys_prepared,
 * bydb_scan_partials_keys_prepared and bydb_query_release_keyed take; the one-key executors (bydb_scan_agg_keyed_prepared,
 * bydb_scan_partials_keyed_prepared) refuse it with BYDB_EINVAL, and the tuple executors refuse a one-key handle with BYDB_EINVAL, the
 * message naming the executor to use.  Every execution answers what bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide answer at
 * that moment for the handle's query and keys: code and device-error text, rows in the same order, each row's series group and each
 * tag's key bytes, values bit for bit, n_tuples and each tag's value count (key_base[t+1] - key_base[t]), and the counters
 * (rows_scanned, rows_matched, page_bytes, blocks_scanned).  The key tables found at the capture answer every replay; their order is
 * not part of the contract, as for the unprepared call.
 *   - Arguments: checked at prepare as bydb_scan_agg_keys_wide checks them, in its order and with its codes (n_keys outside 2..4, the
 *     same (family, tag) twice, a key whose own max_values is not 0, max_values above 65,536, each tag's type, up to 8 predicates);
 *     the query and the keys are copied, strings included.  A refusal that depends on the data (more tuples than max_values:
 *     BYDB_ENOMEM; a block holding more than 256 tuples, a plain string page, a 65-byte value, an int64 column with more than 256 values
 *     in a block, parts that overlap in time: BYDB_ENOTSUP) comes at every execution as the unprepared call gives it, and the handle
 *     keeps the unprepared path for good.
 *   - Schedule: the first execution runs the unprepared path; the second runs the discovery, scan and order once with the key list
 *     to learn each tag's table, the tuples' codes, R and C, captures the step -- the reset kernel, the tuple scan, the order, the fold
 *     into C composite groups (series group, tuple), the form's tail and its read-back -- as ONE CUDA graph, and answers from its first
 *     replay; later executions replay it.  T = 0 (no block selected) needs no graph: no rows, no tuples, zero stats.  C = 0 captures
 *     only a copy of the zero page.  Part lifecycle (a handle that stops naming its captured part drops the step and captures again;
 *     one that names no part gives BYDB_ENOENT), one step per handle of the form last asked for, one execution at a time per handle:
 *     as the keyed prepared forms above.
 *   - Stats of a replay: h2d_bytes = 0; scan_kernel_ms = 0 and device_ms = the whole graph; kernel_launches and d2h_bytes as for
 *     bydb_query_prepare_keyed_wide's replay, with C counting (series group, tuple) groups: a replay launches the unprepared call's
 *     kernels, except that discovery's (K + 1) * ((NB > 0) + 1) + 3 launches give way to the reset kernel.
 *   - Device memory a captured step keeps until bydb_query_release_keyed, or until the step is dropped; it is not charged to
 *     hbm_budget_bytes.  With K tags, nt = K + 1 tables, cap = max_values, S = pow2(max(2*cap, 1024)) and NBp = NB rounded up to a
 *     multiple of 1,024 (at least 1,024), each term rounded up to 256 B,
 *       12*NS + nt*12*S + 32*nt + K*68*cap + 8*cap + 4*NBp + 4*NB + 4*NBp/1024                   discovery's outputs (a copy)
 *     then the table of C groups, perm, scan and order and the tail of bydb_query_prepare_keyed_wide's step.  The handle's page-locked
 *     staging holds the read-back. */
int bydb_query_prepare_keys_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_keys *keys, bydb_prepared_keyed **out);
int bydb_scan_agg_keys_prepared(bydb_ctx *ctx, bydb_prepared_keyed *pq, bydb_keys_result *out);
int bydb_scan_partials_keys_prepared(bydb_ctx *ctx, bydb_prepared_keyed *pq, bydb_keys_partial_rows *out);

/* Prepared map-phase answers: what a data node answers, refresh after refresh, for a query the liaison pushes down with
 * agg_return_partial (a dashboard panel or an alert rule in a cluster).  The handles are those of the finalised forms above.
 *   - Answers: every execution returns what the unprepared form returns at that moment, for the handle's query.
 *       bydb_scan_partials_prepared: bydb_scan_partials (with stats) into a table, then bydb_partials_rows over it -- one row per
 *         group with rows > 0 in group-id order, Partial.Value / .Count typed like the field, is_float per aggregate.  The scan's
 *         device error comes first, then the status the table carries.  top_n is ignored, as bydb_partials_rows ignores it.
 *         stats may be NULL; else it gets the counters of bydb_scan_partials, plus the row kernels' launches and read-back.
 *       bydb_scan_partials_keyed_prepared: bydb_scan_partials_keyed -- rows in insertion order, the key table, counters summed
 *         over the passes, the same refusals and codes.  Free the answer with bydb_keyed_partial_rows_free.
 *     A device error's text names the block that met it first (a type mix, the cap), which varies between unprepared calls too.
 *   - Schedule: the first execution runs the unprepared path, the second captures the step as ONE CUDA graph, later ones replay
 *     it.  Parts that overlap in time (plain form; the keyed form answers BYDB_ENOTSUP as bydb_scan_partials_keyed does), a
 *     discovery that fails, state or pinned staging that cannot be had, or a capture that fails keep the unprepared path.  A
 *     handle that stops naming its captured part drops the step and captures again; one that names no part gives BYDB_ENOENT.
 *   - One step per handle: a handle may answer in its finalised and its partial form, but keeps one captured step at a time; an
 *     execution of the other form drops it and captures its own (bydb_scan_reduce_prepared's per-root graphs are apart).
 *   - The graph ends in a kernel that writes the zero pages, the control word and exactly the present rows into the handle's
 *     page-locked staging through its device address: the row count is known only on the device, so no copy node could be sized.
 *   - Stats of a replay: h2d_bytes = 0; scan_kernel_ms = 0 and device_ms = the whole graph; with V key values (V = 1 for the plain
 *     form), F distinct fields, A aggregations and n_rows rows,
 *       d2h_bytes = 256*V + (8 + 8*F) + n_rows*(8 + 16*A)     the zero pages, the control word, the rows -- no padding;
 *       kernel_launches: plain form = bydb_scan_partials' + 4 (the step's reset kernel, and the three kernels of
 *         bydb_partials_rows: compaction, rows, copy), i.e. its own first execution's + 1; keyed form = bydb_scan_partials_keyed's
 *         (discovery's two kernels give way to the step's reset kernel and the copy kernel).
 *   - Device memory a captured step keeps until the handle is released or the step is dropped; it is not charged to
 *     hbm_budget_bytes.  Each term rounded up to 256 B, with the names of bydb_query_prepare / bydb_query_prepare_keyed:
 *       plain:  56*G*F + 8*G + 8*F                                                                  the partial table
 *               + 256 + 12*NS + 4*(G+1) + NB*(36 + 32*F) + NS*(32*F + 8) + 4*NS*P (left out above 16 Mi entries)   the scan
 *               + 4*G + 16 + (8 + 8*F) + G*(8 + 16*A)                                               compaction and the row image
 *       keyed:  56*GP*F + 8*GP + 8*F                                                                the composite table
 *               + 8*V*F + 8*V*NS + 4*V*NS + 4*NS*V + 4*GP + 4*GP + 16                               passes and insertion order
 *               + 256 + 12*NS + 4*(G+1) + NB*(40 + 32*F) + NS*(32*F + 8) + 4*NS*P (as above)        one scan scratch
 *               + 256*V + (8 + 8*F) + GP*(8 + 16*A)                                                 the zero pages and the row image
 *     and the handle's page-locked staging holds the same read-back at its largest (256*V + 8 + 8*F + G*V*(8 + 16*A)). */
int bydb_scan_partials_prepared(bydb_ctx *ctx, bydb_prepared *pq, bydb_partial_rows *out, bydb_stats *stats);
int bydb_scan_partials_keyed_prepared(bydb_ctx *ctx, bydb_prepared_keyed *pq, bydb_keyed_partial_rows *out);

/* ---- multi-GPU reduce behind the C ABI: one process (or thread) per GPU, no torch, no NCCL ----
 * Replaces the liaison gather + reduceAccumulator.Combine (pkg/query/logical/measure/measure_plan_aggregation.go:96-124,
 * measure_plan_distributed.go:254-328) inside one node: every rank owns a MAILBOX in its GPU's memory; in a collective
 * bydb_scan_reduce each rank's reduce kernel writes its partial table straight into its slot of the ROOT's mailbox (peer
 * memory: the stores travel over NVLink / NVSwitch) and raises an arrival flag there; the root waits for the flags on the
 * device, combines the slots in rank order (deterministic float sums) and finalises.  No data-path library collective.
 *
 *   1. every rank:  bydb_comm_export(ctx, max_table_bytes, max_ranks, &h)     -- allocates the mailbox, h is 128 opaque bytes
 *   2. the caller exchanges the handles by any channel it has (gRPC between data nodes, a pipe, torch all_gather in tests)
 *   3. every rank:  bydb_comm_connect(ctx, rank, nranks, handles)             -- opens the peers' mailboxes (CUDA IPC between
 *                   processes, plain peer access between contexts of one process)
 *   4. every rank, in the same order:  bydb_scan_reduce(ctx, &q, root, &out)  -- q names THIS rank's parts and series; group
 *                   layout, aggregations and Top-N must be the same on all ranks.  The root gets the result; the others get
 *                   n_rows = 0 and their own scan statistics.  A rank that fails to arrive makes the root return BYDB_EIO
 *                   after a bounded wait; a device-side scan error of any rank travels in its table and fails the root's call.
 * max_table_bytes: the largest bydb_partials_layout().total_bytes of the queries to come. */
typedef struct { uint8_t bytes[128]; } bydb_comm_handle;
int bydb_comm_export(bydb_ctx *ctx, uint64_t max_table_bytes, int32_t max_ranks, bydb_comm_handle *out);
int bydb_comm_connect(bydb_ctx *ctx, int32_t rank, int32_t nranks, const bydb_comm_handle *all);
int bydb_scan_reduce(bydb_ctx *ctx, const bydb_query *q, int32_t root, bydb_result *out);
/* The same collective for a prepared query (bydb_query_prepare): from its second execution on, per root, the rank's whole step is
 * replayed as ONE captured CUDA graph -- the epoch of the call travels in a small device block that a memcpy node of the graph
 * refreshes.  Ranks may mix bydb_scan_reduce and bydb_scan_reduce_prepared within one collective. */
int bydb_scan_reduce_prepared(bydb_ctx *ctx, bydb_prepared *pq, int32_t root, bydb_result *out);
/* The same collective with every rank's parts given as HOST file images (cold distributed query, end to end): admitted for
 * the duration of the call (with BYDB_Q_HOST_ZERO_COPY only the block directory is uploaded and the scan pulls the pages it
 * touches over PCIe), scanned into the root's mailbox, dropped.  q->parts / q->n_parts are ignored. */
int bydb_scan_reduce_host(bydb_ctx *ctx, uint32_t n_parts, const bydb_part_files *parts, const bydb_query *q, int32_t root, bydb_result *out);

/* Group-by on a stored tag over the same peer mailboxes: the collective form of bydb_scan_agg_keyed.  Every rank runs key
 * discovery and one scan pass per key value over ITS parts, straight into its slot of the root's mailbox; the root builds the
 * union of the ranks' values, combines their composite tables in rank order (deterministic float sums) and finalises once.
 *   - Every rank passes the SAME series_ids, series_group, n_groups, tmin / tmax, predicates, aggregations, Top-N, flags and
 *     *key (max_values included); only `parts` differ -- they are the rank's shard.  A rank that selects no block of a series
 *     contributes nothing to it.  Each rank hashes those fields; a rank whose hash differs from the root's makes the root fail
 *     with BYDB_EINVAL.
 *   - The root's answer is the answer of bydb_scan_agg_keyed over all ranks' parts: rows in insertion order of the whole scan
 *     (or Top-N order, ties to the group inserted first); n_keys counts the distinct values over all ranks' selected blocks, and
 *     more than max_values of them give BYDB_ENOMEM even when every rank alone is under the cap.  The order of the key table
 *     (key_off / key_bytes) is not part of the contract: identify rows by their key bytes.
 *   - Non-root ranks get n_rows = 0, n_keys = 0 and their own scan statistics.
 *   - Within a rank the rules of bydb_scan_agg_keyed hold (its parts must not overlap in time: BYDB_ENOTSUP; same caps, key-type
 *     errors and predicate limit).  Across ranks, one series may live on several ranks only over time spans that do not
 *     intersect -- the span being the series' selected blocks clipped to [tmin, tmax] -- which covers sharding by series range
 *     and by time window; an intersection makes the root fail with BYDB_ENOTSUP naming the series.
 *   - A rank whose slot is too small for its value count fails with BYDB_EINVAL (and so does the root).  Every failure keeps the
 *     ranks' epochs in step: keyed and plain collectives may alternate, with any roots.
 * Size the mailboxes with bydb_keyed_reduce_slot_bytes (host only, like bydb_partials_layout): the slot a rank needs at
 * max_values key values; pass it (or the largest over the queries to come) to bydb_comm_export as max_table_bytes. */
int bydb_keyed_reduce_slot_bytes(const bydb_query *q, const bydb_group_key *key, uint64_t *out);
int bydb_scan_reduce_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, int32_t root, bydb_keyed_result *out);
/* The same collective with the root emitting partial rows (bydb_scan_partials_keyed's contract) instead of finalising: a node
 * of several GPUs answers the liaison's partial request once, for all its GPUs.  Same fingerprint, slot layout, union and span
 * check; bydb_keyed_reduce_slot_bytes sizes it.  The root gets the union's rows in the insertion order of the whole scan;
 * non-root ranks get n_rows = 0, n_keys = 0 and their own stats.  A rank contributes the same bytes under either keyed form, so
 * ranks may mix bydb_scan_reduce_keyed and this call in one collective: the root's call decides what it returns.  Keyed,
 * keyed-partial and plain collectives keep the epochs in step across failures. */
int bydb_scan_reduce_keyed_partials(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, int32_t root, bydb_keyed_partial_rows *out);

/* The collective form of bydb_scan_agg_keyed_wide / bydb_scan_partials_keyed_wide: group-by on a stored tag with up to 65,536 key
 * values across the ranks of the peer mailboxes.  Every rank runs the wide path's discovery, scan and order over ITS parts and
 * writes its present composite groups (series group, key value) -- their table in its insertion order, their first series, its
 * values and the series' spans -- straight into its slot of the root's mailbox.  The root takes the union of the ranks' values,
 * rebuilds the insertion order of the whole scan, folds each composite group's rows in rank order (deterministic float sums) and
 * answers once.
 *   - Every rank passes the SAME series_ids, series_group, n_groups, tmin / tmax, predicates, aggregations, Top-N, flags and
 *     *key (max_values included); only `parts` differ.  The fingerprint also names the form: a rank calling bydb_scan_reduce_keyed
 *     (or its partial form) in the same collective, or passing other arguments, makes the root fail with BYDB_EINVAL.  The two
 *     calls below may be mixed: every rank contributes the same bytes, the root's call decides its answer's form.
 *   - The root's answer is what bydb_scan_agg_keyed_wide (bydb_scan_partials_keyed_wide) answers over all ranks' parts: rows in
 *     the insertion order of the whole scan, or Top-N order with ties to the group inserted first; n_keys = the distinct values
 *     over all ranks' selected blocks; key bytes, nil rules, typing, BYDB_Q_ROW_PATH_TYPES and the sentinels as there.  Counts,
 *     int64 values and min / max are exact, float sums within bydb_scan_agg_keyed_wide's bound (1e-9 x the sum of |x| over the
 *     group's values + 1e-9 x |reference|) and bit-identical from call to call.  The order of
 *     the key table is not part of the contract.  Non-root ranks get n_rows = 0, n_keys = 0 and their own stats.
 *   - Caps and refusals: max_values 0 means 64, 1..65,536 are accepted, above gives BYDB_EINVAL.  More distinct values over all
 *     ranks than max_values gives BYDB_ENOMEM at the root, even when every rank alone is under the cap.  A block with more than
 *     256 values gives BYDB_ENOTSUP naming the block, parts of one rank that overlap in time BYDB_ENOTSUP, and a series whose
 *     clipped spans on two ranks intersect BYDB_ENOTSUP at the root naming the series (the rule of bydb_scan_reduce_keyed).
 *     Up to 8 predicates (the key takes no predicate slot).
 *   - Insertion order: the root sorts each union composite group by its least (series index of its first row, order of that
 *     rank's span within the series, position in that rank's list).  The fields hold series indexes below 2^31, 64 ranks and
 *     lists below 2^27 groups -- a mailbox slot (at most 4 GiB) holds fewer -- and a rank whose list would not fit is refused
 *     with BYDB_EINVAL, as a rank whose slot is too small is.
 *   - Slots: bydb_keyed_wide_reduce_slot_bytes (host only, like bydb_keyed_reduce_slot_bytes) gives the slot a rank needs at
 *     V = max_values key values and max_present present composite groups; pass it (or the largest over the queries to come) to
 *     bydb_comm_export as max_table_bytes.  A rank whose V_r values and C_r present groups do not fit the exported slot fails with
 *     BYDB_EINVAL (and so does the root); every failure keeps the ranks' epochs in step, with any roots and any collectives.
 *   - Stats of every rank, with V_r, R_r, C_r the V, R, C of bydb_scan_agg_keyed_wide over the rank's parts, NB its parts' blocks and
 *     sort(N) = the sum over the powers of two s from 4,096 to N of log2(s) - 10: rows_scanned, rows_matched, blocks_scanned and
 *     page_bytes are those of its one wide pass;
 *       d2h_bytes = 32 + V_r * (64 + 4) (string key) or 32 + V_r * 8 (int64 key), + 256 + 8 when V_r > 0
 *       kernel_launches = (NB > 0) + 4, and when V_r > 0: + (NB > 0) + 10 + sort(pow2(max(R_r, 2048))) + (C_r > 0)
 *     A rank's values, spans and table travel to the root's mailbox device to device (the header and values from the host) and
 *     are not counted.  The root adds, with V_u, C_u the union's values and composite groups, R ranks, sum V and sum C over the ranks:
 *       d2h_bytes += 16 * R, and when sum V > 0: + 16 + V_u * (64 + 4), and when C_u > 0: + the finalisation read-back of
 *                    bydb_scan_agg over C_u groups (or 8 + 8 * F + C_u * (8 + 16 * A) for the partial form) + 8 * C_u
 *       kernel_launches += when sum V > 0: 6 + (NS > 0 and R > 1) + (sum C > 0), and when C_u > 0: + 8 +
 *                    sort(pow2(max(sum C, 2048))) + the finalisation's kernels (or 1 for the partial form)
 *       h2d_bytes += 8 * (R + 1) when sum V > 0
 *     The root's merge takes, up to 256-byte alignment of each region, with pow2(x) the least power of two >= x,
 *       32 + 8 * (R + 1) + 8 * pow2(max(2 * sum V, 1024)) + 8 * sum V + 68 * cap + 28 * pow2(max(2 * sum C, 1024)) + 20 * sum C
 *       + 8 * pow2(max(sum C, 2048)) (+ the exclusive scans' tile sums)                                  the union and the order
 *       + 8 * (C_u * (7 * F + 1) + F) + 12 * C_u                                                         the folded table
 *       + the finalisation's scratch over C_u groups (or the row image, 8 + 8 * F + C_u * (8 + 16 * A))
 *     of device scratch, and a rank 4 * (NB + C_r) beside its wide pass.  The root's page-locked staging is sized before the
 *     collective for the most composite groups the slots can carry. */
int bydb_keyed_wide_reduce_slot_bytes(const bydb_query *q, const bydb_group_key *key, uint64_t max_present, uint64_t *out);
int bydb_scan_reduce_keyed_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, int32_t root, bydb_keyed_result *out);
int bydb_scan_reduce_keyed_wide_partials(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, int32_t root,
                                         bydb_keyed_partial_rows *out);

/* The collective form of bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide: group-by on a tuple of 2..4 stored tags across the
 * ranks of the peer mailboxes ("latency by endpoint and status code" over a node whose GPUs shard its parts).  Every rank runs
 * bydb_scan_agg_keys_wide's discovery, scan and order over ITS parts and writes its present composite groups (series group, tuple)
 * -- their table in its insertion order, their first series, the series' spans, each tag's values and its tuples' codes in its own
 * tag ids -- straight into its slot of the root's mailbox.  The root takes the union of each tag's values, then of the tuples,
 * rebuilds the insertion order of the whole scan, folds each composite group's rows in rank order (deterministic float sums) and
 * answers once.
 *   - Every rank passes the SAME series_ids, series_group, n_groups, tmin / tmax, predicates, aggregations, Top-N, flags and *keys
 *     (every key's family, tag and value type in GroupBy order, and max_values); only `parts` differ.  The fingerprint covers them
 *     and names the tuple form: a rank passing other keys, the same keys in another order, or calling bydb_scan_reduce_keyed_wide in
 *     the same collective makes the root fail with BYDB_EINVAL.  The two calls below may be mixed: every rank contributes the same
 *     bytes, the root's call decides its answer's form.
 *   - The root's answer is what bydb_scan_agg_keys_wide (bydb_scan_partials_keys_wide) answers over all ranks' parts: rows in the
 *     insertion order of the whole scan, or Top-N order with ties to the group inserted first; n_tuples = the distinct tuples over
 *     all ranks' selected blocks, key_base[t+1] - key_base[t] = tag t's distinct values over all ranks; the per-component nil
 *     rules, typing, BYDB_Q_ROW_PATH_TYPES, the sentinels and the partial form's wire rule as there.  Counts, int64 values and
 *     min / max are exact, float sums within bydb_scan_agg_keyed_wide's bound and bit-identical from call to call.  The order inside
 *     each tag's table and the numbering of the tuples are not part of the contract: identify rows by their key bytes.  Non-root
 *     ranks get n_rows = 0, n_tuples = 0 (and n_tags = 0) and their own stats.
 *   - Caps and refusals: every argument refusal of bydb_scan_agg_keys_wide, with the same codes.  More distinct tuples over all
 *     ranks than max_values (0 = 64) gives BYDB_ENOMEM at the root, even when every rank alone is under the cap; so does a tag with
 *     more distinct values over all ranks than max_values, which is refused before any tuple is recoded (a union tag id must fit
 *     16 bits).  The per-block and per-tag BYDB_ENOTSUP rules hold on the rank where the block lives; parts of one rank that
 *     overlap in time give BYDB_ENOTSUP; a series whose clipped spans on two ranks intersect gives BYDB_ENOTSUP at the root, naming
 *     the series.  Insertion order and its limits as in bydb_scan_reduce_keyed_wide.
 *   - Slots: bydb_keys_wide_reduce_slot_bytes (host only) gives the slot a rank needs at T = V_t = max_values (every tag's values
 *     and the tuples at the cap) and max_present present composite groups; pass it (or the largest over the queries to come) to
 *     bydb_comm_export as max_table_bytes.  A rank whose values, tuples and present groups do not fit the exported slot fails with
 *     BYDB_EINVAL, and so does the root.  Every failure keeps the ranks' epochs in step: plain, keyed, wide and tuple collectives may
 *     follow, with any roots.
 *   - Stats of every rank, with K tags, V_t,r, T_r, R_r, C_r the V_t, T, R, C of bydb_scan_agg_keys_wide over the rank's parts, NB its
 *     parts' blocks and sort(N) as for bydb_scan_reduce_keyed_wide: rows_scanned, rows_matched, blocks_scanned and page_bytes are
 *     those of its one wide pass;
 *       d2h_bytes = 32 * (K + 1) + sum_t V_t,r * (64 + 4 for a string tag, 8 for an int64 tag) + 8 * T_r, + 256 + 8 when T_r > 0
 *       kernel_launches = (K + 1) * ((NB > 0) + 1) + 3, and when T_r > 0: + (NB > 0) + 10 + sort(pow2(max(R_r, 2048))) + (C_r > 0)
 *     A rank's tables, spans, values and codes travel to the root's mailbox device to device (the head, values and codes from the
 *     host) and are not counted.  The root adds, with V_u,t, T_u, C_u the union's tag-t values, tuples and composite groups, R ranks,
 *     sum T and sum C over the ranks:
 *       d2h_bytes += 36 * R, and when sum T > 0: + 48 + 48 + sum_t V_u,t * (64 + 4) + 8 * T_u, and when C_u > 0: + the
 *                    finalisation read-back of bydb_scan_agg over C_u groups (or 8 + 8 * F + C_u * (8 + 16 * A) for the partial
 *                    form) + 8 * C_u
 *       kernel_launches += when sum T > 0: 6 * K + (NS > 0 and R > 1) + 6 + (sum C > 0), and when C_u > 0: + 8 +
 *                    sort(pow2(max(sum C, 2048))) + the finalisation's kernels (or 1 for the partial form)
 *       h2d_bytes += 4 * (K + 2) * (R + 1) when sum T > 0
 *     (a refusal at the root stops these sums where it is found).  The root's merge takes, up to 256-byte alignment of each region,
 *     with pow2(x) the least power of two >= x and sum V_t the ranks' tag-t values summed,
 *       64 + 4 * (K + 2) * (R + 1) + sum_t (8 * pow2(max(2 * sum V_t, 1024)) + 4 * sum V_t + 68 * cap) + 8 * pow2(max(2 * sum T, 1024))
 *       + 4 * sum T + 4 * max(max_t sum V_t, sum T) + 8 * cap + 28 * pow2(max(2 * sum C, 1024)) + 20 * sum C
 *       + 8 * pow2(max(sum C, 2048)) (+ the exclusive scans' tile sums)                                    the unions and the order
 *       + 8 * (C_u * (7 * F + 1) + F) + 12 * C_u                                                           the folded table
 *       + the finalisation's scratch over C_u groups (or the row image, 8 + 8 * F + C_u * (8 + 16 * A))
 *     of device scratch, and a rank 4 * (NB + C_r) beside its wide pass.  The root's page-locked staging is sized before the
 *     collective for the unions' read-back and the most composite groups the slots can carry. */
int bydb_keys_wide_reduce_slot_bytes(const bydb_query *q, const bydb_group_keys *keys, uint64_t max_present, uint64_t *out);
int bydb_scan_reduce_keys_wide(bydb_ctx *ctx, const bydb_query *q, const bydb_group_keys *keys, int32_t root, bydb_keys_result *out);
int bydb_scan_reduce_keys_wide_partials(bydb_ctx *ctx, const bydb_query *q, const bydb_group_keys *keys, int32_t root,
                                        bydb_keys_partial_rows *out);

const char *bydb_last_error(void);
const char *bydb_version(void);

#ifdef __cplusplus
}
#endif
#endif

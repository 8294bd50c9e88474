/*
 * bydb_oracle.h -- CPU ORACLE for the BanyanDB measure-query hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a plain-C restatement of the reference's
 * Go algorithm (apache/skywalking-banyandb, commit 0dd5d684).  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (libbydbgpu.so) never links, loads or
 * calls anything in oracle/.
 *
 * Parity pinning: the Go reference cannot be built here (no Go toolchain, no
 * vendored modules), so the oracle is pinned against every known-answer vector
 * the reference's own tests hold for this path (tests/test_oracle_golden.py
 * transcribes them; see SURVEY.md section 8c), against the expected rows of its
 * end-to-end measure cases (tests/golden/e2e_cases.json, generated from
 * test/cases/measure/data), against the merge / block-selection fixtures of
 * banyand/measure/{query,part_iter}_test.go, and cross-checked by a randomised
 * brute-force model and a second, independent part writer -- it is NOT pinned
 * against outputs of the running reference.  zstd frames (third-party
 * github.com/klauspost/compress v1.18.5, go.mod:171) are "parity unpinned" at
 * the compressed-byte level and pinned at the decompressed level by RFC 8878
 * conformance (system libzstd 1.5.5 via dlopen).
 *
 * Every function cites the reference file:line it follows.
 */
#ifndef BYDB_ORACLE_H
#define BYDB_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- encode types: pkg/encoding/encoding.go:85-99 ---- */
enum {
    OB_ENC_UNKNOWN = 0,
    OB_ENC_CONST = 1,
    OB_ENC_DELTA_CONST = 2,
    OB_ENC_DELTA = 3,
    OB_ENC_DELTA_OF_DELTA = 4,
    OB_ENC_CONST_V = 5,
    OB_ENC_DELTA_CONST_V = 6,
    OB_ENC_DELTA_V = 7,
    OB_ENC_DELTA_OF_DELTA_V = 8,
    OB_ENC_PLAIN = 9,
    OB_ENC_DICTIONARY = 10
};

/* ---- value types: pkg/pb/v1/value.go:39-47 ---- */
enum {
    OB_VT_UNKNOWN = 0,
    OB_VT_STR = 1,
    OB_VT_INT64 = 2,
    OB_VT_FLOAT64 = 3,
    OB_VT_BINARY = 4
};

/* ---- aggregation functions: api/proto/banyandb/model/v1/common.proto:75-80 ---- */
enum { OB_AGG_MEAN = 1, OB_AGG_MAX = 2, OB_AGG_MIN = 3, OB_AGG_COUNT = 4, OB_AGG_SUM = 5 };

/* predicate ops (row filter on a stored tag column) */
enum { OB_OP_EQ = 1, OB_OP_NE = 2, OB_OP_LT = 3, OB_OP_LE = 4, OB_OP_GT = 5, OB_OP_GE = 6 };

/* growable byte buffer */
typedef struct {
    uint8_t *p;
    size_t len, cap;
} ob_buf;
void ob_buf_free(ob_buf *b);
void ob_buf_reset(ob_buf *b);
void ob_buf_append(ob_buf *b, const void *src, size_t n);
void ob_buf_put(ob_buf *b, uint8_t c);

/* a possibly-nil byte string (len < 0 means nil, pkg/encoding/bytes.go:49-56) */
typedef struct {
    const uint8_t *p;
    int64_t len;
} ob_bytes;

/* ---- pkg/encoding/int.go ---- */
void ob_varint64_append(ob_buf *dst, int64_t v);                       /* int.go:75-99  */
void ob_varuint64_append(ob_buf *dst, uint64_t u);                      /* int.go:152-185 */
/* returns bytes consumed, 0 on error */
size_t ob_varuint64_read(const uint8_t *src, size_t n, uint64_t *out);  /* int.go:189-211 */
/* decodes exactly cnt varints; returns bytes consumed or (size_t)-1 on error */
size_t ob_varint64_list_read(const uint8_t *src, size_t n, int64_t *dst, size_t cnt); /* int.go:111-148 */

/* ---- pkg/encoding/int_list.go, delta.go ---- */
/* appends body to dst; returns encode type, *first = firstValue */
int ob_int64_list_encode(ob_buf *dst, const int64_t *a, size_t n, int64_t *first);  /* int_list.go:27-53 */
/* returns 0 ok, <0 error */
int ob_int64_list_decode(int64_t *dst, const uint8_t *src, size_t srclen, int enc, int64_t first, size_t count); /* int_list.go:57-101 */

/* ---- pkg/convert/number.go ---- */
void ob_conv_int64_to_bytes(int64_t v, uint8_t out[8]);   /* number.go:33-45 */
int64_t ob_conv_bytes_to_int64(const uint8_t b[8]);       /* number.go:93-106 */

/* ---- pkg/encoding/float.go ---- */
/* returns 0 ok, -1 cannot encode losslessly */
int ob_float64_to_decimal_list(int64_t *dst, const double *src, size_t n, int16_t *exp); /* float.go:30-66 */
void ob_decimal_list_to_float64(double *dst, const int64_t *vals, size_t n, int16_t exp); /* float.go:69-93 */
int ob_float_to_decimal(double f, int64_t *mant, int16_t *exp);                          /* float.go:107-190 */
double ob_pow10(int n);
extern int ob_force_slow_float;                                                          /* tests only */                                                                   /* Go math.Pow10 */

/* ---- pkg/encoding/bytes.go, dictionary.go, writer.go, reader.go ---- */
void ob_bytes_block_encode(ob_buf *dst, const ob_bytes *a, size_t n);    /* bytes.go:45-72 */
/* decodes n items; out[i].p points into *arena (caller frees arena); returns consumed bytes or -1 */
int64_t ob_bytes_block_decode(ob_bytes *out, size_t n, const uint8_t *src, size_t srclen, ob_buf *arena, int allow_tail);
/* dictionary: returns 0 if >256 distinct (caller must use plain) else 1; appends page body (without type byte) */
int ob_dictionary_encode(ob_buf *dst, const ob_bytes *a, size_t n);      /* dictionary.go:52-88 */
int ob_dictionary_decode(ob_bytes *out, size_t n, const uint8_t *src, size_t srclen, ob_buf *arena); /* dictionary.go:90-114 */
void ob_bitpack_encode(ob_buf *dst, const uint32_t *src, size_t n);      /* dictionary.go:199-219, writer.go */
/* bit writer exposed for golden test (writer_test.go:27-56) */
typedef struct { ob_buf *out; uint8_t cache, available; } ob_bitw;
void ob_bitw_init(ob_bitw *w, ob_buf *out);
void ob_bitw_bool(ob_bitw *w, int b);
void ob_bitw_bits(ob_bitw *w, uint64_t u, int nbits);
void ob_bitw_byte(ob_bitw *w, uint8_t b);
void ob_bitw_flush(ob_bitw *w);
int ob_bit_reader_script(const uint8_t *data, size_t n, const int *ops, size_t n_ops, uint64_t *out); /* reader.go test hook */

/* ---- zstd (pkg/compress/zstd/zstd.go:49-57) via dlopen(libzstd.so.1) ---- */
int ob_zstd_compress(ob_buf *dst, const void *src, size_t n, int level);
int ob_zstd_decompress(ob_buf *dst, const void *src, size_t n);

/* ---- banyand/measure/column.go: numeric / default column pages ---- */
/* cells: for INT64/FLOAT64 value types each non-nil cell is 8 bytes (order-preserving int64 / BE IEEE bits) */
void ob_column_encode(ob_buf *dst, int value_type, const ob_bytes *cells, size_t n);          /* column.go:113-234 */
/* decode to cells (8-byte cells for numeric pages); arena owns memory */
int ob_column_decode(ob_bytes *out, size_t n, int value_type, const uint8_t *src, size_t srclen, ob_buf *arena); /* column.go:276-379 */

/* ===================== part building (banyand/measure/part.go:162-233, block_writer.go) ===================== */
typedef struct ob_builder ob_builder;
typedef struct ob_part ob_part;

typedef struct {
    const char *name;
    int value_type;          /* OB_VT_* */
    const int64_t *i64;      /* value_type INT64 */
    const double *f64;       /* value_type FLOAT64 */
    const ob_bytes *bytes;   /* STR / BINARY (len<0 = nil) */
    const uint8_t *nulls;    /* optional, 1 = null cell (numeric types) */
} ob_column;

typedef struct {
    const char *name;
    int n_cols;
    const ob_column *cols;
} ob_family;

ob_builder *ob_builder_new(void);
void ob_builder_free(ob_builder *b);
/* append n rows (any order; builder sorts by (sid, ts, -version) and dedups like part.go:170-190).
 * All calls must use the same schema. Returns 0 ok. */
int ob_builder_append(ob_builder *b, size_t n, const uint64_t *sids, const int64_t *ts, const int64_t *versions,
                      int n_fields, const ob_column *fields, int n_fams, const ob_family *fams);
/* builds the in-memory part (mustInitFromDataPoints + Flush). */
ob_part *ob_builder_finish(ob_builder *b);
/* one part from n builders with their own schemas and disjoint series: each builder's blocks are cut as
 * ob_builder_finish cuts them, then written in series order, each with its builder's tag families and fields.
 * NULL (ob_last_error) when two builders share a series. */
ob_part *ob_builder_finish_many(ob_builder *const *bs, int n_builders);

/* open a part from raw file images (part.go:312-375). names: "meta.bin","primary.bin","timestamps.bin","fv.bin","<fam>.tf","<fam>.tfm" */
ob_part *ob_part_open(int n_files, const char *const *names, const uint8_t *const *data, const size_t *lens);
void ob_part_free(ob_part *p);
int ob_part_n_files(const ob_part *p);
const char *ob_part_file_name(const ob_part *p, int i);
const uint8_t *ob_part_file_data(const ob_part *p, int i, size_t *len);
/* part metadata (part_metadata.go:32-40) */
void ob_part_meta(const ob_part *p, uint64_t *total_count, uint64_t *blocks_count, int64_t *min_ts, int64_t *max_ts,
                  uint64_t *uncompressed, uint64_t *compressed);

/* ===================== query (banyand/measure/query.go, pkg/query/aggregation, vectorized/measure) ===================== */
typedef struct {
    const char *family;      /* tag family */
    const char *tag;         /* tag name */
    int op;                  /* OB_OP_* */
    int value_type;          /* OB_VT_STR / OB_VT_INT64 */
    ob_bytes str;            /* literal for STR/BINARY */
    int64_t i64;             /* literal for INT64 */
} ob_pred;

typedef struct {
    const char *field;
    int func;                /* OB_AGG_* */
} ob_agg;

/* one component of a group key: a stored tag and its declared type (OB_VT_STR / OB_VT_BINARY or OB_VT_INT64); a block whose
 * column has another type makes the query fail */
enum { OB_MAX_GROUP_KEYS = 4 };
typedef struct {
    const char *family;
    const char *tag;
    int value_type;
} ob_group_key;

typedef struct {
    int n_parts;
    ob_part *const *parts;
    size_t n_series;
    const uint64_t *sids;        /* ascending (query.go:601) */
    const int32_t *groups;       /* dense group id per series; NULL = single group 0 */
    int32_t n_groups;
    int64_t tmin, tmax;          /* inclusive (timestamp/range.go:143) */
    int n_preds;
    const ob_pred *preds;
    int n_aggs;
    const ob_agg *aggs;
    int top_n;                   /* 0 = none */
    int top_agg;                 /* index into aggs */
    int top_desc;                /* 1 = largest first */
    int threads;                 /* decode threads (goroutine-per-block analogue, query_batch.go:195); <=1 serial */
    int per_thread_partials;     /* 0 = reference-shaped (single-thread merge+agg), 1 = best-effort all-core */
    /* per-row group key: a tuple of 1..OB_MAX_GROUP_KEYS stored tags in GroupBy order (n_keys = 0: none).  A row's group is
     * (group of its series, encoded key); groups are emitted in insertion order (pkg/query/vectorized/measure/aggregation.go:
     * 193-254).  The key is encoded as computeKey encodes it (aggregation.go:328-337, appendKeyComponent groupby.go:217-254):
     * an int64 component as 8 little-endian bytes (a nil cell or a block without the column: 0), a string / binary component
     * as a 4-byte little-endian length and the bytes (nil: "").  Runs the serial fold. */
    int n_keys;
    const ob_group_key *keys;
} ob_query;

typedef struct {
    int32_t n_rows;              /* groups emitted (group id order; only groups that appeared) */
    int32_t n_aggs;
    int32_t *group_id;           /* [n_rows] */
    int64_t *rows;               /* [n_rows] rows folded into the group */
    uint8_t *is_float;           /* [n_aggs] output type per agg (aggregation.go:425-430) */
    int64_t *val_i64;            /* [n_rows*n_aggs] */
    double *val_f64;             /* [n_rows*n_aggs] */
    uint64_t rows_scanned;       /* rows decoded from selected blocks (before time trim) */
    uint64_t rows_matched;       /* rows folded */
    uint64_t blocks_scanned;
    /* only with a group key: group_id[r] is then the SERIES group of row r, key[r * n_keys + k] its k-th component -- a
     * string's bytes, or an int64's 8 little-endian bytes */
    int32_t n_keys;
    ob_bytes *key;               /* [n_rows * n_keys] owned */
} ob_result;

int ob_query_run(const ob_query *q, ob_result *out);
void ob_result_free(ob_result *r);
const char *ob_last_error(void);

/* raw scan helper for tests: decode every selected row (after merge+dedup+filter) into flat arrays.
 * Caller frees with ob_rows_free. fields are returned as double (float fields) or int64 (int fields). */
typedef struct {
    size_t n;
    uint64_t *sid;
    int64_t *ts;
    int64_t *version;
    int n_fields;
    uint8_t *is_float;  /* [n_fields] */
    int64_t **i64;      /* [n_fields][n] */
    double **f64;       /* [n_fields][n] */
    uint8_t **null;     /* [n_fields][n] */
} ob_rows;
int ob_scan_rows(const ob_query *q, ob_rows *out);
void ob_rows_free(ob_rows *r);

#ifdef __cplusplus
}
#endif
#endif

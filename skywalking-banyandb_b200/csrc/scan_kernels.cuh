// scan_kernels.cuh -- device-side types shared between the kernels (scan_kernels.cu) and the host
// orchestration (capi.cu).  See DESIGN.md for the HBM layout and the roofline of each kernel.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/bydb_gpu.h"
#include "dense_page.cuh"
#include "part_dir.hpp"

namespace bydb {

constexpr int kWarpsPerCta = 8;          // 256 threads; every warp is an independent block worker
#ifndef BYDB_STAGE_BYTES
#define BYDB_STAGE_BYTES 2048            // experiment knobs (make variant EXTRA="-DBYDB_STAGE_BYTES=4096 -DBYDB_STAGES=3")
#endif
#ifndef BYDB_STAGES
#define BYDB_STAGES 2
#endif
#ifndef BYDB_EXPRESS_STAGES
#define BYDB_EXPRESS_STAGES 2            // the express lane's own ring depth (its stages are 4 KB decode units)
#endif
#ifndef BYDB_EXPRESS_CTAS
#define BYDB_EXPRESS_CTAS 2              // resident CTAs per SM the express lane is compiled for: 127 registers, no spills (DESIGN.md 4.2)
#endif
#ifndef BYDB_EXPRESS_DECODE
#define BYDB_EXPRESS_DECODE 1            // 0: the express lane streams its pages and skips the decode (fetch timing only: WRONG sums)
#endif
#ifndef BYDB_FAST_CTAS
#define BYDB_FAST_CTAS 3                 // resident CTAs per SM the fast lane is compiled for (register cap 65536 / (256 x n))
#endif
constexpr int kStageBytes = BYDB_STAGE_BYTES;  // one TMA bulk copy (cp.async.bulk) per stage
constexpr int kStages = BYDB_STAGES;           // per-warp ring: decode stage k while stage k+1 lands
constexpr int kChunkBytes = 512;         // 32 lanes x 16 B per decode iteration
constexpr int kMaskWords = 264;          // row bitmask: 8448 rows (memPart blocks hold <= 8193 rows)
constexpr int kMaxFcols = 8;             // distinct aggregated fields per query
constexpr int kMaxPreds = 8;             // conjunctive row predicates per query
constexpr int kMaxLit = 64;              // inline literal bytes of a string predicate
constexpr int kMaxParts = 64;            // parts per query

// device error codes written to ScanParams::err[0] (first error wins); err[1] = global block index
enum DevErr : uint32_t {
    kErrNone = 0,
    kErrPlainPage = 1,      // numeric fallback page (EncodeTypePlain, column.go:147-153): needs zstd on device
    kErrZstdDict = 2,       // dictionary whose value block is zstd-compressed (>=128 B, bytes.go:291-304)
    kErrBigBlock = 3,       // predicate on a block with more rows than the smem row mask holds
    kErrCorrupt = 4,        // varint stream does not decode to `count` values / bad header
    kErrTypeMix = 5,        // one field name with int64 and float64 pages in the same query
    kErrBadEnc = 6,         // unknown encode type byte
    kErrTagPlain = 7,       // high-cardinality (>256 values) string tag page: plain bytes block
    kErrOverlap = 8,        // same series in several parts with overlapping time spans: needs version dedup
    kErrPredType = 9,       // predicate literal type does not match the stored tag column type
    kErrTmaTimeout = 10,    // a bulk copy never completed (internal error)
    kErrPeerTimeout = 11,   // multi-GPU reduce: a peer rank never delivered its partial table / never freed the slot
    kErrKeyCap = 12,        // per-row group key: more distinct values than the caller's max_values
    kErrKeyLong = 13,       // per-row group key: a value longer than kMaxLit bytes
    kErrRankOverlap = 14,   // keyed collective: one series on two ranks over time spans that intersect
    kErrKeyBlock = 15,      // wide group key: a block whose key column holds more than kMaxBlockKeys distinct values
    kErrTupleBlock = 16,    // tuple group key: a block holding more than kMaxBlockKeys distinct key tuples
};
constexpr int kOpEqOrNil = 7;  // internal predicate operator of the group-key passes: the cell is nil or equals the literal
constexpr uint32_t kKeyAbsent = 0xffffffffu;  // Krow of a series that never shows the value (a block's first row is below it)

struct DevPartRef {
    const DevBlock *blocks;
    const DevCol *cols;
    const uint8_t *const *files;  // device array of file base pointers (indexed by DevCol::file_id)
    const DevDense *dense;        // dense forms of the pages, parallel to cols (NULL: the part has none)
    uint32_t n_blocks;
    uint32_t block_base;          // global index of blocks[0] in this query
};

struct DevPred {
    int64_t lit_i64;
    uint32_t lit_len;
    uint16_t name_id;
    uint8_t op;
    uint8_t value_type;
    uint8_t lit[kMaxLit];
};

// per (block, field) partial aggregate; `i` views are used for int64 fields, `f` for float64 fields
struct BlockPartial {
    union { double f; int64_t i; } sum, mn, mx;
    int64_t cnt;
};
static_assert(sizeof(BlockPartial) == 32, "BlockPartial layout");

// Whether a group met the column.  The reference creates a group's aggregation slot at its first kept row from a block that
// has the column, null cell or not (aggregation.go:290-312): a group that never met the column keeps the zero value for MIN /
// MAX, one that met only null cells the empty-fold sentinels.  A BlockPartial without values (cnt == 0) holds that bit in
// mn.i (1 = met).  In the partial table a group without values holds it in the maximum word of the other type, which its
// column never uses: 0 = met, the empty maximum (INT64_MIN / -inf) = not met; both combine across tables by maximum.
__host__ __device__ __forceinline__ bool met_column(bool is_float, int64_t cnt, int64_t max_i64, double max_f64) {
    return cnt > 0 || (is_float ? max_i64 == 0 : max_f64 == 0.0);
}

struct ScanParams {
    DevPartRef parts[kMaxParts];  // kernel parameters stay within 4 KB: see the static_asserts below
    uint32_t n_parts;
    uint32_t total_blocks;
    const uint64_t *q_sids;       // ascending
    uint32_t n_series;
    uint32_t n_fcols;
    uint32_t n_preds;
    uint32_t pad0;
    int64_t tmin, tmax;
    uint16_t fcol_name[kMaxFcols];
    uint8_t fcol_need[kMaxFcols]; // bit0: sum wanted (SUM/MEAN), bit1: min/max wanted; 0 = COUNT only
    DevPred preds[kMaxPreds];
    uint32_t *worklist;           // [total_blocks] global block indices selected by plan_blocks
    uint32_t *work_count;
    uint32_t *work_next;
    uint32_t *rest_list;          // [total_blocks] express lane only (else NULL): blocks it left to the regular fast lane
    uint32_t *rest_count;
    uint32_t *rest_next;
    uint32_t *slow_list;          // [total_blocks] blocks the fast lane deferred to the general decoder
    uint32_t *slow_count;
    uint32_t *slow_next;
    int32_t *block_qsid;          // [total_blocks] query-series index or -1
    uint32_t *first_block;        // [n_parts * n_series] first block of the series in the part (0xffffffff = none); may be NULL
    BlockPartial *P;              // [total_blocks * n_fcols]
    uint32_t *Prows;              // [total_blocks] rows that passed range + predicates
    uint32_t *Pfirst;             // [total_blocks] first surviving row of the block (group-key passes only, else NULL)
    int32_t *col_type;            // [n_fcols] 0 unknown / BYDB_VT_INT64 / BYDB_VT_FLOAT64
    uint32_t *err;                // [2]
    unsigned long long *stats;    // [0] rows_scanned [1] rows_matched [2] page_bytes [3] blocks [4] slow-lane blocks [5] slow-lane reasons
    // ---- version dedup across overlapping parts (query.go:995-1004); all NULL when no parts overlap
    int32_t *dd_index;            // [total_blocks] compact index of a block that needs dedup, or -1
    unsigned long long *dd_row_off; // [total_blocks] offset of the block's rows in dd_ts / dd_ver
    uint32_t *dd_list;            // [n_dd_blocks] global block indices
    unsigned long long *dd_counts; // [0] flagged blocks, [1] flagged rows
    int64_t *dd_ts, *dd_ver;      // decoded timestamps / versions of the flagged blocks
    uint32_t *dd_shadow;          // [n_dd_blocks * kMaskWords] 1 = row survives the dedup
    uint32_t n_dd_blocks;
    uint32_t pad1;
};

static_assert(sizeof(ScanParams) + 256 <= 4096, "ScanParams (with WideScanParams beside it) must fit the 4 KB kernel-parameter space");

struct ReduceParams {
    DevPartRef parts[kMaxParts];
    uint32_t n_parts;
    uint32_t n_series;
    uint32_t n_fcols;
    int32_t n_groups;
    const uint64_t *q_sids;
    const int32_t *order;         // [n_series] query-series indices sorted by (group, series)
    const int32_t *group_start;   // [n_groups + 1] into order
    const int32_t *block_qsid;
    const uint32_t *first_block;  // see ScanParams
    const BlockPartial *P;
    const uint32_t *Prows;
    const int32_t *col_type;
    BlockPartial *S;              // [n_series * n_fcols] per-series partials
    int64_t *Srows;               // [n_series]
    uint32_t *err;
    uint32_t dedup_done;          // 1 = overlapping parts were resolved by the dedup kernels
    uint32_t pad2;
    // group-key passes only (else NULL): where the series first shows the pass's key value -- (ts_min of the earliest block
    // with a surviving row, that row's index); INT64_MAX = the series never shows it
    const uint32_t *Pfirst;
    int64_t *Kts;                 // [n_series]
    uint32_t *Krow;               // [n_series]
    // keyed collective, first pass only (else NULL): [lo, hi] of each series' selected blocks over every part; lo > hi = none
    int64_t *span;                // [2 * n_series]
    // partial table (see bydb_gpu.h): written by group_reduce
    double *sum_f64, *max_f64, *negmin_f64;
    int64_t *sum_i64, *cnt, *rows, *max_i64, *notmin_i64, *coltype;
};

struct FinalizeParams {
    int32_t n_groups;
    uint32_t n_fcols;
    uint32_t n_aggs;
    uint32_t row_path_types;      // 1 = COUNT is typed like its field (the row path's N-typed countFunc) instead of int64
    int32_t agg_fcol[32];
    int32_t agg_func[32];
    const double *sum_f64, *max_f64, *negmin_f64;
    const int64_t *sum_i64, *cnt, *rows, *max_i64, *notmin_i64, *coltype;
    int64_t *out_i64;             // [n_groups * n_aggs]
    double *out_f64;              // [n_groups * n_aggs]
    uint8_t *out_is_float;        // [n_aggs]
    uint32_t *err_out;            // DevErr carried in the table's coltype words (0 = none); may be NULL
};

// output row selection on the device: stable compaction of the groups that appeared, or Top-N
constexpr int kMaxDeviceTopN = 2048;
struct SelectParams {
    int32_t n_groups;
    uint32_t n_fcols, n_aggs;
    int32_t top_n, top_agg, top_desc, top_fcol;
    const int64_t *rows, *cnt;
    const int64_t *max_i64;       // the table's maxima: with cnt, whether a group met the column (met_column)
    const double *max_f64;
    const int64_t *coltype;       // the table's column types: met_column reads the word of the FIELD's type, whatever the output type
    const int64_t *val_i64;       // finalized values [n_groups * n_aggs]
    const double *val_f64;
    const uint8_t *is_float;      // [n_aggs]
    uint64_t *keys;               // scratch [n_groups]
    uint8_t *kstate;              // scratch [n_groups]
    int32_t *sel_group;           // outputs, capacity = top_n > 0 ? min(top_n, n_groups) : n_groups
    int64_t *sel_rows;
    int64_t *sel_i64;
    double *sel_f64;
    uint32_t *sel_count;
    const uint32_t *zero_src;     // optional: the step's zero page (64 words), copied to zero_dst so that it travels in the result's
    uint32_t *zero_dst;           // read-back; the kernel runs behind everything that writes the page.  NULL: no copy
};
void launch_select_rows(const SelectParams &p, cudaStream_t s);

// ---- per-row group key (a stored dictionary tag): see "Group key" in scan_kernels.cu
constexpr uint32_t kKeySlots = 1024;   // open-addressing table of the distinct key values (at most 256 are accepted)
constexpr uint32_t kMaxKeyValues = 256;
struct KeyParams {
    DevPartRef parts[kMaxParts];
    uint32_t n_parts, total_blocks;
    const uint64_t *q_sids;
    uint32_t n_series;
    uint32_t cap;                 // distinct values the caller accepts
    int64_t tmin, tmax;
    uint16_t key_name;
    uint16_t pad[3];
    unsigned long long *slots;    // [kKeySlots] 0 = empty, else bit63 | len << 48 | device address of the bytes;
                                  // int64 key: 0 = empty, else the value itself
    uint32_t *count;              // distinct values found
    uint32_t *err;                // [2]
    uint32_t *zero;               // int64 key: 1 = the value 0 occurs (it cannot take a slot)
    uint8_t *vals;                // [cap * kMaxLit] packed by key_pack (int64 key: [cap] values, 8 little-endian bytes each)
    uint32_t *lens;               // [cap]
};
static_assert(sizeof(ReduceParams) <= 4096 && sizeof(KeyParams) + 64 <= 4096, "kernel-parameter space");
// int64_key: the key tag is an int64 column (key_values_i64_kernel), else a dictionary string tag (key_values_kernel)
void launch_key_values(const KeyParams &p, bool int64_key, int grid, cudaStream_t s);

struct KeyOrderParams {
    int32_t n_groups;             // G: groups of series
    uint32_t n_values;            // V
    uint32_t n_series;
    uint32_t pad;
    const int32_t *order, *group_start;
    const int64_t *Kts;           // [V * n_series]
    const uint32_t *Krow;         // [V * n_series]
    int32_t *slot;                // [n_series * V] preset to -1: composite group whose first row is (series, rank)
    int32_t *first_series;        // [V * G] -1 = the composite group never appeared
    int32_t *perm;                // [V * G] composite groups in insertion order, then the ones that never appeared
    uint32_t *n_present;
};
void launch_key_order(const KeyOrderParams &p, cudaStream_t s);
struct TablePtrs {
    double *sum_f64, *max_f64, *negmin_f64;
    int64_t *sum_i64, *cnt, *rows, *max_i64, *notmin_i64, *coltype;
};
// partial-table layout for (G groups, F fields); see bydb_gpu.h
struct TableLayout {
    size_t G, F, GF;
    size_t off_sum_f64, off_max_f64, off_negmin_f64, off_sum_i64, off_cnt, off_rows, off_max_i64, off_notmin_i64, off_coltype, total;
    TableLayout(size_t g, size_t f) : G(g), F(f), GF(g * f) {
        size_t o = 0;
        off_sum_f64 = o; o += GF * 8;
        off_max_f64 = o; o += GF * 8;
        off_negmin_f64 = o; o += GF * 8;
        off_sum_i64 = o; o += GF * 8;
        off_cnt = o; o += GF * 8;
        off_rows = o; o += G * 8;
        off_max_i64 = o; o += GF * 8;
        off_notmin_i64 = o; o += GF * 8;
        off_coltype = o; o += F * 8;
        total = o;
    }
    // the regions of the table at `base`, each from group row g0 on (the coltype words belong to no row)
    TablePtrs at(uint8_t *base, size_t g0 = 0) const {
        const size_t gf = g0 * F;
        return TablePtrs{reinterpret_cast<double *>(base + off_sum_f64) + gf, reinterpret_cast<double *>(base + off_max_f64) + gf,
                         reinterpret_cast<double *>(base + off_negmin_f64) + gf, reinterpret_cast<int64_t *>(base + off_sum_i64) + gf,
                         reinterpret_cast<int64_t *>(base + off_cnt) + gf, reinterpret_cast<int64_t *>(base + off_rows) + g0,
                         reinterpret_cast<int64_t *>(base + off_max_i64) + gf, reinterpret_cast<int64_t *>(base + off_notmin_i64) + gf,
                         reinterpret_cast<int64_t *>(base + off_coltype)};
    }
};

// ---- one-pass group key (bydb_scan_agg_keyed_wide): see "Wide group key" in scan_kernels.cu
constexpr uint32_t kMaxWideKeyValues = 65536;
constexpr uint32_t kMaxBlockKeys = 256;  // distinct key values of one block (a block-local index is one byte)
// the value table of a wide key: slots as KeyParams::slots, slot_mask + 1 of them (a power of two, at least twice the cap)
struct WideKeyParams {
    KeyParams k;                  // k.vals / k.lens: [cap] packed by key_pack_wide_kernel in id order
    uint32_t slot_mask;
    uint32_t int64_key;
    uint32_t *slot_id;            // [slot_mask + 1] id of the value in an occupied slot (int64 key: the value 0, if it occurs, is id 0)
    uint32_t *n_by_rank;          // [total_blocks] distinct values of the selected block of that scan-order rank, else 0
    uint32_t *rank;               // [total_blocks] scan-order rank of a selected block: (series, time) over every part
};
// discovery (one warp per selected block) and the numbering of the values; *k.count = distinct values
void launch_key_values_wide(const WideKeyParams &p, int grid, cudaStream_t s);
// exclusive prefix sum of v[0, n) in place (n a multiple of 1024), tile_sums [n / 1024], *total = the sum
void launch_excl_scan(uint32_t *v, uint32_t n, uint32_t *tile_sums, uint32_t *total, cudaStream_t s);
// A record per (selected block, block-local key value that a surviving row shows), in scan order: the blocks by rank, a block's
// records by their first surviving row.  [u32 value id | u32 first row | u32 rows | i32 series group] then F BlockPartial.
__host__ __device__ __forceinline__ size_t wide_record_bytes(size_t F) { return 16 + sizeof(BlockPartial) * F; }
struct WideScanParams {
    const unsigned long long *slots;
    const uint32_t *slot_id;
    const uint32_t *zero;         // int64 key: the value 0 occurs (id 0)
    uint32_t slot_mask, int64_key;
    uint16_t key_name;
    uint16_t pad[3];
    const uint32_t *rank;         // WideKeyParams::rank
    const uint32_t *rec_off;      // [total_blocks] first record of the block of that rank (exclusive scan of n_by_rank)
    const int32_t *series_group;  // [n_series]
    uint8_t *records;             // [R * wide_record_bytes(F)]
};
// ScanParams supplies the parts, the selection, the predicates, the fields, the column types, err and stats (the plain scan's
// counters: rows_scanned, rows_matched, page_bytes, blocks)
void launch_scan_keyed_wide(const ScanParams &p, const WideScanParams &w, int grid, cudaStream_t s);
int scan_keyed_wide_ctas_per_sm();

// ---- tuple group key (bydb_scan_agg_keys_wide): 2..kMaxKeyTags stored tags.  Every tag has a value table of its own (discovered by
// launch_key_values_wide); a tuple is coded id_0 | id_1 << 16 | id_2 << 32 | id_3 << 48 from its values' ids and enters a table of
// its own as an int64 key does (the all-zero code takes the zero flag).  A record's value id is then the tuple's id.
constexpr uint32_t kMaxKeyTags = 4;
struct WideTag {                  // a tag's value table, as WideScanParams names it
    const unsigned long long *slots;
    const uint32_t *slot_id;
    uint32_t slot_mask;
    uint16_t key_name;
    uint8_t int64_key, pad;
};
struct WideTagSet {
    WideTag tag[kMaxKeyTags];
    uint32_t n_tags, pad;
};
// discovery of the tuples (one warp per selected block) and their numbering: w.k is the tuple table (int64 mode), w.rank /
// w.n_by_rank as for one key, n_by_rank counting the block's distinct tuples
void launch_key_tuples_wide(const WideKeyParams &w, const WideTagSet &tags, int grid, cudaStream_t s);
// the scan with a tuple key: the WideScanParams name the tuple table (int64 mode)
struct WideTupleParams : WideScanParams {
    WideTagSet tags;
};
static_assert(sizeof(ScanParams) + sizeof(WideTupleParams) <= 4096 && sizeof(WideKeyParams) + sizeof(WideTagSet) <= 4096, "kernel-parameter space");
void launch_scan_keys_wide(const ScanParams &p, const WideTupleParams &w, int grid, cudaStream_t s);
int scan_keys_wide_ctas_per_sm();
// the records folded into a partial table of the present composite groups (series group, value id) in insertion order
struct WideReduceParams {
    const uint8_t *records;
    uint32_t n_records, n_fcols;  // R, F
    unsigned long long *comp;     // [comp_mask + 1] composite (series group << 32 | value id) + 1, 0 = empty
    uint32_t *comp_min;           // [comp_mask + 1] lowest record of the composite, preset 0xffffffff
    uint32_t *rec_slot;           // [R] composite slot of a record with rows > 0, else 0xffffffff
    uint32_t comp_mask;
    uint32_t n_sort;              // power of two >= max(R, 2048)
    unsigned long long *keys;     // [n_sort] min record of the composite << 32 | record; ~0 = no rows
    uint32_t *heads;              // [n_sort] 1 = first record of a composite, then (exclusive scan) the composite's index
    uint32_t *tile_sums;          // [n_sort / 1024 + 1]
    uint32_t *ctl;                // [0] records with rows [1] composite groups N_c
    uint32_t *seg_start;          // [R] first sorted record of composite j
    const int32_t *col_type;      // [F] the scan's column types
    const uint32_t *scan_err;     // the scan's DevErr (carried in the table's coltype words)
    TablePtrs table;              // TableLayout(N_c, F)
    int32_t *pairs;               // [2 N_c] series group, value id of composite j
    int32_t *perm;                // [N_c] j (the identity order keyed_partial_rows_kernel reads)
};
// composite slots, sort keys, the sort, the heads and their scan: ctl[1] = N_c afterwards
void launch_wide_order(const WideReduceParams &p, cudaStream_t s);
// the fold into p.table / pairs / perm (p.table sized for ctl[1] groups)
void launch_wide_fold(const WideReduceParams &p, uint32_t n_comp, cudaStream_t s);

// The Partial a data node ships for aggregate `func` of one group of a partial table, word o = group * F + field (emitPartial,
// measure_plan_aggregation.go:67-84; aggregation.PartialToFieldValues): SUM the sum, COUNT the count, MEAN the sum with the count as
// Partial.Count, MAX / MIN the extreme -- the N-typed sentinel for a group that met only nulls, the zero value for one that never
// met the column (met_column).  Both words are typed like the field: the bits of a double when is_float.  The one definition of
// the wire rule: bydb_partials_rows (host) and keyed_partial_rows_kernel (device) both call it.
struct PartialWords {
    uint64_t val, cnt;
};
__host__ __device__ __forceinline__ uint64_t f64_bits(double x) {
#ifdef __CUDA_ARCH__
    return static_cast<uint64_t>(__double_as_longlong(x));
#else
    uint64_t u;
    __builtin_memcpy(&u, &x, 8);
    return u;
#endif
}
__host__ __device__ __forceinline__ PartialWords partial_words(const TablePtrs &t, size_t o, int func, bool is_float) {
    const int64_t n = t.cnt[o];
    const bool met = met_column(is_float, n, t.max_i64[o], t.max_f64[o]);  // else MIN / MAX keep the zero value
    int64_t vi = 0, ci = 0;
    double vf = 0.0, cf = 0.0;
    switch (func) {
        case BYDB_AGG_SUM: vi = t.sum_i64[o]; vf = t.sum_f64[o]; break;
        case BYDB_AGG_COUNT: vi = n; vf = static_cast<double>(n); break;
        case BYDB_AGG_MAX:
            vi = n > 0 ? t.max_i64[o] : met ? INT64_MIN : 0;
            vf = n > 0 ? t.max_f64[o] : met ? -1.7976931348623157e308 : 0.0;
            break;
        case BYDB_AGG_MIN:
            vi = n > 0 ? ~t.notmin_i64[o] : met ? INT64_MAX : 0;
            vf = n > 0 ? -t.negmin_f64[o] : met ? 1.7976931348623157e308 : 0.0;
            break;
        case BYDB_AGG_MEAN: vi = t.sum_i64[o]; vf = t.sum_f64[o]; ci = n; cf = static_cast<double>(n); break;
    }
    return is_float ? PartialWords{f64_bits(vf), f64_bits(cf)} : PartialWords{static_cast<uint64_t>(vi), static_cast<uint64_t>(ci)};
}

// ---- map-phase rows of a keyed query (bydb_scan_partials_keyed): row j < *n_present is composite group perm[j] = v * G + g of the
// UNPERMUTED V x G table, written as [group_id i32 | key_id i32 | val[A] | cnt[A]] (keyed_row_bytes(A) bytes, partial_words).
// The control word in front of the rows: u32 n_present | u32 0 | i64 coltype[F] (the passes' column types merged + status).
__host__ __device__ __forceinline__ size_t keyed_row_bytes(size_t A) { return 8 + 16 * A; }
__host__ __device__ __forceinline__ size_t keyed_ctl_bytes(size_t F) { return 8 + 8 * F; }
struct KeyedRowsParams {
    TablePtrs table;              // composite table TableLayout(V * G, F), as the passes (or the union of the ranks) left it
    const int32_t *perm;          // key_perm_kernel's insertion order
    const uint32_t *n_present;
    const int64_t *pass_coltype;  // [n_passes * n_fcols]
    uint32_t n_groups, n_fcols, n_aggs, n_passes;
    int32_t agg_fcol[32];
    int32_t agg_func[32];
    uint32_t *ctl;                // control word (keyed_ctl_bytes)
    uint8_t *rows;                // [max_rows * keyed_row_bytes(n_aggs)]
};
// grid over max_rows (= V * G) rows; the threads of rows at or above *n_present leave at once
void launch_keyed_partial_rows(const KeyedRowsParams &p, size_t max_rows, cudaStream_t s);
// ---- map-phase rows of a plain table (bydb_partials_rows and the prepared partial forms) run keyed_partial_rows_kernel with one
// pass over the table itself; in front of it, one CTA compacts the groups with rows[g] > 0 in group-id order (stable): perm[j] is
// the j-th present group, *n_present their number -- the shape key_perm_kernel gives (the absent groups are not listed).
void launch_present_groups(const int64_t *rows, uint32_t n_groups, int32_t *perm, uint32_t *n_present, cudaStream_t s);
// The rows of a map-phase answer to page-locked host memory, from inside a graph (a copy node cannot take its size from the
// device): `dst` is the DEVICE address of the staging (cudaHostGetDevicePointer), 16-byte aligned, and receives the page_bytes of
// `pages` (the passes' zero pages, a multiple of 16), then the control word and exactly min(n_present, max_rows) rows of `image`
// (n_present = its first word).  16-byte loads and stores; the rows end on an 8-byte word when ctl_bytes + n * row_bytes is
// not a multiple of 16, and that word goes with one 8-byte store.  Nothing beyond those bytes is written.
struct RowsCopyParams {
    const uint8_t *pages;         // 256-byte aligned
    const uint8_t *image;         // 256-byte aligned: control word (keyed_ctl_bytes), then the rows (keyed_row_bytes each)
    uint8_t *dst;
    size_t page_bytes, ctl_bytes, row_bytes;
    uint32_t max_rows, pad;
};
void launch_rows_to_host(const RowsCopyParams &p, cudaStream_t s);
// ---- the head of a rank's slot in the root's mailbox, in both keyed collectives (KeyedSlot, WideSlot), for V key values.  Every
// region starts on a 256-byte boundary; the root derives a rank's layout from the V_r (and C_r) in its header.
//   header    Header, in 256 bytes
//   lens      [V] u32, values [V][kMaxLit] (an int64 key's 8 little-endian bytes, length 8)
struct SlotHead {
    struct Header {
        uint64_t fp;  // the query's fingerprint
        uint32_t V, C;  // V_r; C_r (WideSlot) or 0 (KeyedSlot)
    };
    size_t off_lens, off_vals, end;  // end: where the slot's own regions begin
    __host__ __device__ static size_t up(size_t o) { return (o + 255) / 256 * 256; }
    __host__ __device__ explicit SlotHead(size_t V) : off_lens(256), off_vals(up(256 + V * 4)), end(up(off_vals + V * kMaxLit)) {}
};
// ---- keyed collective (bydb_scan_reduce_keyed): the slot of a rank that found V key values, for G groups, F fields and NS
// series.  Every region is sized by V, so a rank's need grows with the values it found.
//   head      SlotHead(V)
//   coltype   [V * F] the passes' column types + status
//   Kts, Krow [V * NS] where each series first shows each value (ReduceParams::Kts / Krow)
//   span      [NS][2] the series' selected blocks (ReduceParams::span)
//   table     the composite table TableLayout(V * G, F)
struct KeyedSlot : SlotHead {
    size_t off_coltype, off_kts, off_krow, off_span, off_table, total;
    __host__ __device__ KeyedSlot(size_t G, size_t F, size_t NS, size_t V) : SlotHead(V) {
        off_coltype = end;
        off_kts = up(off_coltype + V * F * 8);
        off_krow = up(off_kts + V * NS * 8);
        off_span = up(off_krow + V * NS * 4);
        off_table = up(off_span + NS * 16);
        total = off_table + 8 * (V * G * (7 * F + 1) + F);  // TableLayout(V * G, F).total
    }
};
struct KeyedUnionParams {
    const uint8_t *slots;         // rank r's slot at slots + r * slot_stride (the root's mailbox, this collective's parity)
    size_t slot_stride;
    uint32_t G, F, NS, cap;       // groups, fields, series, distinct key values accepted
    uint32_t n_ranks, n_values;   // n_values: V_u, the union's size (combine / merge_first only)
    int64_t tmin, tmax;           // the query's range (span check)
    uint8_t *vals;                // [cap * kMaxLit] union values, in order of first appearance by rank, then by the rank's order
    uint32_t *lens;               // [cap]
    int32_t *inv;                 // [n_ranks * cap] inv[r * cap + u]: index of union value u among rank r's values, -1 = absent
    uint32_t *ctl;                // [0] V_u [1] DevErr [2] first series whose spans on two ranks intersect (preset 0xffffffff)
    uint64_t *table;              // union composite table TableLayout(V_u * G, F)
    int64_t *coltype;             // [V_u * F] column types of the union values (permute_table's pass_coltype)
    int64_t *Kts;                 // [V_u * NS]
    uint32_t *Krow;               // [V_u * NS]
};
// key_union_kernel, then rank_span_check_kernel (both read only the headers and spans; ctl is then read back)
void launch_key_union(const KeyedUnionParams &p, cudaStream_t s);
// combine_keyed_kernel and merge_first_kernel into table / coltype / Kts / Krow (p.n_values = V_u > 0)
void launch_combine_keyed(const KeyedUnionParams &p, cudaStream_t s);
// ---- wide keyed collective (bydb_scan_reduce_keyed_wide): the slot of a rank that found V key values and C present composite
// groups, for F fields and NS series.
//   head      SlotHead(V)
//   span      [NS][2] i64 the series' selected blocks (as ReduceParams::span)
//   pairs     [C][2] i32 (series group, value id) of composite j, in the rank's insertion order (wide_fold_kernel)
//   first     [C] u32 the series index of composite j's first row
//   table     the rank's composite table TableLayout(C, F) in its insertion order (wide_fold_kernel)
struct WideSlot : SlotHead {
    size_t off_span, off_pairs, off_first, off_table, total;
    __host__ __device__ WideSlot(size_t F, size_t NS, size_t V, size_t C) : SlotHead(V) {
        off_span = end;
        off_pairs = up(off_span + NS * 16);
        off_first = up(off_pairs + C * 8);
        off_table = up(off_first + C * 4);
        total = off_table + 8 * (C * (7 * F + 1) + F);  // TableLayout(C, F).total
    }
    // what one more composite group adds to the slot (pairs, first, table row), before the regions' rounding
    static size_t comp_bytes(size_t F) { return 8 + 4 + 8 * (7 * F + 1); }
};
// A rank's first appearances: ranks whose records the scan wrote (WideKeyParams::rank, WideScanParams::rec_off) back to series.
//   wide_series_kernel: thread i < NS writes span[i] (the series' selected blocks over every part); thread g < total_blocks writes
//     the series index of a selected block at its scan-order rank, rank_series[rank[g]]
//   wide_first_kernel: composite j < n_comp (its lowest record keys[seg_start[j]]) -> the block holding that record (the last rank
//     whose rec_off does not exceed it) -> first[j] = that block's series index
struct WideFirstParams {
    const uint32_t *rank;             // WideKeyParams::rank
    uint32_t *rank_series;            // [total_blocks]
    int64_t *span;                    // [2 * NS]
    const unsigned long long *keys;   // WideReduceParams::keys, sorted
    const uint32_t *seg_start;        // WideReduceParams::seg_start
    const uint32_t *rec_off;          // WideScanParams::rec_off
    uint32_t n_blocks, n_comp;
    uint32_t *first;                  // [n_comp]
};
static_assert(sizeof(KeyParams) + sizeof(WideFirstParams) <= 4096, "kernel-parameter space");
void launch_wide_series(const KeyParams &k, const WideFirstParams &p, cudaStream_t s);
void launch_wide_first(const WideFirstParams &p, cudaStream_t s);
// The root of the wide collective.  Flat indices: rank r's value v is v_off[r] + v, its composite row j is row_off[r] + j.
//   1. the union of the values (launch_wide_union): every (r, v) enters a table homed by key_home over its bytes; the slot keeps the
//      least (r, v) with those bytes; the least ones are numbered by an exclusive scan in (r, v) order -- ranks in rank order, each
//      rank's values in its order -- and write the union values; vid[r, v] = the union id.  rank_span_check_kernel checks the
//      spans as in the per-value collective.  wide_comp_union_kernel enters each row's composite (g, union id) into a
//      composite table (ctl[1] = C_u) with its order key, the least key of a composite and the set of ranks that hold it.
//   2. the merge (launch_wide_merge): the composites sorted by their least order key are the insertion order of the whole scan;
//      each composite's rows are laid out in rank order, and wide_comp_fold_kernel folds them with combine_word into row c of a
//      TableLayout(C_u, F) table and pairs[c] = (g, u).
// Order key of a row (wide_order_key): series index of its first row << 33 | the span order of its rank within that series << 27
// | its position in its rank's list.  Exact because a series' spans on different ranks are disjoint (the span check): its earlier
// span comes first in the scan.  The fields fit: series indexes are below 2^31, ranks at most 64, a rank's list at most
// kWideMaxRankComposites long.
constexpr uint32_t kWideMaxRankComposites = 1u << 27;
struct WideUnionParams {
    const uint8_t *slots;             // rank r's slot at slots + r * slot_stride (the root's mailbox, this collective's parity)
    size_t slot_stride;
    uint32_t F, NS, cap, n_ranks;
    int64_t tmin, tmax;               // the query's range (span check)
    const uint32_t *v_off, *row_off;  // [n_ranks + 1] exclusive scans of V_r and C_r
    uint32_t n_vals, n_rows;          // sum of V_r, sum of C_r
    uint32_t vmask, cmask;            // slots - 1 of the value and composite tables (powers of two, at least twice the entries)
    unsigned long long *vslot;        // [vmask + 1] least (r << 32 | v) + 1 with the slot's bytes, 0 = empty
    uint32_t *vid;                    // [n_vals] the value's slot, then its union id
    uint32_t *vhead;                  // [align(n_vals, 1024)] 1 = (r, v) is the least with its bytes, then (exclusive scan) its union id
    uint32_t *tiles;                  // [align(max(n_vals, n_rows), 1024) / 1024] the exclusive scans' tile sums
    uint8_t *vals;                    // [cap * kMaxLit] union values
    uint32_t *lens;                   // [cap]
    unsigned long long *comp;         // [cmask + 1] composite (g << 32 | u) + 1, 0 = empty
    unsigned long long *cfirst;       // [cmask + 1] least order key of the composite's rows, preset ~0
    unsigned long long *cranks;       // [cmask + 1] bit r: rank r holds the composite
    uint32_t *cidx;                   // [cmask + 1] the composite's position in insertion order, preset 0xffffffff
    uint32_t *row_slot;               // [n_rows] composite slot of the row
    unsigned long long *row_key;      // [n_rows] order key of the row
    uint32_t n_sort;                  // power of two >= max(n_rows, 2048)
    unsigned long long *keys;         // [n_sort] the composites' least keys, ~0 elsewhere
    uint32_t *seg;                    // [align(n_rows, 1024)] rows of composite c, then (exclusive scan) its first entry in `order`
    uint32_t *order;                  // [n_rows] flat rows, composite by composite, each composite's in rank order
    uint32_t *ctl;                    // [0] V_u [1] C_u [2] DevErr of the span check [3] first series whose spans intersect (preset ~0)
    TablePtrs table;                  // TableLayout(C_u, F)
    int32_t *pairs;                   // [2 * C_u]
    int32_t *perm;                    // [C_u] c (the identity order keyed_partial_rows_kernel reads)
};
// -> kernels launched
uint32_t launch_wide_union(const WideUnionParams &p, cudaStream_t s);
uint32_t launch_wide_merge(const WideUnionParams &p, uint32_t n_comp, cudaStream_t s);
// ---- tuple collective (bydb_scan_reduce_keys_wide): the slot of a rank that found T tuples over K tags (tag t: V_t values, n_vals
// = the sum of the V_t) and C present composite groups, for F fields and NS series.  It is WideSlot(F, NS, n_vals, C) with the tuple
// codes behind it: span, pairs, first and table mean what they mean there, a pair naming the rank's own tuple id.
//   head      SlotHead(n_vals): Header.V = T, Header.C = C, and Tags at byte sizeof(Header); lens / values hold tag 0's V_0
//             values, then tag 1's, ... (a rank's values of tag t start at entry V_0 + .. + V_{t-1})
//   span, pairs, first, table   as in WideSlot
//   codes     [T] u64 the rank's tuple codes id_0 | id_1 << 16 | .. in its own tag ids (WidePass::codes)
struct TupleSlot : WideSlot {
    struct Tags {
        uint32_t K, V[kMaxKeyTags];
    };
    size_t off_codes, total;  // total: the whole slot (WideSlot::total ends at the table)
    __host__ __device__ TupleSlot(size_t F, size_t NS, size_t n_vals, size_t T, size_t C) : WideSlot(F, NS, n_vals, C) {
        off_codes = up(WideSlot::total);
        total = off_codes + T * 8;
    }
};
// The root of the tuple collective: the wide collective's root with a union per tag and one of the tuples in place of the value
// union.  The WideUnionParams fields name, in turn, each tag's value union (launch_tuple_tag_union sets them from tags[t]; its
// v_off / n_vals / vid then count (rank, tag-t value), and ctl points at tag_ctl[t]) and the tuple union (launch_tuple_union:
// v_off / n_vals / vid count (rank, tuple), vslot keeps the least (r, tuple) per union code, vhead numbers them), whose ids the
// composite union, the order and the fold then read as the wide collective reads its value ids.
struct TupleTagUnion {
    const uint32_t *v_off;            // [n_ranks + 1] exclusive scan of the ranks' V_t
    uint32_t n_vals, vmask;           // sum of the ranks' V_t; the value table's slots - 1
    unsigned long long *vslot;        // [vmask + 1]
    uint32_t *vid;                    // [n_vals] the union id of (r, value)
    uint8_t *vals;                    // [cap * kMaxLit] the tag's union values
    uint32_t *lens;                   // [cap]
};
struct TupleUnionParams : WideUnionParams {
    uint32_t n_tags, tag;             // K; the tag whose values a value union reads
    TupleTagUnion tags[kMaxKeyTags];
    uint32_t *tag_ctl;                // [K] each tag's union size V_u,t
    unsigned long long *codes;        // [cap] union tuple u's code in union tag ids
};
// each tag's value union, then the span check (ctl[2], ctl[3] as in the wide collective) -> kernels launched
uint32_t launch_tuple_tag_union(const TupleUnionParams &p, cudaStream_t s);
// the tuple union (ctl[0] = T_u; only when every V_u,t is at most cap, so that a union tag id fits its 16 bits), then the composite
// union (ctl[1] = C_u) -> kernels launched
uint32_t launch_tuple_union(const TupleUnionParams &p, cudaStream_t s);
uint32_t launch_wide_merge(const TupleUnionParams &p, uint32_t n_comp, cudaStream_t s);
// dst[j] = src[perm[j]] for every group row of a partial table; coltype = the passes' column types merged
void launch_permute_table(const TablePtrs &dst, const TablePtrs &src, const int32_t *perm, uint32_t n_groups, uint32_t n_fcols,
                          const int64_t *pass_coltype, uint32_t n_passes, cudaStream_t s);
// ---- a replayed keyed step (bydb_scan_agg_keyed_prepared)
// Everything the plain keyed path memsets, reset by ONE kernel at the head of the graph: the 32-bit words of zero[i] are set to 0
// (the passes' column types, their zero pages), those of ones[i] to 0xffffffff (first_block, the key-order slots).  A NULL range
// or a count of 0 is skipped.
struct KeyedResetParams {
    uint32_t *zero[2];
    size_t n_zero[2];
    uint32_t *ones[2];
    size_t n_ones[2];
};
void launch_keyed_step_reset(const KeyedResetParams &p, cudaStream_t s);
// The (series group, key value) of every selected row, in place of the host's read-back of perm: row r < min(*sel_count, cap)
// is position sel_group[r] of the insertion order, composite group c = perm[sel_group[r]] = key * n_groups + group, and
// pairs[2r] / pairs[2r + 1] = c % n_groups / c / n_groups.
void launch_keyed_row_map(const int32_t *sel_group, const uint32_t *sel_count, const int32_t *perm, uint32_t n_groups, uint32_t cap,
                          int32_t *pairs, cudaStream_t s);
constexpr int kFusedFinalizeGroups = 8192;  // up to here one CTA finalises and selects in a single launch
struct FinalizeParams;
uint32_t launch_finalize_select(const FinalizeParams &fp, const SelectParams &p, cudaStream_t s);  // -> kernels launched
// combines n partial tables of layout `tl`, stride_bytes apart (0 = back to back), into the first one, rank order
void launch_combine_tables(uint8_t *tables, uint32_t n_tables, const TableLayout &tl, cudaStream_t s, size_t stride_bytes = 0);
// peer-mailbox reduce (bydb_comm_*): bounded wait for n epoch flags, release-store of one
void launch_comm_wait(const unsigned long long *flags, uint32_t n, unsigned long long epoch, uint32_t *err, uint32_t err_code, cudaStream_t s);
void launch_comm_signal(unsigned long long *flag, unsigned long long epoch, cudaStream_t s);
// graph-replayable forms: the epoch comes from a device block refreshed by a memcpy node of the graph
struct CommArgs {
    unsigned long long epoch, prev_use;
};
void launch_comm_wait_args(const unsigned long long *flags, uint32_t n, const CommArgs *a, int which, uint32_t *err, uint32_t err_code, cudaStream_t s);
void launch_comm_signal_args(unsigned long long *flag, unsigned long long *status, const CommArgs *a, cudaStream_t s);
void launch_comm_done_args(unsigned long long *done, const CommArgs *a, cudaStream_t s);

// ---- fallback-page normalisation at part admission (unpack_kernels.cu)
constexpr uint8_t kEncRawCells = 0x40;   // numeric page rewritten as [0x40][has_nulls][6 pad][n x u64 LE][n x u8 valid]
constexpr uint8_t kBlockRawLong = 2;     // compressBlock rewritten as [2][u32 LE len][bytes] (an inflated zstd frame)
constexpr uint32_t kUnpackNumeric = 1, kUnpackString = 2;
struct UnpackJob {
    uint64_t out_off;   // into the unpack arena
    uint32_t col;       // index into the part's DevCol table
    uint32_t rows;
    uint32_t out_cap;
    uint32_t kind;
};
struct UnpackParams {
    const DevBlock *blocks;
    DevCol *cols;                   // rewritten in place for the pages that were unpacked
    const uint8_t *const *files;
    uint32_t n_blocks;
    uint32_t arena_file_id;         // slot of the unpack arena in the part's file table
    UnpackJob *jobs;
    unsigned long long max_jobs, n_jobs;
    unsigned long long *counters;   // [0] jobs found [1] arena bytes [2] cursor [3] pages left as they are [4] pages unpacked
    uint8_t *arena;
    uint8_t *scratch;               // n_warps * unpack_scratch_stride()
};
size_t unpack_scratch_stride();
void launch_classify_pages(const UnpackParams &p, cudaStream_t s);
void launch_unpack_pages(const UnpackParams &p, int n_warps, cudaStream_t s);

// ---- dense pages at part admission (scan_kernels.cu, "Dense pages"; the form: dense_page.cuh)
struct DenseParams {
    const DevBlock *blocks;
    const DevCol *cols;
    const uint8_t *const *files;
    DevDense *dense;                // [n_cols] the part's descriptor table, zeroed
    uint32_t n_blocks;
    uint32_t fv_file_id;            // the field pages' file (fv.bin)
    unsigned long long *counters;   // [0] pages classify converted [1] plane bytes [2] most rows of such a page [3] pages written
    uint8_t *arena;                 // write pass: the plane streams (classify left each page's offset in DevDense::planes)
    uint32_t *scratch;              // write pass: scratch_rows words per warp of the grid
    uint32_t scratch_rows;
    uint32_t pad;
};
// classify: a warp per block decodes each narrow field page with the fast lane's decoder and fills its descriptor (planes =
// offset into the arena); write: a warp per block decodes the converted pages again and lays out their planes
void launch_dense_classify(const DenseParams &p, int grid, cudaStream_t s);
void launch_dense_write(const DenseParams &p, int grid, cudaStream_t s);

// ---- write side: numeric field pages encoded on the device (encode_kernels.cu)
struct EncodeParams {
    const void *values;           // int64 / double, the blocks back to back
    const uint64_t *block_off;    // [n_blocks + 1] value offsets
    uint32_t n_blocks;
    uint32_t is_float;
    int64_t *scratch;             // [n_values] decimal integers of a float64 column
    int16_t *exps;                // [n_values]
    uint8_t *slots;               // worst-case page slots
    const uint64_t *slot_off;     // [n_blocks + 1]
    uint32_t *page_len;           // [n_blocks] 0 = the block goes to the CPU writer
    uint8_t *status;              // [n_blocks] 1 = not encoded here
};
void launch_encode_pages(const EncodeParams &p, int grid, cudaStream_t s);
void launch_gather_pages(const EncodeParams &p, const uint64_t *out_off, uint8_t *out, int grid, cudaStream_t s);
void preload_encode_kernels();   // encode_kernels.cu

size_t scan_smem_bytes();
size_t express_smem_bytes();
void launch_plan_blocks(const ScanParams &p, cudaStream_t s);
// start of a replayed step: zeroes the 64 words of the zero page and writes 0xffffffff over first_block[n_first] (may be NULL / 0)
void launch_step_reset(uint32_t *zero_page, uint32_t *first_block, size_t n_first, cudaStream_t s);
// grid_express: the express lane's grid (launched when p.rest_list is set), grid_fast / grid_slow: the regular lanes'
void launch_scan_blocks(const ScanParams &p, int grid_express, int grid_fast, int grid_slow, cudaStream_t s);
void launch_series_reduce(const ReduceParams &p, cudaStream_t s);
void launch_group_reduce(const ReduceParams &p, cudaStream_t s, bool small_groups = false);  // small_groups: no group has more than 32 series
void launch_finalize(const FinalizeParams &p, cudaStream_t s);
void launch_detect_overlap(const ScanParams &p, cudaStream_t s);
void launch_dedup(const ScanParams &p, int grid, cudaStream_t s);
int upload_pow10_table();
void scan_max_ctas_per_sm(int *express, int *fast, int *slow);
void preload_kernels();          // scan_kernels.cu: forces the (lazily loaded) code of every kernel onto the current device
void preload_unpack_kernels();   // unpack_kernels.cu
void preload_index_kernels();    // index_kernels.cu

}  // namespace bydb

// bydb_operator.hpp -- C++ host side above the C ABI: the reference's vectorized operator surface for this path.
//
// The reference's host code is Go (no toolchain in this image), so the layer a Go maintainer would write over the cgo
// shim is mirrored here in C++17, header-only, using nothing but include/bydb_gpu.h:
//
//   ColumnRole / ColumnType / ColumnDef / BatchSchema     pkg/query/vectorized/schema.go:32-66
//   RecordBatch (typed columns + validity)                 pkg/query/vectorized/batch.go:33, typed_column.go:26
//   AggFunc / AggSpec                                      pkg/query/vectorized/measure/aggregation.go:44-66
//   TopSpec (BatchTop)                                     pkg/query/vectorized/measure/top.go:145-214
//   LimitSpec (BatchLimit)                                 pkg/query/vectorized/measure/limit.go:27-73
//   PullOperator { Init, OutputSchema, NextBatch, Close }  pkg/query/vectorized/operator.go:34-52
//   GPUScanAgg                                             the PullOperator INTEGRATION.md installs as scan.Source in
//                                                          plan.Dispatch (dispatch.go:261-268), collapsing Scan -> GroupByAgg (-> Top)
//
// Contracts kept: NextBatch returns (batch, ok) / (nullptr, ok) at EOF / (nullptr, error) and the error is sticky;
// Close is idempotent; batches hold at most batch_size rows and never carry a Selection; the output schema is
// buildAggOutputSchema's (aggregation.go:402-418): the projected tag columns in schema order, then one RoleField column per
// AggSpec typed by aggOutputType (COUNT -> int64, otherwise the input field's type); group rows come in first-appearance
// order of the scan (reversed for an order-by DESC request), non-key projected tags carry the first-seen value.
// A GroupBy key column with per-series values (ScanSpec::SeriesTags: entity / indexed tags) is densified per series; a key column
// that is a stored tag (a tag column absent from SeriesTags) makes the operator call bydb_scan_agg_keyed(_wide), which adds the row's
// value of that tag to the group.  With MaxKeyValues above 256, two to four stored key columns go to bydb_scan_agg_keys_wide as a
// tuple, in GroupBy order; at 256 or below only one may be a stored tag.  Stored keys take the ascending series order only (no
// OrderDesc).
// tests/native/operator_test.cc drives it; the Python mirror (skywalking-banyandb_b200/scan_operator.py) follows the same code.
#pragma once

#include <algorithm>
#include <cstdint>
#include <map>
#include <memory>
#include <numeric>
#include <optional>
#include <string>
#include <utility>
#include <vector>

#include "bydb_gpu.h"

namespace bydb {
namespace vectorized {

enum class ColumnRole { RoleTag = 0, RoleField = 1 };
enum class ColumnType { ColumnTypeInt64 = 0, ColumnTypeFloat64 = 1, ColumnTypeString = 2, ColumnTypeBytes = 3 };

struct ColumnDef {
    std::string Name;
    ColumnRole Role = ColumnRole::RoleTag;
    ColumnType Type = ColumnType::ColumnTypeString;
    std::string TagFamily;  // tags only
};

struct BatchSchema {
    std::vector<ColumnDef> Columns;
};

// one typed column of a batch; Valid[i] == 0 is a null cell
struct Column {
    ColumnType Type = ColumnType::ColumnTypeInt64;
    std::vector<int64_t> Int64;
    std::vector<double> Float64;
    std::vector<std::string> Bytes;
    std::vector<uint8_t> Valid;
};

struct RecordBatch {
    const BatchSchema *Schema = nullptr;
    std::vector<Column> Columns;
    int Len = 0;  // Selection is always nil: rows are materialised
};

enum class AggFunc { AggSum = 0, AggCount = 1, AggMin = 2, AggMax = 3, AggMean = 4 };  // aggregation.go:47-55 (iota order)
// -> modelv1.AggregationFunction (BYDB_AGG_*), the numbering the C ABI takes
inline int32_t to_model_agg(AggFunc f) {
    switch (f) {
        case AggFunc::AggSum: return BYDB_AGG_SUM;
        case AggFunc::AggCount: return BYDB_AGG_COUNT;
        case AggFunc::AggMin: return BYDB_AGG_MIN;
        case AggFunc::AggMax: return BYDB_AGG_MAX;
        case AggFunc::AggMean: return BYDB_AGG_MEAN;
    }
    return 0;
}

struct AggSpec {
    std::string Output;  // name of the output column
    AggFunc Func = AggFunc::AggSum;
    int InputCol = 0;  // index into the input schema (a RoleField column)
};

struct TopSpec {
    int N = 0;
    int AggIndex = 0;
    bool Desc = true;
};

struct LimitSpec {
    uint32_t Offset = 0;
    uint32_t Limit = 100;  // the planner's default (pkg/query/logical/measure/measure_analyzer.go:31)
};

struct Pred {
    std::string Family, Tag;
    int Op = BYDB_OP_EQ;
    bool IsInt = false;
    int64_t Int = 0;
    std::string Bytes;
};

// What measure.Query resolved before the scan (banyand/measure/query.go:88-312)
struct ScanSpec {
    std::vector<bydb_part_h> Parts;
    std::vector<uint64_t> SeriesIDs;  // index order (searchSeriesList), not necessarily ascending
    // entity / indexed tag values per series (storedIndexValue, block.go:509-530): (family, tag) -> one value per series
    std::map<std::pair<std::string, std::string>, std::vector<std::string>> SeriesTags;
    int64_t TMin = INT64_MIN, TMax = INT64_MAX;
    std::vector<Pred> Preds;
    bool OrderDesc = false;
    uint32_t MaxKeyValues = 0;  // distinct values of a stored-tag GroupBy key (bydb_group_key.max_values; 0 = the library's 64);
                                // up to 256 bydb_scan_agg_keyed answers, up to 65,536 bydb_scan_agg_keyed_wide
};

struct Error {
    int Code = 0;
    std::string Msg;
};
using Status = std::optional<Error>;  // nullopt = nil

class PullOperator {
  public:
    virtual ~PullOperator() = default;
    virtual Status Init() = 0;
    virtual const BatchSchema &OutputSchema() const = 0;
    // (batch, nil) | (nullptr, nil) = EOF | (nullptr, err); the error is sticky
    virtual Status NextBatch(std::unique_ptr<RecordBatch> &out) = 0;
    virtual Status Close() = 0;
};

class GPUScanAgg final : public PullOperator {
  public:
    GPUScanAgg(bydb_ctx *ctx, BatchSchema input, std::vector<int> key_indices, std::vector<AggSpec> aggs, ScanSpec scan, int batch_size = 1024,
               std::optional<TopSpec> top = std::nullopt, std::optional<LimitSpec> limit = std::nullopt)
        : ctx_(ctx), in_(std::move(input)), keys_(std::move(key_indices)), aggs_(std::move(aggs)), scan_(std::move(scan)),
          batch_(std::max(1, batch_size)), top_(top), limit_(limit) {
        for (size_t i = 0; i < in_.Columns.size(); ++i)
            if (in_.Columns[i].Role == ColumnRole::RoleTag) tag_idx_.push_back(static_cast<int>(i));
        if (tag_idx_.empty()) tag_idx_ = keys_;
        for (int ti : tag_idx_) out_.Columns.push_back(in_.Columns[static_cast<size_t>(ti)]);
        for (const AggSpec &a : aggs_) {  // aggOutputType, aggregation.go:425-430
            ColumnDef d;
            d.Name = a.Output;
            d.Role = ColumnRole::RoleField;
            const bool in_range = a.InputCol >= 0 && static_cast<size_t>(a.InputCol) < in_.Columns.size();
            d.Type = (a.Func == AggFunc::AggCount || !in_range) ? ColumnType::ColumnTypeInt64 : in_.Columns[static_cast<size_t>(a.InputCol)].Type;
            out_.Columns.push_back(d);
        }
    }
    ~GPUScanAgg() override { (void)Close(); }

    Status Init() override {
        for (const AggSpec &a : aggs_) {
            if (a.InputCol < 0 || static_cast<size_t>(a.InputCol) >= in_.Columns.size()) return fail(BYDB_EINVAL, "AggSpec " + a.Output + ": input column out of range");
            const ColumnDef &c = in_.Columns[static_cast<size_t>(a.InputCol)];
            if (c.Role != ColumnRole::RoleField || (c.Type != ColumnType::ColumnTypeInt64 && c.Type != ColumnType::ColumnTypeFloat64))
                return fail(BYDB_EINVAL, "AggSpec " + a.Output + ": input column must be an int64/float64 field");
        }
        inited_ = true;
        return std::nullopt;
    }

    const BatchSchema &OutputSchema() const override { return out_; }

    Status NextBatch(std::unique_ptr<RecordBatch> &out) override {
        out.reset();
        if (err_) return err_;
        if (closed_) return std::nullopt;
        if (!ran_) {
            if (Status s = run()) {
                err_ = s;  // sticky (model/batch.go:41-46)
                return err_;
            }
        }
        if (cursor_ >= row_end_) return std::nullopt;  // EOF
        const bydb_result &res = result();
        const size_t lo = cursor_, hi = std::min(cursor_ + static_cast<size_t>(batch_), row_end_);
        cursor_ = hi;
        auto b = std::make_unique<RecordBatch>();
        b->Schema = &out_;
        b->Len = static_cast<int>(hi - lo);
        for (int ti : tag_idx_) {
            const ColumnDef &cd = in_.Columns[static_cast<size_t>(ti)];
            Column col;
            col.Type = cd.Type;
            const auto sk = std::find(stored_keys_.begin(), stored_keys_.end(), ti);
            if (sk != stored_keys_.end()) {
                const size_t t = static_cast<size_t>(sk - stored_keys_.begin());
                for (size_t r = lo; r < hi; ++r) {  // the row's key bytes (groupby.go:226-254); a nil cell came back as 0 / ""
                    const uint8_t *kb = nullptr;
                    size_t klen = 0;
                    key_entry(r, t, kb, klen);
                    if (cd.Type == ColumnType::ColumnTypeInt64) {
                        uint64_t u = 0;
                        for (size_t i = 0; i < klen && i < 8; ++i) u |= static_cast<uint64_t>(kb[i]) << (8 * i);
                        col.Int64.push_back(static_cast<int64_t>(u));
                    } else {
                        col.Bytes.emplace_back(reinterpret_cast<const char *>(kb), klen);
                    }
                    col.Valid.push_back(1);
                }
                b->Columns.push_back(std::move(col));
                continue;
            }
            const auto it = scan_.SeriesTags.find({cd.TagFamily, cd.Name});
            for (size_t r = lo; r < hi; ++r) {
                const int g = res.group_id[r];
                if (it == scan_.SeriesTags.end()) {
                    col.Bytes.emplace_back();
                    col.Valid.push_back(0);
                } else {
                    col.Bytes.push_back(it->second[static_cast<size_t>(group_first_series_[static_cast<size_t>(g)])]);
                    col.Valid.push_back(1);
                }
            }
            b->Columns.push_back(std::move(col));
        }
        const size_t A = aggs_.size();
        for (size_t a = 0; a < A; ++a) {
            Column col;
            const bool isf = res.is_float[a] != 0;
            col.Type = isf ? ColumnType::ColumnTypeFloat64 : ColumnType::ColumnTypeInt64;
            for (size_t r = lo; r < hi; ++r) {
                if (isf) col.Float64.push_back(res.val_f64[r * A + a]);
                else col.Int64.push_back(res.val_i64[r * A + a]);
                col.Valid.push_back(1);
            }
            b->Columns.push_back(std::move(col));
        }
        out = std::move(b);
        return std::nullopt;
    }

    Status Close() override {  // idempotent; releases the result exactly once
        if (have_result_) {
            if (stored_keys_.size() > 1) bydb_keys_result_free(ctx_, &tres_);
            else if (stored_keys_.size() == 1) bydb_keyed_result_free(ctx_, &kres_);
            else bydb_result_free(ctx_, &res_);
            have_result_ = false;
        }
        closed_ = true;
        return std::nullopt;
    }

    const bydb_stats &Stats() const { return stats_; }

  private:
    Status fail(int code, std::string msg) { return Error{code, std::move(msg)}; }
    const bydb_result &result() const { return stored_keys_.size() > 1 ? tres_.base : stored_keys_.size() == 1 ? kres_.base : res_; }
    // stored key t of row r: one key's entry key_id[r], or a tuple's entry key_id[r * n_tags + t]
    void key_entry(size_t r, size_t t, const uint8_t *&bytes, size_t &len) const {
        const bool tuple = stored_keys_.size() > 1;
        const int32_t e = tuple ? tres_.key_id[r * tres_.n_tags + t] : kres_.key_id[r];
        const uint32_t *off = tuple ? tres_.key_off : kres_.key_off;
        bytes = (tuple ? tres_.key_bytes : kres_.key_bytes) + off[e];
        len = off[e + 1] - off[e];
    }

    Status run() {
        ran_ = true;
        if (!inited_) return fail(BYDB_EINVAL, "NextBatch before Init");
        if (!ctx_) return fail(BYDB_EINVAL, "no bydb context");
        const size_t ns = scan_.SeriesIDs.size();
        // group key per series = tuple of the key columns' values; dense ids in first-appearance order of the scan
        // (aggregation.go:211-213); an order-by DESC request visits the series list backwards
        // A tag key column without per-series values is a stored tag: bydb_scan_agg_keyed adds its row value to the group, and
        // above 256 values bydb_scan_agg_keys_wide adds the tuple of two to four of them.  Any other key column (a field) still
        // needs per-series values.
        std::vector<const std::vector<std::string> *> keyvals;
        stored_keys_.clear();
        for (int ki : keys_) {
            const ColumnDef &cd = in_.Columns[static_cast<size_t>(ki)];
            const auto it = scan_.SeriesTags.find({cd.TagFamily, cd.Name});
            if (it == scan_.SeriesTags.end() && cd.Role == ColumnRole::RoleTag) {
                if (!stored_keys_.empty() && scan_.MaxKeyValues <= 256)
                    return fail(BYDB_ENOTSUP, "GroupBy key " + cd.TagFamily + "/" + cd.Name + ": at most one stored-tag key per query");
                if (stored_keys_.size() == kMaxStoredKeys)
                    return fail(BYDB_ENOTSUP, "GroupBy key " + cd.TagFamily + "/" + cd.Name + ": at most four stored-tag keys per query");
                stored_keys_.push_back(ki);
                continue;
            }
            if (it == scan_.SeriesTags.end() || it->second.size() != ns)
                return fail(BYDB_EINVAL, "GroupBy key " + cd.TagFamily + "/" + cd.Name + " needs one value per series (entity / indexed tag)");
            keyvals.push_back(&it->second);
        }
        if (!stored_keys_.empty() && scan_.OrderDesc) return fail(BYDB_ENOTSUP, "a stored-tag GroupBy key takes the ascending series order only (OrderDesc)");
        std::map<std::vector<std::string>, int32_t> group_of;
        std::vector<int32_t> gids(ns, 0);
        group_first_series_.clear();
        for (size_t step = 0; step < ns; ++step) {
            const size_t i = scan_.OrderDesc ? ns - 1 - step : step;
            std::vector<std::string> key;
            for (const auto *kv : keyvals) key.push_back((*kv)[i]);
            auto it = group_of.find(key);
            if (it == group_of.end()) {
                it = group_of.emplace(std::move(key), static_cast<int32_t>(group_of.size())).first;
                group_first_series_.push_back(static_cast<int>(i));
            }
            gids[i] = it->second;
        }
        if (keys_.empty()) {
            group_first_series_.clear();
            if (ns) group_first_series_.push_back(scan_.OrderDesc ? static_cast<int>(ns - 1) : 0);
        }
        // the C ABI wants ascending series ids (query.go:601)
        std::vector<size_t> order(ns);
        std::iota(order.begin(), order.end(), size_t{0});
        std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return scan_.SeriesIDs[a] < scan_.SeriesIDs[b]; });
        std::vector<uint64_t> sids(ns);
        std::vector<int32_t> sgroups(ns);
        for (size_t k = 0; k < ns; ++k) {
            sids[k] = scan_.SeriesIDs[order[k]];
            sgroups[k] = gids[order[k]];
        }
        std::vector<bydb_agg> cagg(aggs_.size());
        for (size_t a = 0; a < aggs_.size(); ++a) {
            cagg[a].field = in_.Columns[static_cast<size_t>(aggs_[a].InputCol)].Name.c_str();
            cagg[a].func = to_model_agg(aggs_[a].Func);
            cagg[a].reserved = 0;
        }
        std::vector<bydb_pred> cpred(scan_.Preds.size());
        for (size_t p = 0; p < scan_.Preds.size(); ++p) {
            const Pred &pr = scan_.Preds[p];
            bydb_pred &c = cpred[p];
            c.family = pr.Family.c_str();
            c.tag = pr.Tag.c_str();
            c.op = pr.Op;
            c.value_type = pr.IsInt ? BYDB_VT_INT64 : BYDB_VT_STR;
            c.lit = reinterpret_cast<const uint8_t *>(pr.Bytes.data());
            c.lit_len = pr.Bytes.size();
            c.lit_i64 = pr.Int;
        }
        bydb_query q{};
        q.n_parts = static_cast<uint32_t>(scan_.Parts.size());
        q.parts = scan_.Parts.data();
        q.n_series = ns;
        q.series_ids = sids.data();
        q.series_group = keys_.empty() ? nullptr : sgroups.data();
        q.n_groups = keys_.empty() ? 1 : std::max<int32_t>(static_cast<int32_t>(group_of.size()), 1);
        q.tmin = scan_.TMin;
        q.tmax = scan_.TMax;
        q.n_preds = static_cast<uint32_t>(cpred.size());
        q.preds = cpred.data();
        q.n_aggs = static_cast<uint32_t>(cagg.size());
        q.aggs = cagg.data();
        q.top_n = top_ ? top_->N : 0;
        q.top_agg = top_ ? top_->AggIndex : 0;
        q.top_desc = top_ ? (top_->Desc ? 1 : 0) : 1;
        int rc;
        const bool tuple = stored_keys_.size() > 1;  // MaxKeyValues then counts the distinct tuples; each tag's own max_values is 0
        std::vector<bydb_group_key> ckeys;
        for (int ki : stored_keys_) {
            const ColumnDef &cd = in_.Columns[static_cast<size_t>(ki)];
            bydb_group_key key{};
            key.family = cd.TagFamily.c_str();
            key.tag = cd.Name.c_str();
            key.max_values = tuple ? 0 : scan_.MaxKeyValues;
            key.value_type = cd.Type == ColumnType::ColumnTypeInt64 ? BYDB_VT_INT64 : 0;
            ckeys.push_back(key);
        }
        if (ckeys.empty()) {
            rc = bydb_scan_agg(ctx_, &q, &res_);
        } else if (!tuple) {
            // above the per-value passes' 256 values, the one-pass form (which answers the same rows)
            rc = scan_.MaxKeyValues > 256 ? bydb_scan_agg_keyed_wide(ctx_, &q, &ckeys[0], &kres_) : bydb_scan_agg_keyed(ctx_, &q, &ckeys[0], &kres_);
        } else {
            bydb_group_keys keys{static_cast<uint32_t>(ckeys.size()), scan_.MaxKeyValues, ckeys.data()};
            rc = bydb_scan_agg_keys_wide(ctx_, &q, &keys, &tres_);
        }
        if (rc != 0) return fail(rc, bydb_last_error() ? bydb_last_error() : "bydb_scan_agg failed");
        have_result_ = true;
        stats_ = result().stats;
        // offset / limit window over the (Top-ordered) output rows, limit.go:56-73
        const size_t n = static_cast<size_t>(result().n_rows);
        if (limit_) {
            cursor_ = std::min<size_t>(limit_->Offset, n);
            row_end_ = std::min<size_t>(cursor_ + limit_->Limit, n);
        } else {
            cursor_ = 0;
            row_end_ = n;
        }
        return std::nullopt;
    }

    bydb_ctx *ctx_;
    BatchSchema in_, out_;
    std::vector<int> keys_, tag_idx_;
    std::vector<AggSpec> aggs_;
    ScanSpec scan_;
    int batch_;
    std::optional<TopSpec> top_;
    std::optional<LimitSpec> limit_;
    bydb_result res_{};
    static constexpr size_t kMaxStoredKeys = 4;  // the tags of a bydb_group_keys tuple
    bydb_keyed_result kres_{};  // the result when one GroupBy key is a stored tag
    bydb_keys_result tres_{};   // the result when two to four are
    std::vector<int> stored_keys_;  // input columns of those keys, in GroupBy order
    bydb_stats stats_{};
    std::vector<int> group_first_series_;
    size_t cursor_ = 0, row_end_ = 0;
    bool inited_ = false, ran_ = false, closed_ = false, have_result_ = false;
    Status err_;
};

}  // namespace vectorized
}  // namespace bydb

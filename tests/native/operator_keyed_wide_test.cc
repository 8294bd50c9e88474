// Drives the C++ operator (include/bydb_operator.hpp) with a stored-tag GroupBy key of more than 256 values: a part written with
// bydb_part_write holds 32 series whose string tag "k" takes 1,000 values over the part (at most 200 per block).  With
// MaxKeyValues = 1000 the operator must answer through the one-pass form: every row is checked against
// bydb_scan_agg_keyed_wide called directly, with and without a per-series key, under Top and an offset / limit window.  With
// MaxKeyValues = 256 it stays on the per-value passes, which refuse 1,000 values (BYDB_ENOMEM).  Without a device the program
// checks the output schema and the error contract only.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "bydb_operator.hpp"
#include "bydb_synth.h"

using namespace bydb::vectorized;

static int fails = 0;
#define CHECK(cond, what)                                               \
    do {                                                                \
        if (!(cond)) {                                                  \
            std::printf("FAIL %s (%s:%d)\n", what, __FILE__, __LINE__); \
            ++fails;                                                    \
        }                                                               \
    } while (0)

constexpr int kSeries = 32, kRows = 1000, kValues = 1000, kWindow = 200;

// input columns: 0 svc (per series), 1 k (stored string tag), 2 i (int64 field), 3 f (float64 field)
static BatchSchema input_schema() {
    BatchSchema s;
    s.Columns.push_back({"svc", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"k", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"i", ColumnRole::RoleField, ColumnType::ColumnTypeInt64, ""});
    s.Columns.push_back({"f", ColumnRole::RoleField, ColumnType::ColumnTypeFloat64, ""});
    return s;
}

struct Row {
    std::string svc, k;
    bool svc_valid = false, k_valid = false;
    int64_t sum = 0, count = 0;
    double max = 0;
};

static std::vector<Row> drain(GPUScanAgg &op, Status *err_out) {
    std::vector<Row> rows;
    for (;;) {
        std::unique_ptr<RecordBatch> b;
        Status s = op.NextBatch(b);
        if (s) {
            *err_out = s;
            break;
        }
        if (!b) break;
        for (size_t i = 0; i < static_cast<size_t>(b->Len); ++i) {
            Row r;
            r.svc_valid = b->Columns[0].Valid[i] != 0;
            if (r.svc_valid) r.svc = b->Columns[0].Bytes[i];
            r.k_valid = b->Columns[1].Valid[i] != 0;
            if (r.k_valid) r.k = b->Columns[1].Bytes[i];
            r.sum = b->Columns[2].Int64[i];
            r.count = b->Columns[3].Int64[i];
            r.max = b->Columns[4].Float64[i];
            rows.push_back(r);
        }
    }
    return rows;
}

int main() {
    const std::vector<AggSpec> aggs = {{"s", AggFunc::AggSum, 2}, {"n", AggFunc::AggCount, 2}, {"m", AggFunc::AggMax, 3}};
    {
        ScanSpec none;
        none.MaxKeyValues = kValues;
        GPUScanAgg op(nullptr, input_schema(), {1}, aggs, none);
        const BatchSchema &o = op.OutputSchema();
        CHECK(o.Columns.size() == 5 && o.Columns[1].Name == "k" && o.Columns[1].Type == ColumnType::ColumnTypeString, "stored key column typed string");
        CHECK(!op.Init(), "Init succeeds");
        std::unique_ptr<RecordBatch> b;
        Status e = op.NextBatch(b);
        CHECK(e && !b && e->Code == BYDB_EINVAL, "no context -> (nil, err)");
    }
    bydb_ctx *ctx = nullptr;
    if (bydb_init(nullptr, &ctx) != 0) {
        std::printf("%s (no GPU: contract checks only): %s\n", fails ? "FAILED" : "OK host-only", bydb_last_error());
        return fails ? 1 : 0;
    }
    // the part: series j takes its key from a window of kWindow values starting at j * step (mod kValues), every value occurs
    const int step = (kValues - kWindow + kSeries - 2) / (kSeries - 1);
    std::vector<std::string> pool(kValues);
    std::vector<const char *> pool_c(kValues);
    for (int v = 0; v < kValues; ++v) {
        char buf[16];
        std::snprintf(buf, sizeof buf, "val-%05d", v);
        pool[v] = buf;
    }
    for (int v = 0; v < kValues; ++v) pool_c[v] = pool[v].c_str();
    const size_t n = static_cast<size_t>(kSeries) * kRows;
    std::vector<uint64_t> sids(n);
    std::vector<int64_t> ts(n), ver(n, 1), iv(n), fk(n);
    std::vector<uint32_t> kidx(n);
    for (int j = 0; j < kSeries; ++j)
        for (int r = 0; r < kRows; ++r) {
            const size_t x = static_cast<size_t>(j) * kRows + r;
            sids[x] = 1 + static_cast<uint64_t>(j);
            ts[x] = 1700000000000000000LL + 60000000000LL * r;
            iv[x] = (r * 31 + j * 7) % 1000 - 300;
            fk[x] = (r * 53 + j) % 3000 + 1;  // f = fk / 10
            kidx[x] = static_cast<uint32_t>((j * step + (r * 7 + j) % kWindow) % kValues);
        }
    bydb_wcolumn fields[2] = {};
    fields[0].name = "i";
    fields[0].value_type = BYDB_VT_INT64;
    fields[0].dec_digits = -1;
    fields[0].i64 = iv.data();
    fields[1].name = "f";
    fields[1].value_type = BYDB_VT_FLOAT64;
    fields[1].dec_digits = 1;
    fields[1].dec_k = fk.data();
    bydb_wcolumn tag = {};
    tag.name = "k";
    tag.value_type = BYDB_VT_STR;
    tag.dec_digits = -1;
    tag.str_idx = kidx.data();
    tag.str_values = pool_c.data();
    tag.n_str_values = kValues;
    bydb_write_input in{};
    in.n_rows = n;
    in.series_ids = sids.data();
    in.timestamps = ts.data();
    in.versions = ver.data();
    in.n_fields = 2;
    in.fields = fields;
    in.tag_family = "default";
    in.n_tags = 1;
    in.tags = &tag;
    bydb_part_image *img = nullptr;
    CHECK(bydb_part_write(&in, &img) == 0, "write part");
    std::vector<bydb_file> files(bydb_part_image_n_files(img));
    for (uint32_t i = 0; i < files.size(); ++i) {
        files[i].name = bydb_part_image_file_name(img, i);
        files[i].data = bydb_part_image_file_data(img, i, &files[i].len);
    }
    bydb_part_files pf{static_cast<uint32_t>(files.size()), files.data()};
    bydb_part_h h = 0;
    CHECK(bydb_part_register(ctx, 1, &pf, &h) == 0, "register");
    ScanSpec scan;
    scan.Parts = {h};
    scan.MaxKeyValues = kValues;
    std::vector<std::string> svc;
    for (int i = kSeries - 1; i >= 0; --i) {  // index order is not ascending
        scan.SeriesIDs.push_back(1 + static_cast<uint64_t>(i));
        svc.push_back("svc_" + std::to_string(i % 3));
    }
    scan.SeriesTags[{"default", "svc"}] = svc;
    bydb_agg cagg[3] = {{"i", BYDB_AGG_SUM, 0}, {"i", BYDB_AGG_COUNT, 0}, {"f", BYDB_AGG_MAX, 0}};
    // svc groups in index order (series 32 first): svc_1 (i = 31), svc_0 (i = 30), svc_2 (i = 29)
    const char *group_svc[3] = {"svc_1", "svc_0", "svc_2"};
    auto direct = [&](bool per_series, int top_n, bydb_keyed_result *r) {
        std::vector<uint64_t> ids;
        std::vector<int32_t> groups;
        for (int i = 0; i < kSeries; ++i) {
            ids.push_back(1 + static_cast<uint64_t>(i));
            groups.push_back(per_series ? (i % 3 == 1 ? 0 : i % 3 == 0 ? 1 : 2) : 0);
        }
        bydb_query q{};
        q.n_parts = 1;
        q.parts = &h;
        q.n_series = kSeries;
        q.series_ids = ids.data();
        q.series_group = groups.data();
        q.n_groups = per_series ? 3 : 1;
        q.tmin = INT64_MIN;
        q.tmax = INT64_MAX;
        q.n_aggs = 3;
        q.aggs = cagg;
        q.top_n = top_n;
        q.top_agg = 1;
        q.top_desc = 1;
        bydb_group_key key{"default", "k", kValues, 0};
        return bydb_scan_agg_keyed_wide(ctx, &q, &key, r);
    };
    auto key_of = [](const bydb_keyed_result &r, size_t i) {
        const int32_t k = r.key_id[i];
        return std::string(reinterpret_cast<const char *>(r.key_bytes + r.key_off[k]), r.key_off[k + 1] - r.key_off[k]);
    };
    {  // per-series key svc + the stored key k
        GPUScanAgg op(ctx, input_schema(), {0, 1}, aggs, scan, 300);
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "svc + k: no error");
        bydb_keyed_result r{};
        CHECK(direct(true, 0, &r) == 0, "direct wide call (svc + k)");
        CHECK(r.n_keys == kValues && rows.size() == static_cast<size_t>(r.base.n_rows) && rows.size() > 256, "svc + k: row count");
        int64_t total = 0;
        for (size_t i = 0; i < rows.size() && i < static_cast<size_t>(r.base.n_rows); ++i) {
            CHECK(rows[i].svc_valid && rows[i].svc == group_svc[r.base.group_id[i]], "svc from the group's first series");
            CHECK(rows[i].k_valid && rows[i].k == key_of(r, i), "k from the row's key bytes");
            CHECK(rows[i].sum == r.base.val_i64[i * 3] && rows[i].count == r.base.val_i64[i * 3 + 1] && rows[i].max == r.base.val_f64[i * 3 + 2],
                  "aggregates as the direct call");
            total += rows[i].count;
        }
        CHECK(total == static_cast<int64_t>(n), "every datapoint counted once");
        bydb_keyed_result_free(ctx, &r);
    }
    {  // the stored key alone: Top 40 by COUNT, then the window offset 5 limit 20
        GPUScanAgg op(ctx, input_schema(), {1}, aggs, scan, 7, TopSpec{40, 1, true}, LimitSpec{5, 20});
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "k under Top: no error");
        bydb_keyed_result r{};
        CHECK(direct(false, 40, &r) == 0, "direct wide call (k, Top 40)");
        CHECK(r.base.n_rows == 40 && rows.size() == 20, "Top 40 then offset 5 limit 20");
        for (size_t i = 0; i < rows.size() && i + 5 < static_cast<size_t>(r.base.n_rows); ++i) {
            CHECK(rows[i].k_valid && rows[i].k == key_of(r, i + 5), "k as the direct call");
            CHECK(rows[i].svc_valid && rows[i].svc == "svc_1", "a per-series tag carries the first series' value");
            CHECK(rows[i].count == r.base.val_i64[(i + 5) * 3 + 1] && rows[i].sum == r.base.val_i64[(i + 5) * 3], "aggregates as the direct call");
        }
        bydb_keyed_result_free(ctx, &r);
    }
    {  // MaxKeyValues = 256 keeps the per-value passes, which refuse 1,000 values
        ScanSpec narrow = scan;
        narrow.MaxKeyValues = 256;
        GPUScanAgg op(ctx, input_schema(), {1}, aggs, narrow, 64);
        (void)op.Init();
        std::unique_ptr<RecordBatch> b;
        Status e = op.NextBatch(b);
        CHECK(e && !b && e->Code == BYDB_ENOMEM, "MaxKeyValues 256 over 1,000 values: ENOMEM from the per-value passes");
        ScanSpec over = scan;
        over.MaxKeyValues = 65537;
        GPUScanAgg op2(ctx, input_schema(), {1}, aggs, over, 64);
        (void)op2.Init();
        Status e2 = op2.NextBatch(b);
        CHECK(e2 && e2->Code == BYDB_EINVAL, "MaxKeyValues above 65,536: EINVAL");
    }
    bydb_part_release(ctx, h);
    bydb_part_image_free(img);
    bydb_shutdown(ctx);
    std::printf("%s\n", fails ? "FAILED" : "OK full");
    return fails ? 1 : 0;
}

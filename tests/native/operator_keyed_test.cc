// Drives the C++ operator (include/bydb_operator.hpp) with a GroupBy key that is a stored tag: without a device the output
// schema types the stored key column; with one, a synthetic part with the int64 tag "code" and the string tag "zone" runs a
// per-series key plus the stored string key, the stored int64 key alone under Top and an offset / limit window, and the
// refusals (two stored keys, OrderDesc).  Every row is checked against bydb_scan_agg_keyed called directly.
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

// input columns: 0 svc (per series), 1 zone (stored string), 2 code (stored int64), 3 latency (field)
static BatchSchema input_schema() {
    BatchSchema s;
    s.Columns.push_back({"svc", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"zone", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"code", ColumnRole::RoleTag, ColumnType::ColumnTypeInt64, "default"});
    s.Columns.push_back({"latency", ColumnRole::RoleField, ColumnType::ColumnTypeFloat64, ""});
    return s;
}

struct Row {
    std::string svc, zone;
    int64_t code = 0;
    bool svc_valid = false, zone_valid = false, code_valid = false;
    double sum = 0;
    int64_t count = 0;
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
        CHECK(b->Len > 0 && b->Len <= 2, "batch length within (0, 2]");
        for (size_t i = 0; i < static_cast<size_t>(b->Len); ++i) {
            Row r;
            const Column &svc = b->Columns[0], &zone = b->Columns[1], &code = b->Columns[2];
            r.svc_valid = svc.Valid[i] != 0;
            if (r.svc_valid) r.svc = svc.Bytes[i];
            r.zone_valid = zone.Valid[i] != 0;
            if (r.zone_valid && zone.Bytes.size() > i) r.zone = zone.Bytes[i];
            r.code_valid = code.Valid[i] != 0;
            if (r.code_valid && code.Type == ColumnType::ColumnTypeInt64 && code.Int64.size() > i) r.code = code.Int64[i];
            r.sum = b->Columns[3].Float64[i];
            r.count = b->Columns[4].Int64[i];
            rows.push_back(r);
        }
    }
    return rows;
}

int main() {
    {
        GPUScanAgg op(nullptr, input_schema(), {0, 2}, {{"s", AggFunc::AggSum, 3}, {"n", AggFunc::AggCount, 3}}, ScanSpec{});
        const BatchSchema &o = op.OutputSchema();
        CHECK(o.Columns.size() == 5 && o.Columns[2].Name == "code" && o.Columns[2].Type == ColumnType::ColumnTypeInt64, "stored int64 key column typed int64");
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
    bydb_synth_field fld = {"latency", BYDB_SYN_F_LATENCY, 0};
    bydb_synth_spec sp{};
    sp.n_series = 10;
    sp.n_points = 700;
    sp.sid0 = 5;
    sp.sid_step = 2;
    sp.t0 = 1700000000000000000LL;
    sp.t_step = 60000000000LL;
    sp.n_fields = 1;
    sp.fields = &fld;
    sp.code_tag = 3;  // int64 "code" and string "zone"
    sp.seed = 7;
    bydb_part_image *img = nullptr;
    CHECK(bydb_synth_part(&sp, &img) == 0, "synth part");
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
    std::vector<std::string> svc;
    for (int i = 9; i >= 0; --i) {  // index order is not ascending
        scan.SeriesIDs.push_back(5 + 2 * static_cast<uint64_t>(i));
        svc.push_back("svc_" + std::to_string(i % 3));
    }
    scan.SeriesTags[{"default", "svc"}] = svc;
    const std::vector<AggSpec> aggs = {{"sum_v", AggFunc::AggSum, 3}, {"n", AggFunc::AggCount, 3}};
    bydb_agg cagg[2] = {{"latency", BYDB_AGG_SUM, 0}, {"latency", BYDB_AGG_COUNT, 0}};

    // the direct call: series ascending, series_group = svc's first appearance in index order (svc_0 is series 9 -> group 0)
    auto direct = [&](bool per_series, const char *tag, uint32_t vt, int top_n, bydb_keyed_result *r) {
        std::vector<uint64_t> sids;
        std::vector<int32_t> groups;
        for (int i = 0; i < 10; ++i) {
            sids.push_back(5 + 2 * static_cast<uint64_t>(i));
            groups.push_back(per_series ? (i % 3 == 0 ? 0 : i % 3 == 2 ? 1 : 2) : 0);  // svc_0, svc_2, svc_1 first seen in that order
        }
        bydb_query q{};
        q.n_parts = 1;
        q.parts = &h;
        q.n_series = 10;
        q.series_ids = sids.data();
        q.series_group = groups.data();
        q.n_groups = per_series ? 3 : 1;
        q.tmin = INT64_MIN;
        q.tmax = INT64_MAX;
        q.n_aggs = 2;
        q.aggs = cagg;
        q.top_n = top_n;
        q.top_agg = 1;
        q.top_desc = 1;
        bydb_group_key key{"default", tag, 0, vt};
        return bydb_scan_agg_keyed(ctx, &q, &key, r);
    };
    const char *group_svc[3] = {"svc_0", "svc_2", "svc_1"};
    {  // per-series key svc + stored string key zone
        GPUScanAgg op(ctx, input_schema(), {0, 1}, aggs, scan, 2);
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "svc + zone: no error");
        bydb_keyed_result r{};
        CHECK(direct(true, "zone", 0, 0, &r) == 0, "direct call (zone)");
        CHECK(rows.size() == static_cast<size_t>(r.base.n_rows) && rows.size() >= 3, "svc + zone: row count");
        int64_t total = 0;
        for (size_t i = 0; i < rows.size() && i < static_cast<size_t>(r.base.n_rows); ++i) {
            const int32_t k = r.key_id[i];
            const std::string zone(reinterpret_cast<const char *>(r.key_bytes + r.key_off[k]), r.key_off[k + 1] - r.key_off[k]);
            CHECK(rows[i].svc_valid && rows[i].svc == group_svc[r.base.group_id[i]], "svc from the group's first series");
            CHECK(rows[i].zone_valid && rows[i].zone == zone, "zone from the row's key bytes");
            CHECK(!rows[i].code_valid, "a non-key stored tag is null");
            CHECK(rows[i].count == r.base.val_i64[i * 2 + 1] && rows[i].sum == r.base.val_f64[i * 2], "aggregates as the direct call");
            total += rows[i].count;
        }
        CHECK(total == 10 * 700, "every datapoint counted once");
        bydb_keyed_result_free(ctx, &r);
    }
    {  // stored int64 key code alone: Top 4 by COUNT, then the window offset 1 limit 2
        GPUScanAgg op(ctx, input_schema(), {2}, aggs, scan, 2, TopSpec{4, 1, true}, LimitSpec{1, 2});
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "code: no error");
        bydb_keyed_result r{};
        CHECK(direct(false, "code", BYDB_VT_INT64, 4, &r) == 0, "direct call (code)");
        CHECK(r.base.n_rows == 4 && rows.size() == 2, "Top 4 then offset 1 limit 2");
        for (size_t i = 0; i < rows.size() && i + 1 < static_cast<size_t>(r.base.n_rows); ++i) {
            const int32_t k = r.key_id[i + 1];
            CHECK(r.key_off[k + 1] - r.key_off[k] == 8, "int64 key bytes");
            int64_t v = 0;
            std::memcpy(&v, r.key_bytes + r.key_off[k], 8);
            CHECK(rows[i].code_valid && rows[i].code == v, "code decoded from little-endian key bytes");
            CHECK(v % 100 == 0 && v >= 0 && v <= 500, "code in {0, 100, .., 500}");
            CHECK(rows[i].svc_valid && rows[i].svc == "svc_0", "a per-series tag carries the first series' value");
            CHECK(!rows[i].zone_valid, "a non-key stored tag is null");
            CHECK(rows[i].count == r.base.val_i64[(i + 1) * 2 + 1], "count as the direct call");
        }
        bydb_keyed_result_free(ctx, &r);
    }
    {  // refusals
        GPUScanAgg two(ctx, input_schema(), {1, 2}, aggs, scan, 2);
        (void)two.Init();
        std::unique_ptr<RecordBatch> b;
        Status e = two.NextBatch(b);
        CHECK(e && e->Code == BYDB_ENOTSUP && e->Msg.find("default/code") != std::string::npos, "two stored keys: ENOTSUP naming the second");
        ScanSpec rev = scan;
        rev.OrderDesc = true;
        GPUScanAgg desc(ctx, input_schema(), {2}, aggs, rev, 2);
        (void)desc.Init();
        Status e2 = desc.NextBatch(b);
        CHECK(e2 && e2->Code == BYDB_ENOTSUP, "OrderDesc with a stored key: ENOTSUP");
        GPUScanAgg field_key(ctx, input_schema(), {3}, aggs, scan, 2);  // a field column is never a stored tag
        (void)field_key.Init();
        Status e3 = field_key.NextBatch(b);
        CHECK(e3 && e3->Code == BYDB_EINVAL, "a field column as a key without per-series values: EINVAL");
    }
    bydb_part_release(ctx, h);
    bydb_part_image_free(img);
    bydb_shutdown(ctx);
    std::printf("%s\n", fails ? "FAILED" : "OK full");
    return fails ? 1 : 0;
}

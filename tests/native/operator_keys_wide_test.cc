// Drives the C++ operator (include/bydb_operator.hpp) with two to four stored-tag GroupBy keys: a part written with bydb_part_write
// holds 32 series whose row carries a tuple u of 1,000 (at most 200 per block), stored as a string tag "ep" (u / 10), an int64 tag
// "code" (200 + u % 10), a string tag "z" (u % 2) and an int64 tag "w" (u % 3).  With MaxKeyValues = 1000 the operator must answer
// through bydb_scan_agg_keys_wide: every row is checked against that call made directly, with a per-series key, under Top and an
// offset / limit window, and with four stored keys.  A fifth stored key, two stored keys at MaxKeyValues 256 and OrderDesc are
// refused with BYDB_ENOTSUP.  Without a device the program checks the output schema and the error contract only.
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

constexpr int kSeries = 32, kRows = 1000, kTuples = 1000;
constexpr size_t kTags = 5;  // svc ep code z w

// input columns: 0 svc (per series), 1 ep (stored string), 2 code (stored int64), 3 z (stored string), 4 w (stored int64),
// 5 i (int64 field), 6 f (float64 field)
static BatchSchema input_schema() {
    BatchSchema s;
    s.Columns.push_back({"svc", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"ep", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"code", ColumnRole::RoleTag, ColumnType::ColumnTypeInt64, "default"});
    s.Columns.push_back({"z", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
    s.Columns.push_back({"w", ColumnRole::RoleTag, ColumnType::ColumnTypeInt64, "default"});
    s.Columns.push_back({"i", ColumnRole::RoleField, ColumnType::ColumnTypeInt64, ""});
    s.Columns.push_back({"f", ColumnRole::RoleField, ColumnType::ColumnTypeFloat64, ""});
    return s;
}

// a tag cell as bytes: a string's bytes, an int64's 8 little-endian bytes; "" with valid = false for a null cell
struct Row {
    std::string tag[kTags];
    bool valid[kTags] = {};
    int64_t sum = 0, count = 0;
    double max = 0;
};

static std::string le(int64_t v) {
    std::string s(8, '\0');
    for (int i = 0; i < 8; ++i) s[static_cast<size_t>(i)] = static_cast<char>((static_cast<uint64_t>(v) >> (8 * i)) & 0xff);
    return s;
}

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
            for (size_t t = 0; t < kTags; ++t) {
                const Column &c = b->Columns[t];
                r.valid[t] = c.Valid[i] != 0;
                if (r.valid[t]) r.tag[t] = c.Type == ColumnType::ColumnTypeInt64 ? le(c.Int64[i]) : c.Bytes[i];
            }
            r.sum = b->Columns[kTags].Int64[i];
            r.count = b->Columns[kTags + 1].Int64[i];
            r.max = b->Columns[kTags + 2].Float64[i];
            rows.push_back(r);
        }
    }
    return rows;
}

static Status first_error(GPUScanAgg &op) {
    (void)op.Init();
    std::unique_ptr<RecordBatch> b;
    return op.NextBatch(b);
}

int main() {
    const std::vector<AggSpec> aggs = {{"s", AggFunc::AggSum, 5}, {"n", AggFunc::AggCount, 5}, {"m", AggFunc::AggMax, 6}};
    {
        ScanSpec none;
        none.MaxKeyValues = kTuples;
        GPUScanAgg op(nullptr, input_schema(), {1, 2}, aggs, none);
        const BatchSchema &o = op.OutputSchema();
        CHECK(o.Columns.size() == kTags + 3 && o.Columns[1].Name == "ep" && o.Columns[1].Type == ColumnType::ColumnTypeString &&
                  o.Columns[2].Name == "code" && o.Columns[2].Type == ColumnType::ColumnTypeInt64,
              "stored key columns typed as the input");
        CHECK(o.Columns[kTags + 1].Type == ColumnType::ColumnTypeInt64 && o.Columns[kTags + 2].Type == ColumnType::ColumnTypeFloat64, "aggregate columns typed");
        CHECK(!op.Init(), "Init succeeds");
        std::unique_ptr<RecordBatch> b;
        Status e = op.NextBatch(b);
        CHECK(e && !b && e->Code == BYDB_EINVAL, "no context -> (nil, err)");
        Status again = op.NextBatch(b);
        CHECK(again && again->Code == BYDB_EINVAL && !b, "the error is sticky");
        CHECK(!op.Close() && !op.Close(), "Close is idempotent");
    }
    bydb_ctx *ctx = nullptr;
    if (bydb_init(nullptr, &ctx) != 0) {
        std::printf("%s (no GPU: contract checks only): %s\n", fails ? "FAILED" : "OK host-only", bydb_last_error());
        return fails ? 1 : 0;
    }
    std::vector<std::string> eps(kTuples / 10);
    std::vector<const char *> eps_c(eps.size());
    for (size_t e = 0; e < eps.size(); ++e) {
        char buf[48];
        std::snprintf(buf, sizeof buf, "/api/ep-%03d", static_cast<int>(e));
        eps[e] = buf;
    }
    for (size_t e = 0; e < eps.size(); ++e) eps_c[e] = eps[e].c_str();
    const char *zs[2] = {"z0", "z1"};
    const size_t n = static_cast<size_t>(kSeries) * kRows;
    std::vector<uint64_t> sids(n);
    std::vector<int64_t> ts(n), ver(n, 1), iv(n), fk(n), code(n), w(n);
    std::vector<uint32_t> ep(n), z(n);
    for (int j = 0; j < kSeries; ++j)
        for (int r = 0; r < kRows; ++r) {
            const size_t x = static_cast<size_t>(j) * kRows + r;
            const int u = (j * 31 + r / 5) % kTuples;
            sids[x] = 1 + static_cast<uint64_t>(j);
            ts[x] = 1700000000000000000LL + 60000000000LL * r;
            iv[x] = (r * 31 + j * 7) % 1000 - 300;
            fk[x] = (r * 53 + j) % 3000 + 1;  // f = fk / 10
            ep[x] = static_cast<uint32_t>(u / 10);
            code[x] = 200 + u % 10;
            z[x] = static_cast<uint32_t>(u % 2);
            w[x] = u % 3;
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
    bydb_wcolumn tags[4] = {};
    tags[0].name = "ep";
    tags[0].value_type = BYDB_VT_STR;
    tags[0].dec_digits = -1;
    tags[0].str_idx = ep.data();
    tags[0].str_values = eps_c.data();
    tags[0].n_str_values = static_cast<uint32_t>(eps_c.size());
    tags[1].name = "code";
    tags[1].value_type = BYDB_VT_INT64;
    tags[1].dec_digits = -1;
    tags[1].i64 = code.data();
    tags[2].name = "z";
    tags[2].value_type = BYDB_VT_STR;
    tags[2].dec_digits = -1;
    tags[2].str_idx = z.data();
    tags[2].str_values = zs;
    tags[2].n_str_values = 2;
    tags[3].name = "w";
    tags[3].value_type = BYDB_VT_INT64;
    tags[3].dec_digits = -1;
    tags[3].i64 = w.data();
    bydb_write_input in{};
    in.n_rows = n;
    in.series_ids = sids.data();
    in.timestamps = ts.data();
    in.versions = ver.data();
    in.n_fields = 2;
    in.fields = fields;
    in.tag_family = "default";
    in.n_tags = 4;
    in.tags = tags;
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
    scan.MaxKeyValues = kTuples;
    std::vector<std::string> svc;
    for (int i = kSeries - 1; i >= 0; --i) {  // index order is not ascending
        scan.SeriesIDs.push_back(1 + static_cast<uint64_t>(i));
        svc.push_back("svc_" + std::to_string(i % 3));
    }
    scan.SeriesTags[{"default", "svc"}] = svc;
    bydb_agg cagg[3] = {{"i", BYDB_AGG_SUM, 0}, {"i", BYDB_AGG_COUNT, 0}, {"f", BYDB_AGG_MAX, 0}};
    // svc groups in index order (series 32 first): svc_1 (i = 31), svc_0 (i = 30), svc_2 (i = 29)
    const char *group_svc[3] = {"svc_1", "svc_0", "svc_2"};
    const char *names[kTags] = {"svc", "ep", "code", "z", "w"};
    // the direct call over the stored tags `cols` (input columns 1..4) in that order
    auto direct = [&](bool per_series, int top_n, const std::vector<int> &cols, bydb_keys_result *r) {
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
        std::vector<bydb_group_key> keys;
        for (int c : cols) keys.push_back({"default", names[c], 0, static_cast<uint32_t>(c == 2 || c == 4 ? BYDB_VT_INT64 : 0)});
        bydb_group_keys gk{static_cast<uint32_t>(keys.size()), kTuples, keys.data()};
        return bydb_scan_agg_keys_wide(ctx, &q, &gk, r);
    };
    auto key_of = [](const bydb_keys_result &r, size_t i, size_t t) {
        const int32_t e = r.key_id[i * r.n_tags + t];
        return std::string(reinterpret_cast<const char *>(r.key_bytes + r.key_off[e]), r.key_off[e + 1] - r.key_off[e]);
    };
    // rows[i] (operator) against row i + off of the direct answer over the stored columns `cols`
    auto same_rows = [&](const std::vector<Row> &rows, const bydb_keys_result &r, size_t off, const std::vector<int> &cols, bool per_series) {
        for (size_t i = 0; i < rows.size() && i + off < static_cast<size_t>(r.base.n_rows); ++i) {
            const size_t j = i + off;
            for (size_t t = 1; t < kTags; ++t) {
                size_t at = cols.size();
                for (size_t c = 0; c < cols.size(); ++c)
                    if (static_cast<size_t>(cols[c]) == t) at = c;
                if (at == cols.size()) CHECK(!rows[i].valid[t], "a non-key stored tag is null");
                else CHECK(rows[i].valid[t] && rows[i].tag[t] == key_of(r, j, at), "a stored key column holds the row's key bytes");
            }
            CHECK(rows[i].valid[0] && rows[i].tag[0] == (per_series ? group_svc[r.base.group_id[j]] : "svc_1"), "svc from the group's first series");
            CHECK(rows[i].sum == r.base.val_i64[j * 3] && rows[i].count == r.base.val_i64[j * 3 + 1] && rows[i].max == r.base.val_f64[j * 3 + 2],
                  "aggregates as the direct call");
        }
    };
    {  // per-series key svc + the stored keys (ep, code), in batches of 300
        GPUScanAgg op(ctx, input_schema(), {0, 1, 2}, aggs, scan, 300);
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "svc + ep + code: no error");
        bydb_keys_result r{};
        CHECK(direct(true, 0, {1, 2}, &r) == 0, "direct tuple call (svc + ep + code)");
        CHECK(r.n_tuples == kTuples && rows.size() == static_cast<size_t>(r.base.n_rows) && rows.size() > 256, "svc + ep + code: row count");
        same_rows(rows, r, 0, {1, 2}, true);
        int64_t total = 0;
        for (const Row &row : rows) total += row.count;
        CHECK(total == static_cast<int64_t>(n), "every datapoint counted once");
        bydb_keys_result_free(ctx, &r);
    }
    {  // (code, ep) alone, the keys in GroupBy order: Top 40 by COUNT, then the window offset 5 limit 20, in batches of 7
        GPUScanAgg op(ctx, input_schema(), {2, 1}, aggs, scan, 7, TopSpec{40, 1, true}, LimitSpec{5, 20});
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "code + ep under Top: no error");
        bydb_keys_result r{};
        CHECK(direct(false, 40, {2, 1}, &r) == 0, "direct tuple call (code + ep, Top 40)");
        CHECK(r.base.n_rows == 40 && rows.size() == 20, "Top 40 then offset 5 limit 20");
        same_rows(rows, r, 5, {2, 1}, false);
        bydb_keys_result_free(ctx, &r);
    }
    {  // four stored keys
        GPUScanAgg op(ctx, input_schema(), {1, 2, 3, 4}, aggs, scan, 128);
        CHECK(!op.Init(), "Init");
        Status err;
        auto rows = drain(op, &err);
        CHECK(!err, "four stored keys: no error");
        bydb_keys_result r{};
        CHECK(direct(false, 0, {1, 2, 3, 4}, &r) == 0, "direct tuple call (four tags)");
        CHECK(r.n_tags == 4 && rows.size() == static_cast<size_t>(r.base.n_rows) && !rows.empty(), "four stored keys: row count");
        same_rows(rows, r, 0, {1, 2, 3, 4}, false);
        bydb_keys_result_free(ctx, &r);
    }
    {  // refusals: a fifth stored key, two stored keys at MaxKeyValues 256, OrderDesc
        BatchSchema five = input_schema();
        five.Columns.push_back({"v", ColumnRole::RoleTag, ColumnType::ColumnTypeString, "default"});
        GPUScanAgg op5(ctx, five, {1, 2, 3, 4, 7}, aggs, scan, 64);
        Status e5 = first_error(op5);
        CHECK(e5 && e5->Code == BYDB_ENOTSUP && e5->Msg.find("default/v") != std::string::npos, "a fifth stored key: ENOTSUP naming it");
        ScanSpec narrow = scan;
        narrow.MaxKeyValues = 256;
        GPUScanAgg op2(ctx, input_schema(), {1, 2}, aggs, narrow, 64);
        Status e2 = first_error(op2);
        CHECK(e2 && e2->Code == BYDB_ENOTSUP && e2->Msg.find("default/code") != std::string::npos, "two stored keys at MaxKeyValues 256: ENOTSUP");
        ScanSpec desc = scan;
        desc.OrderDesc = true;
        GPUScanAgg opd(ctx, input_schema(), {1, 2}, aggs, desc, 64);
        Status ed = first_error(opd);
        CHECK(ed && ed->Code == BYDB_ENOTSUP, "stored keys with OrderDesc: ENOTSUP");
    }
    bydb_part_release(ctx, h);
    bydb_part_image_free(img);
    bydb_shutdown(ctx);
    std::printf("%s\n", fails ? "FAILED" : "OK full");
    return fails ? 1 : 0;
}

/* A plain C99 caller of bydb_scan_partials_keyed through include/bydb_gpu.h alone, the way a data node's cgo shim answers the
 * liaison's partial request for a group-by on a stored tag.  It builds a synthetic part (include/bydb_synth.h), runs the call
 * grouped by argv[1] ("region": a string tag, or "code": an int64 tag) and prints every row as
 *     row <group> <key bytes in hex> <Partial.Value per aggregate> | <Partial.Count per aggregate>
 * (int64 words as %lld, float64 words as %.17g), then "OK".  Without a GPU it prints "init refused" and "OK". */
#include <inttypes.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "bydb_gpu.h"
#include "bydb_synth.h"

int main(int argc, char **argv) {
    int (*f_rows)(bydb_ctx *, const bydb_query *, const bydb_group_key *, bydb_keyed_partial_rows *) = bydb_scan_partials_keyed;
    int (*f_red)(bydb_ctx *, const bydb_query *, const bydb_group_key *, int32_t, bydb_keyed_partial_rows *) = bydb_scan_reduce_keyed_partials;
    void (*f_free)(bydb_ctx *, bydb_keyed_partial_rows *) = bydb_keyed_partial_rows_free;
    (void)f_red;
    const char *tag = argc > 1 ? argv[1] : "region";
    const uint32_t vt = strcmp(tag, "code") == 0 ? BYDB_VT_INT64 : 0;

    bydb_ctx *ctx = NULL;
    int rc = bydb_init(NULL, &ctx);
    if (rc != 0) {
        printf("init refused: %d %s\nOK\n", rc, bydb_last_error());
        return ctx == NULL ? 0 : 1;
    }
    bydb_synth_field fld[2] = {{"latency", BYDB_SYN_F_LATENCY, 0}, {"calls", BYDB_SYN_I_FLUCT, 0}};
    bydb_synth_spec sp;
    memset(&sp, 0, sizeof sp);
    sp.n_series = 6; sp.n_points = 3000; sp.sid0 = 1; sp.sid_step = 1; sp.t0 = 1700000000000000000LL; sp.t_step = 60000000000LL;
    sp.n_fields = 2; sp.fields = fld; sp.region_values = 5; sp.region_run = 8; sp.code_tag = 1; sp.threads = 1; sp.seed = 11;
    bydb_part_image *img = NULL;
    if (bydb_synth_part(&sp, &img) != 0 || !img) { printf("synth failed\n"); return 1; }
    bydb_file files[16];
    const uint32_t nf = bydb_part_image_n_files(img);
    if (nf > 16) return 1;
    for (uint32_t i = 0; i < nf; ++i) {
        files[i].name = bydb_part_image_file_name(img, i);
        files[i].data = bydb_part_image_file_data(img, i, &files[i].len);
    }
    bydb_part_files pf = {nf, files};
    bydb_part_h h = 0;
    if (bydb_part_register(ctx, 77, &pf, &h) != 0) { printf("register failed: %s\n", bydb_last_error()); return 1; }

    bydb_agg aggs[5] = {{"latency", BYDB_AGG_SUM, 0}, {"latency", BYDB_AGG_MEAN, 0}, {"latency", BYDB_AGG_MAX, 0},
                        {"calls", BYDB_AGG_MIN, 0}, {"calls", BYDB_AGG_COUNT, 0}};
    uint64_t sids[6] = {1, 2, 3, 4, 5, 6};
    int32_t grp[6] = {0, 1, 0, 2, 1, 0};
    bydb_query q;
    memset(&q, 0, sizeof q);
    q.parts = &h; q.n_parts = 1; q.series_ids = sids; q.n_series = 6; q.series_group = grp; q.n_groups = 3;
    q.aggs = aggs; q.n_aggs = 5;
    q.tmin = sp.t0 + 100 * sp.t_step; q.tmax = sp.t0 + 2500 * sp.t_step;
    bydb_group_key gk = {"default", tag, 0, vt};
    bydb_keyed_partial_rows r;
    if (f_rows(ctx, &q, &gk, &r) != 0) { printf("scan_partials_keyed failed: %s\n", bydb_last_error()); return 1; }
    printf("rows %d keys %d aggs %d\n", r.base.n_rows, r.n_keys, r.base.n_aggs);
    for (int32_t i = 0; i < r.base.n_rows; ++i) {
        printf("row %d ", r.base.group_id[i]);
        const uint32_t a0 = r.key_off[r.key_id[i]], a1 = r.key_off[r.key_id[i] + 1];
        for (uint32_t b = a0; b < a1; ++b) printf("%02x", r.key_bytes[b]);
        for (int pass = 0; pass < 2; ++pass) {
            printf(pass ? " |" : "");
            for (int32_t a = 0; a < r.base.n_aggs; ++a) {
                const size_t o = (size_t)i * (size_t)r.base.n_aggs + (size_t)a;
                if (r.base.is_float[a]) printf(" %.17g", pass ? r.base.cnt_f64[o] : r.base.val_f64[o]);
                else printf(" %" PRId64, pass ? r.base.cnt_i64[o] : r.base.val_i64[o]);
            }
        }
        printf("\n");
    }
    f_free(ctx, &r);
    bydb_part_release(ctx, h);
    bydb_part_image_free(img);
    bydb_shutdown(ctx);
    printf("OK\n");
    return 0;
}

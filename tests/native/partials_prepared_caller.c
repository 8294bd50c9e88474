/* A plain C99 caller of the prepared map-phase forms through include/bydb_gpu.h alone, the way a data node's cgo shim keeps a
 * prepared plan per pushed-down query: bydb_scan_partials_prepared (a group-by on series tags) and
 * bydb_scan_partials_keyed_prepared (a group-by on the stored tag "region") are run six times each on a synthetic part, and every
 * answer is compared, bit for bit, with the unprepared calls (bydb_scan_partials into device memory + bydb_partials_rows, and
 * bydb_scan_partials_keyed).  Replays must move nothing host-to-device and read back exactly the header's d2h_bytes.  Prints
 * "OK" at the end; without a GPU it prints "init refused" and "OK". */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "bydb_gpu.h"
#include "bydb_synth.h"

/* the two CUDA runtime calls the shim uses to own the partial table (libcudart) */
extern int cudaMalloc(void **p, size_t n);
extern int cudaFree(void *p);

#define RUNS 6

static int same_rows(const bydb_partial_rows *a, const bydb_partial_rows *b) {
    if (a->n_rows != b->n_rows || a->n_aggs != b->n_aggs) return 0;
    const size_t n = (size_t)a->n_rows, w = n * (size_t)a->n_aggs;
    if (n && memcmp(a->group_id, b->group_id, n * 4) != 0) return 0;
    if (a->n_aggs && memcmp(a->is_float, b->is_float, (size_t)a->n_aggs) != 0) return 0;
    if (w && (memcmp(a->val_i64, b->val_i64, w * 8) || memcmp(a->val_f64, b->val_f64, w * 8) || memcmp(a->cnt_i64, b->cnt_i64, w * 8) ||
              memcmp(a->cnt_f64, b->cnt_f64, w * 8)))
        return 0;
    return 1;
}

static int same_keys(const bydb_keyed_partial_rows *a, const bydb_keyed_partial_rows *b) {
    if (a->n_keys != b->n_keys || !same_rows(&a->base, &b->base)) return 0;
    for (int32_t i = 0; i < a->base.n_rows; ++i) {
        const uint32_t a0 = a->key_off[a->key_id[i]], a1 = a->key_off[a->key_id[i] + 1];
        const uint32_t b0 = b->key_off[b->key_id[i]], b1 = b->key_off[b->key_id[i] + 1];
        if (a1 - a0 != b1 - b0 || memcmp(a->key_bytes + a0, b->key_bytes + b0, a1 - a0) != 0) return 0;
    }
    return 1;
}

int main(void) {
    int (*f_plain)(bydb_ctx *, bydb_prepared *, bydb_partial_rows *, bydb_stats *) = bydb_scan_partials_prepared;
    int (*f_keyed)(bydb_ctx *, bydb_prepared_keyed *, bydb_keyed_partial_rows *) = bydb_scan_partials_keyed_prepared;
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
    if (bydb_part_register(ctx, 78, &pf, &h) != 0) { printf("register failed: %s\n", bydb_last_error()); return 1; }

    bydb_agg aggs[5] = {{"latency", BYDB_AGG_SUM, 0}, {"latency", BYDB_AGG_MEAN, 0}, {"latency", BYDB_AGG_MAX, 0},
                        {"calls", BYDB_AGG_MIN, 0}, {"calls", BYDB_AGG_MEAN, 0}};
    uint64_t sids[6] = {1, 2, 3, 4, 5, 6};
    int32_t grp[6] = {0, 3, 0, 2, 3, 0};  /* group 1 never appears */
    bydb_query q;
    memset(&q, 0, sizeof q);
    q.parts = &h; q.n_parts = 1; q.series_ids = sids; q.n_series = 6; q.series_group = grp; q.n_groups = 4;
    q.aggs = aggs; q.n_aggs = 5;
    q.tmin = sp.t0 + 100 * sp.t_step; q.tmax = sp.t0 + 2500 * sp.t_step;
    const uint64_t F = 2, A = 5;

    /* ---- plain: the shim's unprepared sequence against the prepared handle */
    bydb_partials_layout_t lay;
    void *d_table = NULL;
    if (bydb_partials_layout(&q, &lay) != 0 || cudaMalloc(&d_table, lay.total_bytes) != 0) { printf("table failed\n"); return 1; }
    bydb_prepared *pq = NULL;
    if (bydb_query_prepare(ctx, &q, &pq) != 0) { printf("prepare failed: %s\n", bydb_last_error()); return 1; }
    for (int run = 0; run < RUNS; ++run) {
        bydb_stats st0, st;
        bydb_partial_rows want, got;
        if (bydb_scan_partials(ctx, &q, d_table, lay.total_bytes, NULL, &st0) != 0 ||
            bydb_partials_rows(ctx, &q, d_table, lay.total_bytes, NULL, &want) != 0) {
            printf("unprepared plain failed: %s\n", bydb_last_error());
            return 1;
        }
        if (f_plain(ctx, pq, &got, &st) != 0) { printf("prepared plain failed: %s\n", bydb_last_error()); return 1; }
        if (!same_rows(&got, &want) || want.n_rows != 3 || st.rows_matched != st0.rows_matched) { printf("plain run %d differs\n", run); return 1; }
        const uint64_t d2h = 256 + 8 + 8 * F + (uint64_t)got.n_rows * (8 + 16 * A);
        if (run >= 1 && (st.h2d_bytes != 0 || st.d2h_bytes != d2h || st.kernel_launches != st0.kernel_launches + 4)) {
            printf("plain run %d stats: h2d %llu d2h %llu launches %u\n", run, (unsigned long long)st.h2d_bytes, (unsigned long long)st.d2h_bytes,
                   st.kernel_launches);
            return 1;
        }
        printf("plain run %d rows %d d2h %llu\n", run, got.n_rows, (unsigned long long)st.d2h_bytes);
        bydb_partial_rows_free(ctx, &want);
        bydb_partial_rows_free(ctx, &got);
    }
    bydb_query_release(ctx, pq);
    cudaFree(d_table);

    /* ---- keyed: grouped by (series group, region) */
    bydb_group_key gk = {"default", "region", 0, 0};
    bydb_prepared_keyed *kq = NULL;
    if (bydb_query_prepare_keyed(ctx, &q, &gk, &kq) != 0) { printf("prepare_keyed failed: %s\n", bydb_last_error()); return 1; }
    for (int run = 0; run < RUNS; ++run) {
        bydb_keyed_partial_rows want, got;
        if (bydb_scan_partials_keyed(ctx, &q, &gk, &want) != 0) { printf("unprepared keyed failed: %s\n", bydb_last_error()); return 1; }
        if (f_keyed(ctx, kq, &got) != 0) { printf("prepared keyed failed: %s\n", bydb_last_error()); return 1; }
        if (!same_keys(&got, &want) || want.base.n_rows == 0 || got.stats.rows_matched != want.stats.rows_matched) {
            printf("keyed run %d differs\n", run);
            return 1;
        }
        const uint64_t d2h = 256 * (uint64_t)got.n_keys + 8 + 8 * F + (uint64_t)got.base.n_rows * (8 + 16 * A);
        if (run >= 1 && (got.stats.h2d_bytes != 0 || got.stats.d2h_bytes != d2h || got.stats.kernel_launches != want.stats.kernel_launches)) {
            printf("keyed run %d stats: h2d %llu d2h %llu launches %u\n", run, (unsigned long long)got.stats.h2d_bytes,
                   (unsigned long long)got.stats.d2h_bytes, got.stats.kernel_launches);
            return 1;
        }
        printf("keyed run %d rows %d keys %d d2h %llu\n", run, got.base.n_rows, got.n_keys, (unsigned long long)got.stats.d2h_bytes);
        bydb_keyed_partial_rows_free(ctx, &want);
        bydb_keyed_partial_rows_free(ctx, &got);
    }
    bydb_query_release_keyed(ctx, kq);
    bydb_part_release(ctx, h);
    bydb_part_image_free(img);
    bydb_shutdown(ctx);
    printf("OK\n");
    return 0;
}

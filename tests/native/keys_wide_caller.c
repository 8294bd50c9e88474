/* A plain C99 caller of bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide through their declared prototypes, linked against
 * libbydbgpu.so the way a cgo shim links it.  Without arguments it runs the argument refusals that need no device; with a path to
 * a part directory written by the project's writer (files named as on disk), it also runs a two-tag query on device 0 and prints
 * its rows as "group key_a key_b rows". */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "bydb_gpu.h"

static int expect(const char *what, int rc, int want) {
    if (rc != want) {
        printf("%s: %d, want %d (%s)\n", what, rc, want, bydb_last_error());
        return 1;
    }
    return 0;
}

static int refusals(bydb_ctx *ctx) {
    bydb_query q;
    memset(&q, 0, sizeof q);
    bydb_group_key k[5];
    memset(k, 0, sizeof k);
    const char *tags[5] = {"a", "b", "c", "d", "e"};
    for (int i = 0; i < 5; ++i) {
        k[i].family = "default";
        k[i].tag = tags[i];
    }
    bydb_group_keys keys;
    memset(&keys, 0, sizeof keys);
    keys.keys = k;
    bydb_keys_result r;
    bydb_keys_partial_rows pr;
    int bad = 0;
    keys.n_keys = 2;
    bad |= expect("NULL ctx", bydb_scan_agg_keys_wide(NULL, &q, &keys, &r), BYDB_EINVAL);
    bad |= expect("NULL out", bydb_scan_partials_keys_wide(ctx, &q, &keys, NULL), BYDB_EINVAL);
    if (!ctx) return bad;
    keys.n_keys = 1;
    bad |= expect("one key", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), BYDB_EINVAL);
    keys.n_keys = 5;
    bad |= expect("five keys", bydb_scan_partials_keys_wide(ctx, &q, &keys, &pr), BYDB_EINVAL);
    keys.n_keys = 3;
    k[2].tag = "a";
    bad |= expect("a tag twice", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), BYDB_EINVAL);
    k[2].tag = "c";
    k[1].max_values = 8;
    bad |= expect("a key's own cap", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), BYDB_EINVAL);
    k[1].max_values = 0;
    keys.max_values = 65537;
    bad |= expect("cap above 65,536", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), BYDB_EINVAL);
    keys.max_values = 0;
    k[0].value_type = BYDB_VT_FLOAT64;
    bad |= expect("float key", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), BYDB_EINVAL);
    bydb_keys_result_free(ctx, NULL);
    bydb_keys_partial_rows_free(ctx, NULL);
    return bad;
}

int main(int argc, char **argv) {
    if (refusals(NULL)) return 1;
    if (argc < 2) {
        printf("OK\n");
        return 0;
    }
    bydb_cfg cfg;
    memset(&cfg, 0, sizeof cfg);
    bydb_ctx *ctx = NULL;
    if (expect("init", bydb_init(&cfg, &ctx), 0)) return 1;
    if (refusals(ctx)) return 1;
    /* argv[1..]: name=path of each part file */
    bydb_file files[16];
    void *bufs[16];
    int nf = 0;
    for (int i = 1; i < argc && nf < 16; ++i, ++nf) {
        char *eq = strchr(argv[i], '=');
        *eq = 0;
        FILE *fp = fopen(eq + 1, "rb");
        fseek(fp, 0, SEEK_END);
        long n = ftell(fp);
        fseek(fp, 0, SEEK_SET);
        bufs[nf] = malloc(n ? (size_t)n : 1);
        if (fread(bufs[nf], 1, (size_t)n, fp) != (size_t)n) return 1;
        fclose(fp);
        files[nf].name = argv[i];
        files[nf].data = (const uint8_t *)bufs[nf];
        files[nf].len = (uint64_t)n;
    }
    bydb_part_files pf = {(uint32_t)nf, files};
    bydb_part_h h = 0;
    if (expect("register", bydb_part_register(ctx, 1, &pf, &h), 0)) return 1;
    uint64_t sids[2] = {1, 2};
    bydb_agg agg = {"v", BYDB_AGG_COUNT, 0};
    bydb_query q;
    memset(&q, 0, sizeof q);
    q.n_parts = 1;
    q.parts = &h;
    q.n_series = 2;
    q.series_ids = sids;
    q.n_groups = 1;
    q.tmin = INT64_MIN;
    q.tmax = INT64_MAX;
    q.n_aggs = 1;
    q.aggs = &agg;
    bydb_group_key k[2] = {{"default", "a", 0, BYDB_VT_STR}, {"default", "b", 0, BYDB_VT_INT64}};
    bydb_group_keys keys = {2, 0, k};
    bydb_keys_result r;
    if (expect("two-tag query", bydb_scan_agg_keys_wide(ctx, &q, &keys, &r), 0)) return 1;
    for (int i = 0; i < r.base.n_rows; ++i) {
        const int32_t ea = r.key_id[2 * i], eb = r.key_id[2 * i + 1];
        long long b = 0;
        memcpy(&b, r.key_bytes + r.key_off[eb], 8);
        printf("%d %.*s %lld %lld\n", r.base.group_id[i], (int)(r.key_off[ea + 1] - r.key_off[ea]), (const char *)r.key_bytes + r.key_off[ea], b,
               (long long)r.base.rows[i]);
    }
    printf("tuples %d tags %u\n", r.n_tuples, r.n_tags);
    bydb_keys_result_free(ctx, &r);
    bydb_part_release(ctx, h);
    bydb_shutdown(ctx);
    for (int i = 0; i < nf; ++i) free(bufs[i]);
    printf("OK\n");
    return 0;
}

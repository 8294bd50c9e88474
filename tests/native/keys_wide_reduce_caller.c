/* A plain C99 caller of the tuple collective (bydb_keys_wide_reduce_slot_bytes, bydb_scan_reduce_keys_wide and
 * bydb_scan_reduce_keys_wide_partials) through their declared prototypes, linked against libbydbgpu.so the way a cgo shim links
 * it.  Host only: NULL arguments are refused with BYDB_EINVAL before anything touches a device, and the slot of a two-tag query is
 * sized without one. */
#include <stdio.h>
#include <string.h>

#include "bydb_gpu.h"

int main(void) {
    int (*f_slot)(const bydb_query *, const bydb_group_keys *, uint64_t, uint64_t *) = bydb_keys_wide_reduce_slot_bytes;
    int (*f_agg)(bydb_ctx *, const bydb_query *, const bydb_group_keys *, int32_t, bydb_keys_result *) = bydb_scan_reduce_keys_wide;
    int (*f_part)(bydb_ctx *, const bydb_query *, const bydb_group_keys *, int32_t, bydb_keys_partial_rows *) =
        bydb_scan_reduce_keys_wide_partials;
    uint64_t sid = 1;
    bydb_agg agg;
    memset(&agg, 0, sizeof agg);
    agg.field = "latency";
    agg.func = BYDB_AGG_SUM;
    bydb_query q;
    memset(&q, 0, sizeof q);
    q.series_ids = &sid;
    q.n_series = 1;
    q.aggs = &agg;
    q.n_aggs = 1;
    q.tmin = 0;
    q.tmax = 1;
    bydb_group_key k[2];
    memset(k, 0, sizeof k);
    k[0].family = "default";
    k[0].tag = "endpoint";
    k[1].family = "default";
    k[1].tag = "status";
    k[1].value_type = BYDB_VT_INT64;
    bydb_group_keys keys;
    memset(&keys, 0, sizeof keys);
    keys.n_keys = 2;
    keys.max_values = 4096;
    keys.keys = k;
    uint64_t bytes = 0;
    int rc;
    if ((rc = f_slot(NULL, &keys, 16, &bytes)) != BYDB_EINVAL) { printf("slot, NULL query: %d\n", rc); return 1; }
    if ((rc = f_slot(&q, NULL, 16, &bytes)) != BYDB_EINVAL) { printf("slot, NULL keys: %d\n", rc); return 1; }
    if ((rc = f_slot(&q, &keys, 16, NULL)) != BYDB_EINVAL) { printf("slot, NULL out: %d\n", rc); return 1; }
    if ((rc = f_slot(&q, &keys, 16, &bytes)) != 0 || bytes == 0) { printf("slot: %d %llu\n", rc, (unsigned long long)bytes); return 1; }
    bydb_keys_result res;
    bydb_keys_partial_rows rows;
    if ((rc = f_agg(NULL, &q, &keys, 0, &res)) != BYDB_EINVAL) { printf("NULL ctx: %d\n", rc); return 1; }
    if ((rc = f_agg(NULL, &q, &keys, 0, NULL)) != BYDB_EINVAL) { printf("NULL out: %d\n", rc); return 1; }
    if ((rc = f_part(NULL, &q, &keys, 0, &rows)) != BYDB_EINVAL) { printf("partials, NULL ctx: %d\n", rc); return 1; }
    if ((rc = f_part(NULL, &q, &keys, 0, NULL)) != BYDB_EINVAL) { printf("partials, NULL out: %d\n", rc); return 1; }
    printf("OK\n");
    return 0;
}

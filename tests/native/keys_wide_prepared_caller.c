/* A plain C99 caller of the prepared tuple group-by (bydb_query_prepare_keys_wide, bydb_scan_agg_keys_prepared,
 * bydb_scan_partials_keys_prepared) through its declared prototypes, linked against libbydbgpu.so the way a cgo shim links it.
 * Host only: a NULL context or out pointer is refused with BYDB_EINVAL before anything touches a device. */
#include <stdio.h>
#include <string.h>

#include "bydb_gpu.h"

int main(void) {
    int (*f_prep)(bydb_ctx *, const bydb_query *, const bydb_group_keys *, bydb_prepared_keyed **) = bydb_query_prepare_keys_wide;
    int (*f_agg)(bydb_ctx *, bydb_prepared_keyed *, bydb_keys_result *) = bydb_scan_agg_keys_prepared;
    int (*f_part)(bydb_ctx *, bydb_prepared_keyed *, bydb_keys_partial_rows *) = bydb_scan_partials_keys_prepared;
    void (*f_rel)(bydb_ctx *, bydb_prepared_keyed *) = bydb_query_release_keyed;
    bydb_query q;
    memset(&q, 0, sizeof q);
    bydb_group_key tags[2];
    memset(tags, 0, sizeof tags);
    tags[0].family = "default";
    tags[0].tag = "endpoint";
    tags[1].family = "default";
    tags[1].tag = "status";
    tags[1].value_type = BYDB_VT_INT64;
    bydb_group_keys keys;
    keys.n_keys = 2;
    keys.max_values = 4096;
    keys.keys = tags;
    bydb_prepared_keyed *h = (bydb_prepared_keyed *)1;
    int rc = f_prep(NULL, &q, &keys, &h);
    if (rc != BYDB_EINVAL) { printf("NULL ctx: %d\n", rc); return 1; }
    if (f_prep(NULL, &q, &keys, NULL) != BYDB_EINVAL) { printf("NULL out\n"); return 1; }
    bydb_keys_result r;
    bydb_keys_partial_rows pr;
    if (f_agg(NULL, NULL, &r) != BYDB_EINVAL) { printf("agg: NULL ctx\n"); return 1; }
    if (f_part(NULL, NULL, &pr) != BYDB_EINVAL) { printf("partials: NULL ctx\n"); return 1; }
    f_rel(NULL, NULL);  /* releasing no handle is a no-op */
    printf("OK\n");
    return 0;
}

/* A plain C99 caller of bydb_query_prepare_keyed_wide through its declared prototype, linked against libbydbgpu.so the way a cgo
 * shim links it.  Host only: a NULL context or out pointer is refused with BYDB_EINVAL before anything touches a device. */
#include <stdio.h>
#include <string.h>

#include "bydb_gpu.h"

int main(void) {
    int (*f_prep)(bydb_ctx *, const bydb_query *, const bydb_group_key *, bydb_prepared_keyed **) = bydb_query_prepare_keyed_wide;
    int (*f_agg)(bydb_ctx *, bydb_prepared_keyed *, bydb_keyed_result *) = bydb_scan_agg_keyed_prepared;
    int (*f_part)(bydb_ctx *, bydb_prepared_keyed *, bydb_keyed_partial_rows *) = bydb_scan_partials_keyed_prepared;
    void (*f_rel)(bydb_ctx *, bydb_prepared_keyed *) = bydb_query_release_keyed;
    (void)f_agg; (void)f_part;
    bydb_query q;
    memset(&q, 0, sizeof q);
    bydb_group_key key;
    memset(&key, 0, sizeof key);
    key.family = "default";
    key.tag = "endpoint";
    key.max_values = 4096;
    bydb_prepared_keyed *h = (bydb_prepared_keyed *)1;
    int rc = f_prep(NULL, &q, &key, &h);
    if (rc != BYDB_EINVAL) { printf("NULL ctx: %d\n", rc); return 1; }
    if (f_prep(NULL, &q, &key, NULL) != BYDB_EINVAL) { printf("NULL out\n"); return 1; }
    f_rel(NULL, NULL);  /* releasing no handle is a no-op */
    printf("OK\n");
    return 0;
}

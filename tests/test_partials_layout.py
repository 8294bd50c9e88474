"""bydb_partials_layout (host only, no GPU): the partial table's offsets and counts, restated from bydb_gpu.h's layout.

A table for G groups and F distinct aggregated fields is, in 8-byte words: sum_f64 [GF] | max_f64 [GF] | negmin_f64 [GF] |
sum_i64 [GF] | cnt [GF] | rows [G] | max_i64 [GF] | notmin_i64 [GF] | coltype [F].  The four ranges a caller all-reduces are
the float sums, the float maxima (max, -min), the int64 sums (sum, count, rows) and the int64 maxima (max, ~min, coltype).
F counts each field once, however many aggregations name it.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O


def _layout(q):
    from bydb_b200.capi import _Layout, _check, _mk_query, load_library
    keep = []
    lay = _Layout()
    _check(load_library().bydb_partials_layout(C.byref(_mk_query(q, keep)), C.byref(lay)))
    return {k: getattr(lay, k) for k, _ in _Layout._fields_}


@pytest.mark.parametrize("G,aggs", [
    (1, [("a", O.AGG_SUM)]),
    (1, [("a", O.AGG_SUM), ("a", O.AGG_MIN), ("a", O.AGG_MAX), ("a", O.AGG_MEAN), ("a", O.AGG_COUNT)]),
    (2, [("a", O.AGG_MEAN), ("b", O.AGG_MAX)]),
    (7, [("x", O.AGG_MIN), ("y", O.AGG_SUM), ("x", O.AGG_MAX), ("z", O.AGG_COUNT), ("y", O.AGG_MEAN)]),
    (33, [("f", O.AGG_COUNT), ("f", O.AGG_SUM)]),
    (2049, [(f"f{k % 5}", O.AGG_SUM) for k in range(9)]),
    (5, [(f"f{k}", O.AGG_MAX) for k in range(8)]),
])
def test_partials_layout_restated(bydb, G, aggs):
    NS = max(G, 3)
    sids = np.arange(1, NS + 1, dtype=np.uint64)
    groups = (np.arange(NS) % G).astype(np.int32) if G > 1 else None
    lay = _layout(bydb.Query([], sids, aggs, series_group=groups, n_groups=G))
    F =len(dict.fromkeys(f for f, _ in aggs))
    GF = G * F
    assert lay == dict(total_bytes=8 * (7 * GF + G + F),
                       off_sum_f64=0, n_sum_f64=GF,
                       off_max_f64=8 * GF, n_max_f64=2 * GF,
                       off_sum_i64=8 * 3 * GF, n_sum_i64=2 * GF + G,
                       off_max_i64=8 * (5 * GF + G), n_max_i64=2 * GF + F)
    # the four ranges tile the table without gaps: the last one ends at the table's end
    assert lay["off_max_f64"] == lay["off_sum_f64"] + 8 * lay["n_sum_f64"]
    assert lay["off_sum_i64"] == lay["off_max_f64"] + 8 * lay["n_max_f64"]
    assert lay["off_max_i64"] == lay["off_sum_i64"] + 8 * lay["n_sum_i64"]
    assert lay["total_bytes"] == lay["off_max_i64"] + 8 * lay["n_max_i64"]

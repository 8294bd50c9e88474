"""The query shape every partial-table call shares, and the HBM budget of a failed mailbox export.

bydb_partials_layout (host logic, no device) refuses a query with more than 8 distinct aggregated fields, like every scan does:
no scan can produce a partial table for it.  A failed mailbox allocation in bydb_comm_export gives its budget reservation back,
so the context can still admit parts afterwards.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import build_part, grid


def _layout(bydb, q):
    from bydb_b200.capi import _Layout, _mk_query, load_library
    keep = []
    lay = _Layout()
    L = load_library()
    rc = L.bydb_partials_layout(C.byref(_mk_query(q, keep)), C.byref(lay))
    return rc, {k: getattr(lay, k) for k, _ in _Layout._fields_}, (L.bydb_last_error() or b"").decode()


def test_partials_layout_refuses_more_than_eight_fields(bydb):
    G, NS = 3, 7
    sids = np.arange(1, NS + 1, dtype=np.uint64)
    groups = (np.arange(NS) % G).astype(np.int32)
    # 8 distinct fields over 9 aggregations: accepted, with the table layout of bydb_gpu.h (G x F words per range)
    aggs = [(f"f{i}", O.AGG_SUM) for i in range(8)] + [("f3", O.AGG_MAX)]
    rc, lay, _ = _layout(bydb, bydb.Query([], sids, aggs, series_group=groups, n_groups=G))
    assert rc == 0
    F = 8
    GF = G * F
    assert lay == dict(total_bytes=8 * (7 * GF + G + F), off_sum_f64=0, n_sum_f64=GF, off_max_f64=8 * GF, n_max_f64=2 * GF,
                       off_sum_i64=24 * GF, n_sum_i64=2 * GF + G, off_max_i64=8 * (5 * GF + G), n_max_i64=2 * GF + F)
    # a ninth distinct field: refused like every scan refuses it
    rc, _, msg = _layout(bydb, bydb.Query([], sids, aggs + [("f8", O.AGG_COUNT)], series_group=groups, n_groups=G))
    assert rc == bydb.capi.EINVAL
    assert "too many distinct aggregated fields" in msg


@pytest.mark.gpu
def test_failed_mailbox_export_gives_its_budget_back(bydb):
    import torch

    max_table_bytes, max_ranks = 1 << 32, 64
    mailbox = 4096 + 2 * max_ranks * max_table_bytes  # control page + 2 parities x 64 slots of 4 GiB: 512 GiB and 4 KiB
    assert mailbox > torch.cuda.get_device_properties(0).total_memory
    rng = np.random.default_rng(11)
    sids, ts, ver = grid(4, 500)
    part = build_part(sids, ts, ver, [("latency", O.VT_FLOAT64, np.round(rng.normal(30, 6, sids.size), 2), None),
                                      ("calls", O.VT_INT64, rng.integers(0, 1000, sids.size), None)])
    aggs = [("latency", O.AGG_SUM), ("calls", O.AGG_MAX)]
    q = lambda h: bydb.Query([h], np.unique(sids), aggs)  # noqa: E731
    with bydb.Context(device=0) as free:
        want = free.scan_agg(q(free.register_part(1, part.files())))
    with bydb.Context(device=0, hbm_budget_bytes=mailbox + 64) as ctx:
        # within the budget, but no device holds it: the allocation fails (an error code, not a device fault)
        with pytest.raises(bydb.BydbError) as ei:
            ctx.comm_export(max_table_bytes, max_ranks)
        assert ei.value.code == bydb.capi.ENOMEM
        h = ctx.register_part(1, part.files())  # needs the mailbox's reservation back
        got = ctx.scan_agg(q(h))
    assert got.group_id.tolist() == want.group_id.tolist()
    assert got.rows.tolist() == want.rows.tolist()
    assert got.val_f64.view(np.uint64).tolist() == want.val_f64.view(np.uint64).tolist()
    assert got.val_i64.tolist() == want.val_i64.tolist()

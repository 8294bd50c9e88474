"""bydb_keyed_wide_reduce_slot_bytes (host only, no GPU): the mailbox slot of the wide keyed collective, restated from its layout.

A rank that found V key values and C present composite groups writes into its slot, each region starting on a 256-byte boundary:
a 256-byte header (query fingerprint, V, C), the value lengths [V] u32, the values [V][64], the series' spans [NS][2] i64, the
composite groups' (series group, value id) pairs [C][2] i32, their first series [C] u32, and their partial table of C groups
(bydb_gpu.h's layout: 7 * C * F + C words, then F coltype words).  The slot to export is that layout at V = max_values (0 = 64)
and C = max_present.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O


def up(o):
    return (o + 255) // 256 * 256


def slot_bytes(F, NS, V, Cp):
    o = up(256 + V * 4)              # header | lens
    o = up(o + V * 64)               # values
    o = up(o + NS * 16)              # spans
    o = up(o + Cp * 8)               # pairs
    o = up(o + Cp * 4)               # first series
    return o + 8 * (7 * Cp * F + Cp + F)


AGG_SETS = {
    1: [("a", O.AGG_SUM)],
    3: [("a", O.AGG_MAX), ("b", O.AGG_MIN), ("c", O.AGG_SUM), ("a", O.AGG_COUNT)],
    8: [(f, O.AGG_SUM) for f in "abcdefgh"],
}


@pytest.mark.parametrize("F", sorted(AGG_SETS))
@pytest.mark.parametrize("NS,G", [(1, 1), (12, 4), (1000, 7)])
@pytest.mark.parametrize("max_values", [0, 1, 256, 257, 65536])
@pytest.mark.parametrize("max_present", [0, 1, 1 << 20])
def test_slot_bytes_restated(bydb, F, NS, G, max_values, max_present):
    aggs = AGG_SETS[F]
    sids = np.arange(1, NS + 1, dtype=np.uint64)
    groups = (np.arange(NS) % G).astype(np.int32) if G > 1 else None
    q = bydb.Query([], sids, aggs, series_group=groups, n_groups=G)
    want = slot_bytes(F, NS, max_values or 64, max_present)
    for vt in (0, bydb.VT_STR, bydb.VT_INT64):
        assert bydb.keyed_wide_reduce_slot_bytes(q, "default", "k", max_values, max_present, vt) == want


def test_slot_bytes_grow_with_every_field(bydb):
    """F from 1 to 8 fields, the groups of the query do not enter the slot (only present composite groups do)"""
    sids = np.arange(1, 6, dtype=np.uint64)
    for F in range(1, 9):
        aggs = [("f%d" % c, O.AGG_SUM) for c in range(F)] + [("f0", O.AGG_COUNT)]
        for G in (1, 5):
            q = bydb.Query([], sids, aggs, series_group=(np.arange(5) % G).astype(np.int32), n_groups=G)
            assert bydb.keyed_wide_reduce_slot_bytes(q, "default", "k", 300, 1000) == slot_bytes(F, 5, 300, 1000)


def test_slot_bytes_refusals(bydb):
    q = bydb.Query([], np.arange(1, 3, dtype=np.uint64), [("a", O.AGG_SUM)])
    for mv, vt in [(65537, 0), (0, 3), (0, 7)]:
        with pytest.raises(bydb.BydbError) as e:
            bydb.keyed_wide_reduce_slot_bytes(q, "default", "k", mv, 10, vt)
        assert e.value.code == -22
    # NULL query, NULL key, NULL output
    L = bydb.capi.load_library()
    keep: list = []
    cq = bydb.capi._mk_query(q, keep)
    gk = bydb.capi._GroupKey(b"default", b"k", 0, 0)
    out = C.c_uint64()
    assert L.bydb_keyed_wide_reduce_slot_bytes(None, C.byref(gk), 1, C.byref(out)) == -22
    assert L.bydb_keyed_wide_reduce_slot_bytes(C.byref(cq), None, 1, C.byref(out)) == -22
    assert L.bydb_keyed_wide_reduce_slot_bytes(C.byref(cq), C.byref(gk), 1, None) == -22
    # the per-value form's cap (256) does not bind the wide form
    assert L.bydb_keyed_wide_reduce_slot_bytes(C.byref(cq), C.byref(gk), 1, C.byref(out)) == 0
    assert out.value == slot_bytes(1, 2, 64, 1)

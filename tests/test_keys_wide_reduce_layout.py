"""bydb_keys_wide_reduce_slot_bytes (host only, no GPU): the mailbox slot of the tuple collective, restated from its layout.

A rank that found V_t values of each of its K tags, T tuples and C present composite groups writes into its slot, each region
starting on a 256-byte boundary: a 256-byte header (query fingerprint, T, C, then K and each V_t), the value lengths [sum V_t] u32,
the values [sum V_t][64] (tag 0's, then tag 1's, ...), the series' spans [NS][2] i64, the composite groups' (series group, tuple id)
pairs [C][2] i32, their first series [C] u32, their partial table of C groups (7 * C * F + C words, then F coltype words), and last
the tuple codes [T] u64.  The slot to export is that layout at T = V_t = max_values (0 = 64) and C = max_present.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O


def up(o):
    return (o + 255) // 256 * 256


def slot_bytes(F, NS, K, max_values, Cp):
    cap = max_values or 64
    n_vals = K * cap
    o = up(256 + n_vals * 4)         # header | lens
    o = up(o + n_vals * 64)          # values
    o = up(o + NS * 16)              # spans
    o = up(o + Cp * 8)               # pairs
    o = up(o + Cp * 4)               # first series
    o = up(o + 8 * (7 * Cp * F + Cp + F))  # table
    return o + cap * 8               # tuple codes


AGG_SETS = {
    1: [("a", O.AGG_SUM)],
    3: [("a", O.AGG_MAX), ("b", O.AGG_MIN), ("c", O.AGG_SUM), ("a", O.AGG_COUNT)],
    8: [(f, O.AGG_SUM) for f in "abcdefgh"],
}


def tags(bydb, K, mixed=True):
    return [("default", "t%d" % t, bydb.VT_INT64 if mixed and t % 2 else 0) for t in range(K)]


@pytest.mark.parametrize("K", [2, 3, 4])
@pytest.mark.parametrize("F", sorted(AGG_SETS))
@pytest.mark.parametrize("NS,G", [(1, 1), (12, 4), (1000, 7)])
@pytest.mark.parametrize("max_values", [0, 1, 256, 257, 65536])
@pytest.mark.parametrize("max_present", [0, 1, 1 << 20])
def test_slot_bytes_restated(bydb, K, F, NS, G, max_values, max_present):
    sids = np.arange(1, NS + 1, dtype=np.uint64)
    groups = (np.arange(NS) % G).astype(np.int32) if G > 1 else None
    q = bydb.Query([], sids, AGG_SETS[F], series_group=groups, n_groups=G)
    want = slot_bytes(F, NS, K, max_values, max_present)
    for mixed in (False, True):
        assert bydb.keys_wide_reduce_slot_bytes(q, tags(bydb, K, mixed), max_values, max_present) == want


def test_slot_bytes_grow_with_every_field_and_tag(bydb):
    """F from 1 to 8 fields and K from 2 to 4 tags; the groups of the query do not enter the slot (only present groups do)"""
    sids = np.arange(1, 6, dtype=np.uint64)
    for F in range(1, 9):
        aggs = [("f%d" % c, O.AGG_SUM) for c in range(F)] + [("f0", O.AGG_COUNT)]
        for G in (1, 5):
            q = bydb.Query([], sids, aggs, series_group=(np.arange(5) % G).astype(np.int32), n_groups=G)
            sizes = [bydb.keys_wide_reduce_slot_bytes(q, tags(bydb, K), 300, 1000) for K in (2, 3, 4)]
            assert sizes == [slot_bytes(F, 5, K, 300, 1000) for K in (2, 3, 4)]
            assert sizes[0] < sizes[1] < sizes[2]


def test_slot_bytes_refusals(bydb):
    """bydb_scan_agg_keys_wide's argument refusals, with its codes, and NULL arguments"""
    q = bydb.Query([], np.arange(1, 3, dtype=np.uint64), [("a", O.AGG_SUM)])
    two = tags(bydb, 2)
    bad = [
        (two[:1], 0),                                           # one tag
        (tags(bydb, 5), 0),                                     # five tags
        ([two[0], two[0]], 0),                                  # the same tag twice
        ([two[0], ("default", "t1", 3)], 0),                    # a bad value type
        (two, 65537),                                           # max_values above 65,536
    ]
    for keys, mv in bad:
        with pytest.raises(bydb.BydbError) as e:
            bydb.keys_wide_reduce_slot_bytes(q, keys, mv, 10)
        assert e.value.code == -22, (keys, mv)
    L = bydb.capi.load_library()
    keep: list = []
    cq = bydb.capi._mk_query(q, keep)
    gks = bydb.capi._group_keys(two, 0, keep)
    out = C.c_uint64()
    assert L.bydb_keys_wide_reduce_slot_bytes(None, C.byref(gks), 1, C.byref(out)) == -22
    assert L.bydb_keys_wide_reduce_slot_bytes(C.byref(cq), None, 1, C.byref(out)) == -22
    assert L.bydb_keys_wide_reduce_slot_bytes(C.byref(cq), C.byref(gks), 1, None) == -22
    # a key's own max_values must be 0 (the cap is the tuple's)
    arr = (bydb.capi._GroupKey * 2)(bydb.capi._GroupKey(b"default", b"t0", 5, 0), bydb.capi._GroupKey(b"default", b"t1", 0, 0))
    own = bydb.capi._GroupKeys(2, 0, arr)
    assert L.bydb_keys_wide_reduce_slot_bytes(C.byref(cq), C.byref(own), 1, C.byref(out)) == -22
    # the wide cap binds, not the per-value one
    assert L.bydb_keys_wide_reduce_slot_bytes(C.byref(cq), C.byref(gks), 1, C.byref(out)) == 0
    assert out.value == slot_bytes(1, 2, 2, 0, 1)

"""bydb_keyed_reduce_slot_bytes (host only, no GPU): the mailbox slot of a keyed collective, restated from its layout.

A rank that found V key values writes into its slot, each region starting on a 256-byte boundary: a 256-byte header (query
fingerprint, V), the value lengths [V] u32, the values [V][64], the passes' column types [V * F] i64, Kts [V * NS] i64, Krow
[V * NS] u32, the series' spans [NS][2] i64, and the composite partial table of V * G groups (bydb_gpu.h's layout: 7 * G * F + G
words, then F coltype words).  The slot to export is that layout at V = max_values (0 = 64).
"""
import numpy as np
import pytest

from oracle import oracle as O


def up(o):
    return (o + 255) // 256 * 256


def slot_bytes(G, F, NS, V):
    o = up(256 + V * 4)              # header | lens
    o = up(o + V * 64)               # values
    o = up(o + V * F * 8)            # column types
    o = up(o + V * NS * 8)           # Kts
    o = up(o + V * NS * 4)           # Krow
    o = up(o + NS * 16)              # spans
    return o + 8 * (7 * V * G * F + V * G + F)


@pytest.mark.parametrize("G,aggs,NS,max_values", [
    (1, [("a", O.AGG_SUM)], 1, 1),
    (4, [("a", O.AGG_SUM), ("b", O.AGG_MEAN), ("a", O.AGG_COUNT)], 12, 0),
    (7, [("a", O.AGG_MAX), ("b", O.AGG_MIN), ("c", O.AGG_SUM)], 1000, 256),
    (300, [("a", O.AGG_COUNT)], 5, 4),
])
def test_slot_bytes_restated(bydb, G, aggs, NS, max_values):
    sids = np.arange(1, NS + 1, dtype=np.uint64)
    groups = (np.arange(NS) % G).astype(np.int32) if G > 1 else None
    q = bydb.Query([], sids, aggs, series_group=groups, n_groups=G)
    F = len(dict.fromkeys(f for f, _ in aggs))
    want = slot_bytes(G, F, NS, max_values or 64)
    assert bydb.keyed_reduce_slot_bytes(q, "default", "k", max_values) == want
    assert bydb.keyed_reduce_slot_bytes(q, "default", "k", max_values, bydb.VT_INT64) == want


def test_slot_bytes_refusals(bydb):
    q = bydb.Query([], np.arange(1, 3, dtype=np.uint64), [("a", O.AGG_SUM)])
    for mv, vt in [(257, 0), (0, 3)]:
        with pytest.raises(bydb.BydbError) as e:
            bydb.keyed_reduce_slot_bytes(q, "default", "k", mv, vt)
        assert e.value.code == -22

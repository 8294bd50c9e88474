"""Map-phase rows of a group-by on a stored tag (bydb_scan_partials_keyed / bydb_scan_reduce_keyed_partials, DESIGN.md 4.6): what a
data node answers when the liaison pushes a stored-tag group-by down with agg_return_partial.

keyed_partial_rows_kernel runs one thread per (row j < n_present, aggregate) behind key_order_kernel / key_perm_kernel, reads
composite group perm[j] straight from the unpermuted V x G table and writes [group | key id | Partial.Value[A] | Partial.Count[A]]
through partial_words, the rule bydb_partials_rows uses for a plain group.  Checked here:
  - one node against the oracle (string and int64 keys, nulls, a group that met only nulls, one that never met the column, COUNT of
    a float field): per function the oracle's keyed query over the node's parts, MEAN = SUM's value + COUNT's count, rows in the
    oracle's keyed order; and against bydb_scan_agg_keyed on the same context: Val() of the partials (function.go restated, MEAN
    quirks included) equals its values bit for bit;
  - the liaison: reduceAccumulator.Combine + Val() restated over several nodes' rows (series shards, time shards, a value only
    one node holds, a node that selects no block) equals the oracle's keyed query over all parts -- the model itself is pinned
    without a GPU on rows the oracle makes;
  - the emission boundaries (no, one, every composite group present; G x V around 256 x 32 and above 2^20; 1 and 32
    aggregations), d2h_bytes against the header's formula, the refusals of bydb_scan_agg_keyed, the collective (3 ranks as
    threads, mixed with bydb_scan_reduce_keyed and plain collectives) and a plain C caller through the header alone.
"""
import dataclasses
import os
import shutil
import subprocess
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, to_gpu_query
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, F, I, Series
from tests.test_gpu_keyed import FAM, KT, build_keyed, mk, std_fields
from tests.test_gpu_keyed_int64 import KX, int_tag, twin
from tests.test_gpu_keyed_reduce import R, Case, Ranks, plain_ok, quiet, series_case, slot_for, time_case  # noqa: F401
from tests.test_gpu_masks import I64_MAX, I64_MIN

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENOMEM, EINVAL, ENOTSUP = -12, -22, -95
FNS = (SUM, COUNT, MIN, MAX, MEAN)
AGGS10 = [(f, fn) for f in ("i", "f") for fn in FNS]
_pid = [500_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def _wrap(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


# ------------------------------------------------------------------ data
S_POOL = [b"a", b"b", b"c", None, b"d", b"e", b"z", b"y"]
I_POOL = [5, -7, 1 << 40, None, 0, 3, 99, -1]


def node_parts(int64):
    """two time-disjoint parts of one node.  Part A: series 1 (its `c` rows have null fields: that group met only nulls), series 2
    over two blocks with nil keys and 10% null cells, series 3 with one value.  Part B, 20000 rows later, carries no `i` field:
    series 1's `z` there never met `i`, series 4 adds `a` (already met on another series of its group) and `y`."""
    pool = I_POOL if int64 else S_POOL
    rng = np.random.default_rng(3)

    def series(sid, idx, row0, nulls=None, only_f=False):
        cells = [pool[k] for k in idx]
        f = std_fields(sid, len(cells))
        nl = np.zeros(len(cells), bool) if nulls is None else nulls
        fields = {"f": (F, f["f"][1], nl)} if only_f else {"i": (I, f["i"][1], nl), "f": (F, f["f"][1], nl)}
        tags = {KT: int_tag(cells), KX: twin(cells)} if int64 else {KT: cells}
        return Series(sid, fields, tags, row0=row0)

    i1 = [k % 3 for k in range(400)]
    a = [series(1, i1, 0, np.array([k == 2 for k in i1])),
         series(2, [int(x) for x in rng.choice([0, 1, 3, 4], 9000)], 0, rng.random(9000) < 0.1),
         series(3, [5] * 50, 0)]
    b = [series(1, [6] * 30, 20000, only_f=True), series(4, [0, 7] * 30, 20000, only_f=True)]
    return [(build_keyed(a), a), (build_keyed(b), b)]


GID = {1: 0, 2: 1, 3: 0, 4: 1}


# ------------------------------------------------------------------ the oracle's node rows, the liaison, Val()
def oracle_rows(oq, aggs, okey):
    """the rows a node answers with, made from the oracle's keyed queries: Partial.Value per function (MEAN: SUM's), Partial.Count
    (MEAN: COUNT's), typed like the field (COUNT of a float field is a float).  The oracle takes at most 30 aggregations: it runs
    the distinct ones.  okey: the string tag to key on, or None for the group key oq already names."""
    uniq = list(dict.fromkeys(aggs))
    key = {} if okey is None else dict(group_key=(FAM, okey))
    own = {fn: O.run_query(dataclasses.replace(oq, aggs=[(f, fn) for f, _ in uniq], **key)) for fn in (SUM, COUNT, MIN, MAX)}
    s = own[SUM]
    n, A = s.group_id.size, len(aggs)
    col = [uniq.index(x) for x in aggs]
    isf = np.array([bool(s.is_float[col[a]]) for a in range(A)])
    out = dict(group_id=s.group_id.astype(np.int32), key=list(s.key), is_float=isf, val_i64=np.zeros((n, A), np.int64),
               val_f64=np.zeros((n, A), np.float64), cnt_i64=np.zeros((n, A), np.int64), cnt_f64=np.zeros((n, A), np.float64))
    for a, (f, fn) in enumerate(aggs):
        src, u = own[SUM if fn == MEAN else fn], col[a]
        v = src.val_i64[:, u] if fn == COUNT else (src.val_f64[:, u] if isf[a] else src.val_i64[:, u])
        (out["val_f64"] if isf[a] else out["val_i64"])[:, a] = v
        if fn == MEAN:
            (out["cnt_f64"] if isf[a] else out["cnt_i64"])[:, a] = own[COUNT].val_i64[:, u]
    return out


def cell(rows, i, a):
    isf = rows["is_float"][a]
    return ((rows["val_f64"] if isf else rows["val_i64"])[i, a].item(), (rows["cnt_f64"] if isf else rows["cnt_i64"])[i, a].item())


def val(fn, isf, v, c):
    """Val() of a (combined) Partial (pkg/query/aggregation/function.go): MEAN divides (Go's integer division truncates) and
    reports 1 below 1; everything else is the value"""
    if fn != MEAN:
        return v
    if c == 0:
        return 0.0 if isf else 0
    q = v / c if isf else abs(v) // c * (1 if v >= 0 else -1)
    return (1.0 if isf else 1) if q < 1 else q


def liaison(node_rows, aggs):
    """reduceAccumulator.Combine over the nodes' rows keyed by (series group, key bytes), then Val(); int64 sums wrap"""
    acc = {}
    for rows in node_rows:
        for i, ck in enumerate(zip(rows["group_id"].tolist(), rows["key"])):
            e = acc.setdefault(ck, [None] * len(aggs))
            for a, (_, fn) in enumerate(aggs):
                v, c = cell(rows, i, a)
                if e[a] is None:
                    e[a] = (v, c)
                    continue
                pv, pc = e[a]
                isf = rows["is_float"][a]
                if fn in (SUM, COUNT, MEAN):
                    e[a] = (pv + v, pc + c) if isf else (_wrap(pv + v), _wrap(pc + c))
                else:
                    e[a] = (max(pv, v) if fn == MAX else min(pv, v), 0)
    isf = next((r["is_float"] for r in node_rows if r["group_id"].size), None)
    return {ck: [val(fn, bool(isf[a]), *e[a]) for a, (_, fn) in enumerate(aggs)] for ck, e in acc.items()}


def check_liaison(got, want, aggs, ctx):
    """the liaison's answer against the oracle's keyed query over all parts"""
    exp = {ck: [want.val_f64[i, a] if want.is_float[a] else want.val_i64[i, a] for a in range(len(aggs))]
           for i, ck in enumerate(zip(want.group_id.tolist(), want.key))}
    assert set(got) == set(exp), f"{ctx}: composite groups {sorted(set(got) ^ set(exp))[:8]}"
    for ck, vals in exp.items():
        for a, ((f, fn), w) in enumerate(zip(aggs, vals)):
            g = got[ck][a]
            if isinstance(g, float) and fn in (SUM, MEAN):
                assert abs(g - w) <= 1e-9 * max(abs(w), 1.0), f"{ctx}: {ck} agg {a} ({f},{fn}): {g!r} vs {w!r}"
            elif isinstance(g, float) and fn != COUNT:
                assert _bits(g) == _bits(w), f"{ctx}: {ck} agg {a} ({f},{fn}): {g!r} vs {w!r} (bit-exact)"
            else:
                assert g == w, f"{ctx}: {ck} agg {a} ({f},{fn}): {g!r} vs {w!r}"


def check_rows(got, want, aggs, ctx, rel=1e-12):
    """one node's rows: (group, key) sequence, typing, Partial.Count exactly; int64 values exactly, float MIN / MAX / COUNT bit
    for bit, float sums within `rel` relative (the float fields here hold positive values only: |sum| is the sum of |x|)"""
    seq = list(zip(got["group_id"].tolist(), got["key"]))
    assert seq == list(zip(want["group_id"].tolist(), want["key"])), f"{ctx}: row order {seq[:8]} vs {list(zip(want['group_id'].tolist(), want['key']))[:8]}"
    if not seq:
        return
    assert got["is_float"].tolist() == list(want["is_float"]), f"{ctx}: typing"
    for a, (f, fn) in enumerate(aggs):
        isf = bool(got["is_float"][a])
        assert (got["cnt_f64"] if isf else got["cnt_i64"])[:, a].tolist() == (want["cnt_f64"] if isf else want["cnt_i64"])[:, a].tolist(), \
            f"{ctx}: Partial.Count of agg {a}"
        if not isf:
            assert got["val_i64"][:, a].tolist() == want["val_i64"][:, a].tolist(), f"{ctx}: agg {a} ({f},{fn})"
        elif fn in (MIN, MAX, COUNT):
            assert got["val_f64"][:, a].view(np.uint64).tolist() == np.asarray(want["val_f64"][:, a], np.float64).view(np.uint64).tolist(), \
                f"{ctx}: agg {a} ({f},{fn}) bit for bit"
        else:
            for i, ck in enumerate(seq):
                x, y = float(got["val_f64"][i, a]), float(want["val_f64"][i, a])
                assert abs(x - y) <= rel * abs(y), f"{ctx}: {ck} agg {a} ({f},{fn}): {x!r} vs {y!r}"


def same_as_keyed(rows, res, aggs, ctx):
    """Val() of the partial rows equals bydb_scan_agg_keyed's values bit for bit, row for row"""
    assert list(zip(rows["group_id"].tolist(), rows["key"])) == list(zip(res.group_id.tolist(), res.key)), f"{ctx}: order vs keyed"
    for i in range(res.group_id.size):
        for a, (f, fn) in enumerate(aggs):
            v, c = cell(rows, i, a)
            mine = val(fn, bool(rows["is_float"][a]), v, c)
            theirs = res.value(i, a)
            ok = _bits(mine) == _bits(theirs) if isinstance(theirs, float) else mine == theirs
            assert ok, f"{ctx}: row {i} agg {a} ({f},{fn}): Val {mine!r}, keyed {theirs!r}"


def d2h_formula(n_keys, cap, F_, A, n_rows):
    up = lambda x: (x + 255) // 256 * 256  # noqa: E731
    disc = 256 + up(64 * cap) + up(4 * cap)
    return disc if n_keys == 0 else disc + 256 * n_keys + 8 + 8 * F_ + n_rows * (8 + 16 * A)


def table_bytes(G, V, F_):
    return 8 * (G * V * (7 * F_ + 1) + F_)


class Node:
    """parts registered on one context; queries run as partial rows, as the finalised keyed call and through the oracle"""

    def __init__(self, bydb, ctx, parts, gid, int64=False):
        self.bydb, self.ctx, self.parts, self.gid, self.int64 = bydb, ctx, parts, gid, int64
        self.series = [s for _, ss in parts for s in ss]

    def __enter__(self):
        pid = _next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, (p, _) in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def oq(self, aggs, preds=(), tmin=I64_MIN, tmax=I64_MAX, gid=None):
        gid = gid or self.gid
        sids = np.array(sorted(gid), dtype=np.uint64)
        return O.Query([p for p, _ in self.parts], sids, list(aggs), groups=np.array([gid[int(s)] for s in sids], np.int32),
                       n_groups=max(gid.values()) + 1, tmin=tmin, tmax=tmax, preds=list(preds))

    def rows(self, oq, max_values=256):
        q = to_gpu_query(self.bydb, self.handles, oq)
        return self.ctx.scan_partials_keyed(q, FAM, KT, max_values, self.bydb.VT_INT64 if self.int64 else 0)

    def check(self, aggs, ctx, gid=None, max_values=256, **kw):
        oq = self.oq(aggs, gid=gid, **kw)
        got = self.rows(oq, max_values)
        want = oracle_rows(oq, aggs, KX if self.int64 else KT)
        check_rows(got, want, aggs, ctx, 1e-9)
        res = self.ctx.scan_agg_keyed(to_gpu_query(self.bydb, self.handles, oq), FAM, KT, max_values, self.bydb.VT_INT64 if self.int64 else 0)
        same_as_keyed(got, res, aggs, ctx)
        assert got["n_keys"] == res.n_keys, ctx
        st, rs = got["stats"], res.stats
        assert (st.rows_scanned, st.rows_matched, st.blocks_scanned) == (rs.rows_scanned, rs.rows_matched, rs.blocks_scanned), f"{ctx}: counters"
        F_ = len(dict.fromkeys(f for f, _ in aggs))
        assert st.d2h_bytes == d2h_formula(got["n_keys"], max_values or 64, F_, len(aggs), len(got["key"])), f"{ctx}: d2h {st.d2h_bytes}"
        return got


# ------------------------------------------------------------------ 1. one node against the oracle
@gpu
@pytest.mark.parametrize("int64", [False, True], ids=["string", "int64"])
def test_one_node_against_the_oracle(bydb, gpu_ctx, int64):
    with Node(bydb, gpu_ctx, node_parts(int64), GID, int64) as n:
        got = n.check(AGGS10, "all rows")
        keys = dict(zip(zip(got["group_id"].tolist(), got["key"]), range(len(got["key"]))))
        k = (lambda v: struct.pack("<q", v)) if int64 else (lambda v: v)
        c, z = (k(I_POOL[2]), k(I_POOL[6])) if int64 else (b"c", b"z")
        i_min, i_max = AGGS10.index(("i", MIN)), AGGS10.index(("i", MAX))
        row = keys[(0, c)]                                  # met only null cells: the N-typed sentinels
        assert (got["val_i64"][row, i_min], got["val_i64"][row, i_max]) == (I64_MAX, I64_MIN)
        row = keys[(0, z)]                                  # never met the column: the zero value
        assert (got["val_i64"][row, i_min], got["val_i64"][row, i_max]) == (0, 0)
        assert got["is_float"][AGGS10.index(("f", COUNT))], "COUNT of a float field is N-typed"
        n.check(AGGS10, "time cut", tmin=T0 + 100 * STEP, tmax=T0 + 20010 * STEP)
        n.check([("f", MEAN), ("i", SUM)], "one group per series", gid={1: 0, 2: 1, 3: 2, 4: 3})


# ------------------------------------------------------------------ 2. the liaison
def liaison_cases():
    sc, tc = series_case(), time_case()
    # a fourth node whose part holds none of the query's series: it selects no block (0 rows, 0 keys)
    empty = build_keyed([mk(900, [b"a", b"b"] * 10)])
    return [("series", sc, KT, KT), ("time", tc, KT, KX)], empty


def liaison_check(case, okey, node_rows, label, kw):
    aggs = kw.get("aggs", AGGS10)
    want = O.run_query(dataclasses.replace(case.oquery([p for s in case.shards for p in s], **kw), group_key=(FAM, okey)))
    check_liaison(liaison(node_rows, aggs), want, aggs, label)


LIAISON_QUERIES = [dict(aggs=AGGS10), dict(aggs=[("f", MEAN), ("i", MAX)], tmin=T0 + 50 * STEP, tmax=T0 + 700 * STEP)]


def test_liaison_model_on_oracle_rows():
    """the liaison model itself, without a GPU: node rows the oracle makes, folded, give the oracle's answer over all parts"""
    cases, empty = liaison_cases()
    for label, case, _, okey in cases:
        for kw in LIAISON_QUERIES:
            nodes = [oracle_rows(case.oquery(case.shards[r], **kw), kw["aggs"], okey) for r in range(R)]
            nodes.append(oracle_rows(case.oquery([empty], **kw), kw["aggs"], okey))
            assert nodes[-1]["group_id"].size == 0
            assert sum(r["group_id"].size for r in nodes) > len({ck for r in nodes for ck in zip(r["group_id"].tolist(), r["key"])}), \
                f"{label}: some group must span nodes"
            liaison_check(case, okey, nodes, f"oracle/{label}/{kw}", kw)


@gpu
def test_liaison_over_gpu_nodes(bydb, gpu_ctx):
    """three data nodes (series shards, then time shards, with values only one node holds) and one that selects no block"""
    cases, empty = liaison_cases()
    for label, case, key, okey in cases:
        vt = bydb.VT_INT64 if okey == KX else 0
        pid = _next_pid()
        hs = [[gpu_ctx.register_part(pid + 10 * r + i, p.files()) for i, p in enumerate(case.shards[r])] for r in range(R)]
        he = gpu_ctx.register_part(pid + 99, empty.files())
        try:
            for kw in LIAISON_QUERIES:
                nodes = []
                for r in range(R):
                    oq = case.oquery(case.shards[r], **kw)
                    rows = gpu_ctx.scan_partials_keyed(to_gpu_query(bydb, hs[r], oq), FAM, key, 256, vt)
                    check_rows(rows, oracle_rows(oq, kw["aggs"], okey), kw["aggs"], f"{label}/node {r}", 1e-9)
                    nodes.append(rows)
                none = gpu_ctx.scan_partials_keyed(to_gpu_query(bydb, [he], case.oquery([empty], **kw)), FAM, key, 256, vt)
                assert none["group_id"].size == 0 and none["n_keys"] == 0 and not none["key"]
                nodes.append(none)
                liaison_check(case, okey, nodes, f"gpu/{label}/{kw}", kw)
        finally:
            for h in [h for hh in hs for h in hh] + [he]:
                gpu_ctx.release_part(h)


# ------------------------------------------------------------------ 3. emission boundaries
POOL256 = [b""] + [b"v%03d" % i for i in range(255)]


def full_part(G):
    """G series (one per group), each showing all 256 values: every composite group present"""
    ss = [mk(sid, [POOL256[(k + 7 * sid) % 256] for k in range(256 + sid % 5)]) for sid in range(1, G + 1)]
    return [(build_keyed(ss), ss)]


@gpu
def test_no_one_and_every_composite_group(bydb, gpu_ctx):
    with Node(bydb, gpu_ctx, node_parts(False), GID) as n:
        # V > 0, n_present = 0: a predicate removes every row
        got = n.check([("i", SUM)], "nothing left", preds=[O.Pred(FAM, KT, O.OP_EQ, b"nope")])
        assert got["n_keys"] > 0 and got["group_id"].size == 0
    # n_present = 1 at the last composite index (V - 1) * G + G - 1: every series holds one value of its own; the series of the
    # value last in the key table is put into the last group, and a predicate keeps only that value
    ss = [mk(sid, [b"u%d" % sid] * (10 + sid)) for sid in range(1, 6)]
    with Node(bydb, gpu_ctx, [(build_keyed(ss), ss)], {s: s - 1 for s in range(1, 6)}) as n:
        last = n.check([("i", SUM)], "one value per series")["key_table"][-1]
        holder = int(last[1:])
        others = [s for s in range(1, 6) if s != holder]
        gid = {**{s: i for i, s in enumerate(others)}, holder: len(others)}
        got = n.check([("f", MAX), ("i", COUNT)], "last composite", gid=gid, preds=[O.Pred(FAM, KT, O.OP_EQ, last)])
        assert list(zip(got["group_id"].tolist(), got["key"])) == [(len(others), last)]
    for G in (31, 32, 33):
        with Node(bydb, gpu_ctx, full_part(G), {s: s - 1 for s in range(1, G + 1)}) as n:
            for aggs in ([("i", SUM)], [(("i", "f")[k % 2], FNS[k % 5]) for k in range(32)]):
                got = n.check(aggs, f"every group present, G={G}, A={len(aggs)}")
                assert got["n_keys"] == 256 and got["group_id"].size == 256 * G


@gpu
def test_more_than_2_20_composite_groups(bydb, gpu_ctx):
    """G = 4097 groups x 256 values = 1 048 832 composite groups, 4 present per group: the rows cross PCIe, the table does not"""
    G = 4097
    ss = [mk(sid, [POOL256[(4 * sid + k) % 256] for k in range(4)]) for sid in range(1, G + 1)]
    with Node(bydb, gpu_ctx, [(build_keyed(ss), ss)], {s: s - 1 for s in range(1, G + 1)}) as n:
        got = n.check([("i", SUM), ("f", MIN), ("i", MEAN)], "GP > 2^20")
        assert got["n_keys"] == 256 and got["group_id"].size == 4 * G
        assert got["stats"].d2h_bytes < table_bytes(G, 256, 2) // 100


# ------------------------------------------------------------------ 4. refusals
@gpu
def test_refusals_are_those_of_the_keyed_call(bydb, gpu_ctx):
    a = [mk(1, [b"a", b"b", b"c"] * 20), mk(2, [b"d"] * 30)]
    over = [mk(3, [b"a"] * 40, row0=10)]                                    # overlaps part A in time
    mix = [Series(5, {"i": (F, np.linspace(1.5, 9.5, 20), None), "f": (F, np.ones(20), None)}, {KT: [b"a"] * 20}, row0=50000)]
    parts = [build_keyed(a), build_keyed(over), build_keyed(mix)]
    pid = _next_pid()
    hs = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(parts)]
    try:
        def q(handles, sids, preds=()):
            sids = np.array(sids, np.uint64)
            return bydb.Query(handles, sids, [("i", SUM), ("f", MAX)], series_group=np.zeros(sids.size, np.int32), n_groups=1,
                              preds=list(preds))
        seven = [bydb.Pred(FAM, KT, bydb.OP_NE, b"x%d" % k) for k in range(8)]
        cases = [("overlap", q(hs[:2], [1, 2, 3]), KT, 256, 0, ENOTSUP), ("max_values", q(hs[:1], [1, 2]), KT, 2, 0, ENOMEM),
                 ("8 predicates", q(hs[:1], [1, 2], seven), KT, 256, 0, ENOTSUP), ("key type", q(hs[:1], [1, 2]), KT, 256, 99, EINVAL),
                 ("int64 on a string tag", q(hs[:1], [1, 2]), KT, 256, bydb.VT_INT64, EINVAL),
                 ("type mix", q([hs[0], hs[2]], [1, 2, 5]), KT, 256, 0, EINVAL)]
        ok = q(hs[:1], [1, 2])
        want = gpu_ctx.scan_partials_keyed(ok, FAM, KT)
        for label, qq, key, mv, vt, code in cases:
            for call in (gpu_ctx.scan_agg_keyed, gpu_ctx.scan_partials_keyed):
                with pytest.raises(bydb.BydbError) as e:
                    call(qq, FAM, key, mv, vt)
                assert e.value.code == code, (label, call.__name__, e.value)
            again = gpu_ctx.scan_partials_keyed(ok, FAM, KT)
            assert again["key"] == want["key"] and again["val_i64"].tolist() == want["val_i64"].tolist(), label
        # seven predicates of its own are accepted
        assert gpu_ctx.scan_partials_keyed(q(hs[:1], [1, 2], seven[:7]), FAM, KT)["n_keys"] == 4
    finally:
        for h in hs:
            gpu_ctx.release_part(h)


# ------------------------------------------------------------------ 5. the collective
def whole_rows(bydb, gpu_ctx, case, key, vt, kw):
    pid = _next_pid()
    whole = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(case.whole)]
    try:
        return gpu_ctx.scan_partials_keyed(to_gpu_query(bydb, whole, case.oquery(case.whole, **kw)), FAM, key, 256, vt)
    finally:
        for h in whole:
            gpu_ctx.release_part(h)


def collective(bydb, gpu_ctx, ranks, case, root, key, vt, okey, mixed=False, **kw):
    aggs = kw.get("aggs", AGGS10)
    kw = {**kw, "aggs": aggs}
    qs = [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], **kw)) for r in range(R)]

    def body(r):
        if mixed and r != root:
            return ranks.ctxs[r].scan_reduce_keyed(qs[r], FAM, key, root=root, max_values=256, value_type=vt)
        return ranks.ctxs[r].scan_reduce_keyed_partials(qs[r], FAM, key, root=root, max_values=256, value_type=vt)
    res, codes = ranks.run(body)
    assert codes == [0] * R, codes
    got = res[root]
    label = f"root{root}/mixed={mixed}/{kw}"
    check_rows(got, whole_rows(bydb, gpu_ctx, case, key, vt, kw), aggs, label)
    check_rows(got, oracle_rows(case.oquery([p for s in case.shards for p in s], **kw), aggs, okey), aggs, label + "/oracle", 1e-9)
    for r in range(R):
        if r != root:
            rows = res[r].group_id.size if mixed else res[r]["group_id"].size
            nk = res[r].n_keys if mixed else res[r]["n_keys"]
            assert rows == 0 and nk == 0, f"{label}: rank {r}"
    return got


@gpu
def test_collective_partial_rows(bydb, gpu_ctx, quiet):  # noqa: F811
    sc, tc = series_case(), time_case()
    ranks = Ranks(bydb, max(slot_for(bydb, sc), slot_for(bydb, tc)))
    try:
        for it in range(6):
            root = it % R
            ranks.register(sc.shards)
            collective(bydb, gpu_ctx, ranks, sc, root, KT, 0, KT, mixed=it % 2 == 1)
            plain_ok(bydb, gpu_ctx, ranks, sc, root)
            ranks.register(tc.shards)
            collective(bydb, gpu_ctx, ranks, tc, (root + 1) % R, KT, bydb.VT_INT64, KX, aggs=[("f", MEAN), ("i", MIN)], mixed=it % 3 == 0)
            # a finalising keyed collective in between: the same slots, the epochs in step
            qs = [to_gpu_query(bydb, ranks.hs[r], tc.oquery(tc.shards[r])) for r in range(R)]
            res, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed(qs[r], FAM, KT, root=root, max_values=256, value_type=bydb.VT_INT64))
            assert codes == [0] * R and res[root].group_id.size > 0
        # a rank that passes another query: the root refuses, the next collective answers
        ranks.register(sc.shards)
        qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r], aggs=[("i", SUM)] if r == 1 else AGGS10)) for r in range(R)]
        _, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed_partials(qs[r], FAM, KT, root=0, max_values=256))
        assert codes == [EINVAL, 0, 0], codes
        collective(bydb, gpu_ctx, ranks, sc, 0, KT, 0, KT)
    finally:
        ranks.close()


# ------------------------------------------------------------------ 6. plain C
def _caller(tmp_path, bydb):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "keyed_partials_caller"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "keyed_partials_caller.c"), "-L", lib_dir, "-lbydbgpu", "-Wl,-rpath," + lib_dir])
    return exe


def test_c_caller_builds_against_the_header(tmp_path, bydb):
    out = subprocess.run([str(_caller(tmp_path, bydb))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr


@gpu
@pytest.mark.parametrize("tag", ["region", "code"])
def test_c_caller_prints_the_wrappers_rows(tmp_path, bydb, gpu_ctx, tag):
    out = subprocess.run([str(_caller(tmp_path, bydb)), tag], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "init refused" not in out.stdout, out.stdout + out.stderr
    synth = __import__("bydb_b200.synth").synth
    img = synth.synth_part(6, 3000, [("latency", synth.F_LATENCY), ("calls", synth.I_FLUCT)], region_values=5, region_run=8,
                           code_tag=True, seed=11, threads=1)
    t0, step = 1_700_000_000_000_000_000, 60_000_000_000
    h = gpu_ctx.register_part(_next_pid(), img.files())
    try:
        q = bydb.Query([h], np.arange(1, 7, dtype=np.uint64), [("latency", SUM), ("latency", MEAN), ("latency", MAX), ("calls", MIN), ("calls", COUNT)],
                       series_group=np.array([0, 1, 0, 2, 1, 0], np.int32), n_groups=3, tmin=t0 + 100 * step, tmax=t0 + 2500 * step)
        r = gpu_ctx.scan_partials_keyed(q, "default", tag, 0, bydb.VT_INT64 if tag == "code" else 0)
    finally:
        gpu_ctx.release_part(h)
    A = 5
    lines = [f"rows {len(r['key'])} keys {r['n_keys']} aggs {A}"]
    for i, (g, k) in enumerate(zip(r["group_id"].tolist(), r["key"])):
        parts = []
        for names in (("val_f64", "val_i64"), ("cnt_f64", "cnt_i64")):
            parts.append("".join(" %.17g" % r[names[0]][i, a] if r["is_float"][a] else " %d" % r[names[1]][i, a] for a in range(A)))
        lines.append(f"row {g} {k.hex()}{parts[0]} |{parts[1]}")
    printed = [ln for ln in out.stdout.splitlines() if ln.startswith(("rows ", "row "))]
    assert len(r["key"]) > 5 and printed == lines, "\n".join(printed[:6] + ["--"] + lines[:6])

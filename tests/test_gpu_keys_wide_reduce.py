"""Group-by on a tuple of 2..4 stored tags across ranks (bydb_scan_reduce_keys_wide / _partials, DESIGN.md 5): R = 3 ranks as
threads, one context each on device r % device_count.  Every rank passes the same query and keys but its parts.  Each answer of
the root is checked
  - against bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide on one context over one part holding every rank's rows: rows
    identified by their key bytes, group ids and rows in the same order, int64 values and min / max exactly, floats within 1e-9
    relative, n_tuples, and each tag's table as a set;
  - for the pair (string a, int64 b), against the wide keyed collective (itself oracle-pinned) on the injective twin tag c: the
    same rows in the same order, values bit for bit, n_tuples == n_keys; and against the oracle through the twin;
  - against the header's formulas: rows_matched summed over the ranks, every other rank's empty answer and own counters, and
    d2h_bytes / kernel_launches of the non-root ranks and the root.
"""
import dataclasses

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0, assert_parity, to_gpu_query
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, Series
from tests.test_gpu_keyed import FAM, build_keyed, std_fields
from tests.test_gpu_keyed_reduce import EINVAL, ENOMEM, ENOTSUP, R, Case, Ranks, _next_pid, plain_ok, quiet  # noqa: F401
from tests.test_gpu_keyed_wide_reduce import sort_launches
from tests.test_gpu_keys_wide import INT, STR, comp, int_tag, le, twin
from tests.test_gpu_masks import I64_MAX, I64_MIN

gpu = pytest.mark.gpu

PAIR = [(FAM, "a", STR), (FAM, "b", INT)]
THREE = [(FAM, "d", STR), (FAM, "b", INT), (FAM, "a", STR)]
FOUR = [(FAM, "e", INT), (FAM, "a", STR), (FAM, "d", STR), (FAM, "b", INT)]
TAG_TYPES = {"a": STR, "b": INT, "d": STR, "e": INT, "z": STR}
B_POOL = [0, -1, 7, I64_MIN, I64_MAX, 3, 42]


def std_cells(rank, sid, x):
    """the tags of row x of series sid on `rank`: a string a with nils and a value of this rank only, an int64 b with nils and
    the extremes, d and e that follow a and b (so a block holds at most 7 * 8 * 2 tuples), z for predicates"""
    a = None if (x + sid) % 11 == 0 else b"only%d" % rank if x % 17 == 5 else b"a%d" % ((x // 3 + sid) % 5)
    bi = (x * 5 + sid) % 7
    b = None if (x + 2 * sid) % 13 == 0 else B_POOL[bi]
    return {"a": a, "b": b, "d": b"d%d" % ((x // 7) % 2), "e": None if b is None else bi % 3 - 1, "z": b"z%d" % (x % 4)}


def tag_columns(cells):
    cols = {}
    for name, ty in TAG_TYPES.items():
        vals = [c[name] for c in cells]
        cols[name] = int_tag(vals) if ty == INT else vals
    cols["c"] = twin([comp(c["a"], STR) for c in cells], [comp(c["b"], INT) for c in cells])
    return cols


def build_case(pieces, gid, cells=std_cells):
    """pieces: (rank, sid, row0, n), each a contiguous window of one series' rows.  -> Case whose rank r holds one part with its
    pieces and whose `whole` is one part with every series in full"""
    by_sid = {}
    for r, sid, row0, n in pieces:
        by_sid.setdefault(sid, []).append((row0, n, r))
    per_rank, whole = [[] for _ in range(R)], []
    for sid, ps in sorted(by_sid.items()):
        ps.sort()
        lo = ps[0][0]
        total = ps[-1][0] + ps[-1][1] - lo
        f = std_fields(sid, total)
        all_cells = [None] * total
        for row0, n, r in ps:
            a = row0 - lo
            cs = [cells(r, sid, row0 + i) for i in range(n)]
            all_cells[a:a + n] = cs
            per_rank[r].append(Series(sid, {k: (vt, v[a:a + n], None) for k, (vt, v, _) in f.items()}, tag_columns(cs), row0=row0))
        whole.append(Series(sid, f, tag_columns(all_cells), row0=lo))
    return Case([[build_keyed(ss)] for ss in per_rank], [build_keyed(whole)], gid)


def series_case():
    """9 series by series range (3 per rank)"""
    return build_case([(r, sid, 0, 300 + 37 * sid) for r in range(R) for sid in range(3 * r + 1, 3 * r + 4)],
                      {sid: sid % 4 for sid in range(1, 10)})


def time_case():
    """6 series, each cut into three time windows, window r on rank r"""
    pieces = []
    for sid in range(1, 7):
        row0 = 0
        for r in range(R):
            n = 200 + 10 * sid + 7 * r
            pieces.append((r, sid, row0, n))
            row0 += n
    return build_case(pieces, {sid: sid % 2 for sid in range(1, 7)})


QUERIES = [
    dict(),
    dict(aggs=[("i", COUNT), ("f", SUM)], top=(5, 0, True)),
    dict(aggs=[("i", COUNT), ("f", MIN)], top=(4, 0, False)),
    dict(aggs=[("f", MEAN), ("i", MAX), ("i", SUM)], tmin=T0 + 50 * STEP, tmax=T0 + 700 * STEP),
    dict(aggs=[("i", SUM), ("f", MAX), ("i", MIN)], preds=[O.Pred(FAM, "z", O.OP_NE, b"z1")]),
]


def tuple_slot(bydb, case, keys, max_values, max_present, **kw):
    return bydb.keys_wide_reduce_slot_bytes(to_gpu_query(bydb, [], case.oquery([], **kw)), keys, max_values, max_present)


def call(ranks, r, q, root, keys, max_values, partial):
    fn = ranks.ctxs[r].scan_reduce_keys_wide_partials if partial else ranks.ctxs[r].scan_reduce_keys_wide
    return fn(q, keys, root=root, max_values=max_values)


def field(x, name):
    return x[name] if isinstance(x, dict) else getattr(x, name)


def stats_of(x):
    return field(x, "stats")


def n_rows_of(x):
    return len(field(x, "group_id"))


def whole_answer(bydb, gpu_ctx, case, keys, max_values, partial, flags=0, **kw):
    pid = _next_pid()
    whole = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(case.whole)]
    try:
        q = dataclasses.replace(to_gpu_query(bydb, whole, case.oquery(case.whole, **kw)), flags=flags)
        return (gpu_ctx.scan_partials_keys_wide if partial else gpu_ctx.scan_agg_keys_wide)(q, keys, max_values)
    finally:
        for h in whole:
            gpu_ctx.release_part(h)


def same_tuples(got, one, ctx):
    """the collective's answer against the single context's: rows by key bytes in order, exact integers, floats within 1e-9"""
    assert field(got, "group_id").tolist() == field(one, "group_id").tolist(), f"{ctx}: group ids"
    assert field(got, "key") == field(one, "key"), f"{ctx}: keys {field(got, 'key')[:4]} vs {field(one, 'key')[:4]}"
    assert field(got, "n_tuples") == field(one, "n_tuples"), f"{ctx}: n_tuples"
    assert [set(t) for t in field(got, "key_tables")] == [set(t) for t in field(one, "key_tables")], f"{ctx}: key tables"
    assert all(len(t) == len(set(t)) for t in field(got, "key_tables")), f"{ctx}: a tag table repeats a value"
    assert np.asarray(field(got, "is_float")).tolist() == np.asarray(field(one, "is_float")).tolist(), f"{ctx}: typing"
    if isinstance(got, dict):
        for k in ("val_i64", "cnt_i64"):
            assert np.asarray(got[k]).tolist() == np.asarray(one[k]).tolist(), f"{ctx}: {k}"
        for k in ("val_f64", "cnt_f64"):
            assert np.allclose(got[k], one[k], rtol=1e-9, atol=0, equal_nan=True), f"{ctx}: {k}"
    else:
        assert got.rows.tolist() == one.rows.tolist(), f"{ctx}: rows"
        assert got.val_i64.tolist() == one.val_i64.tolist(), f"{ctx}: int64 values"
        assert np.allclose(got.val_f64, one.val_f64, rtol=1e-9, atol=0, equal_nan=True), f"{ctx}: float values"


def to_twin(k):
    return twin([k[0]], [k[1]])[0]


def bits(x):
    return np.ascontiguousarray(x).tobytes()


def check_twin(bydb, ranks, case, qs, root, got, max_values, partial, kw, ctx, oracle=True):
    """the pair (a, b) against the wide keyed collective on the twin c, bit for bit, and that against the oracle"""
    res, codes = ranks.run(lambda r: (ranks.ctxs[r].scan_reduce_keyed_wide_partials if partial else ranks.ctxs[r].scan_reduce_keyed_wide)(
        qs[r], FAM, "c", root=root, max_values=max_values))
    assert codes == [0] * R, f"{ctx}: twin {codes}"
    w = res[root]
    assert [to_twin(k) for k in field(got, "key")] == field(w, "key"), f"{ctx}: twin keys"
    assert field(got, "n_tuples") == field(w, "n_keys"), f"{ctx}: n_tuples vs the twin's n_keys"
    names = ("group_id", "is_float", "val_i64", "cnt_i64", "val_f64", "cnt_f64") if partial else ("group_id", "is_float", "rows", "val_i64", "val_f64")
    for k in names:
        assert bits(np.asarray(field(got, k))) == bits(np.asarray(field(w, k))), f"{ctx}: twin {k}"
    if oracle and not partial:
        want = O.run_query(dataclasses.replace(case.oquery([p for s in case.shards for p in s], **kw), group_key=(FAM, "c")))
        if w.group_id.size or want.group_id.size:
            assert_parity(w, want, kw.get("aggs", K.AGGS), ctx)
        assert w.key == want.key, f"{ctx}: twin keys vs oracle"


def check(bydb, gpu_ctx, ranks, case, root, keys=PAIR, max_values=256, partial=False, forms=None, twin_check=True, flags=0, label="", **kw):
    """one tuple collective against the single-context call, the twin collective and the header's counters; -> the root's answer.
    forms: per rank, True = the partial call (the root's decides the answer), default: every rank `partial`"""
    forms = forms or [partial] * R
    partial = forms[root]
    ctx = f"{label}/root{root}/{'partial' if partial else 'final'}/{len(keys)}/{kw}"
    qs = [dataclasses.replace(to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], **kw)), flags=flags) for r in range(R)]
    res, codes = ranks.run(lambda r: call(ranks, r, qs[r], root, keys, max_values, forms[r]))
    assert codes == [0] * R, f"{ctx}: {codes}"
    got = res[root]
    one = whole_answer(bydb, gpu_ctx, case, keys, max_values, partial, flags=flags, **kw)
    same_tuples(got, one, ctx)
    if twin_check and keys == PAIR:
        check_twin(bydb, ranks, case, qs, root, got, max_values, partial, kw, ctx, oracle=flags == 0)
    assert sum(stats_of(res[r]).rows_matched for r in range(R)) == stats_of(one).rows_matched, ctx
    # every rank's own counters: its one wide pass, as bydb_scan_partials_keys_wide over its shard counts it
    Kt = len(keys)
    width = [8 if ty == INT else 68 for _, _, ty in keys]
    own_d2h, own_launch, sum_t, sum_c = [], [], 0, 0
    for r in range(R):
        alone = ranks.ctxs[r].scan_partials_keys_wide(qs[r], keys, max_values)
        T, C = alone["n_tuples"], len(alone["group_id"])
        sa = alone["stats"]
        sum_t, sum_c = sum_t + T, sum_c + C
        mine = stats_of(res[r])
        assert (mine.rows_scanned, mine.blocks_scanned, mine.rows_matched, mine.page_bytes) == \
            (sa.rows_scanned, sa.blocks_scanned, sa.rows_matched, sa.page_bytes), f"{ctx}: rank {r} counters"
        disc = 32 * (Kt + 1) + sum(len(tb) * w for tb, w in zip(alone["key_tables"], width)) + 8 * T
        own_d2h.append(disc + (264 if T else 0))
        own_launch.append(sa.kernel_launches + (1 if T else 0))
        if r != root:
            assert n_rows_of(res[r]) == 0 and field(res[r], "n_tuples") == 0, f"{ctx}: rank {r} got rows"
            assert mine.d2h_bytes == own_d2h[r], f"{ctx}: rank {r} d2h {mine.d2h_bytes} vs {own_d2h[r]}"
            assert mine.kernel_launches == own_launch[r], f"{ctx}: rank {r} launches {mine.kernel_launches} vs {own_launch[r]}"
    st, so = stats_of(got), stats_of(one)
    Tu, Cu = field(got, "n_tuples"), n_rows_of(got)
    vu = [len(tb) for tb in field(got, "key_tables")]
    d2h = own_d2h[root] + 36 * R + ((96 + sum(vu) * 68 + 8 * Tu) if sum_t else 0)
    if Cu:
        disc = 32 * (Kt + 1) + sum(v * w for v, w in zip(vu, width)) + 8 * Tu + 264  # the single-context call's own pass
        d2h += so.d2h_bytes - disc                                                    # the same answer over the same C_u groups
    assert st.d2h_bytes == d2h, f"{ctx}: root d2h {st.d2h_bytes} vs {d2h}"
    if partial:
        launches = own_launch[root] + ((6 * Kt + 1 + 6 + (1 if sum_c else 0)) if sum_t else 0)
        if Cu:
            launches += 8 + sort_launches(sum_c) + 1
        assert st.kernel_launches == launches, f"{ctx}: root launches {st.kernel_launches} vs {launches}"
    return got


def refused(bydb, ranks, case, root, want_codes, qs=None, keys=PAIR, max_values=256, partial=False, **kw):
    qs = qs or [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], **kw)) for r in range(R)]
    _, codes = ranks.run(lambda r: call(ranks, r, qs[r], root, keys, max_values, partial))
    assert codes == want_codes, (codes, want_codes)


def slot_of(bydb, *cases):
    return max(tuple_slot(bydb, c, FOUR, 512, 2048) for c in cases)


# ------------------------------------------------------------------ tests
@gpu
def test_series_and_time_shards(bydb, gpu_ctx, quiet):
    """series shards and time shards with the pair (a, b): every query (Top-N both ways, a time cut, a predicate), both answer
    forms, row-path typing, roots 0 and 2, against the single context, the twin collective and the oracle"""
    sc, tc = series_case(), time_case()
    ranks = Ranks(bydb, slot_of(bydb, sc, tc))
    try:
        for case, name in ((sc, "series"), (tc, "time")):
            ranks.register(case.shards)
            for root in (0, 2):
                for kw in QUERIES:
                    check(bydb, gpu_ctx, ranks, case, root, label=name, **kw)
                check(bydb, gpu_ctx, ranks, case, root, partial=True, label=name, **QUERIES[3])
            check(bydb, gpu_ctx, ranks, case, 1, flags=bydb.capi.Q_ROW_PATH_TYPES, label=name + "-rowpath", **QUERIES[3])
            got = [check(bydb, gpu_ctx, ranks, case, 1, label=name + "-repeat") for _ in range(2)]
            assert bits(got[0].val_f64) == bits(got[1].val_f64) and got[0].key == got[1].key
    finally:
        ranks.close()


@gpu
def test_three_and_four_tags(bydb, gpu_ctx, quiet):
    """3- and 4-tag keys of mixed types (tag values present on one rank only, the same tuple under different local ids on every
    rank) over series and time shards, both forms, against the single context"""
    sc, tc = series_case(), time_case()
    ranks = Ranks(bydb, slot_of(bydb, sc, tc))
    try:
        for case, name in ((sc, "series"), (tc, "time")):
            ranks.register(case.shards)
            for keys in (THREE, FOUR):
                for root in (0, 2):
                    got = check(bydb, gpu_ctx, ranks, case, root, keys=keys, max_values=512, label=name, **QUERIES[0])
                    assert {b"only0", b"only1", b"only2"} <= set(got.key_tables[keys.index((FAM, "a", STR))])
                    check(bydb, gpu_ctx, ranks, case, root, keys=keys, max_values=512, label=name, **QUERIES[1])
                    check(bydb, gpu_ctx, ranks, case, root, keys=keys, max_values=512, partial=True, label=name, **QUERIES[4])
    finally:
        ranks.close()


@gpu
def test_union_edges(bydb, gpu_ctx, quiet):
    """a rank without a selected block, all ranks empty, union tuples at exactly max_values and at max_values + 1 while every rank
    alone is under it (ENOMEM at the root only)"""
    sc = series_case()
    ranks = Ranks(bydb, slot_of(bydb, sc), sc.shards)
    try:
        got = check(bydb, gpu_ctx, ranks, sc, 0, label="full")
        T = got.n_tuples
        alone = [ranks.ctxs[r].scan_partials_keys_wide(to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])), PAIR, 256)["n_tuples"]
                 for r in range(R)]
        assert max(alone) < T, (alone, T)
        for root in (0, 2):
            got = check(bydb, gpu_ctx, ranks, sc, root, max_values=T, label="exact")
            assert got.n_tuples == T
            want = [0] * R
            want[root] = ENOMEM
            refused(bydb, ranks, sc, root, want, max_values=T - 1)
            check(bydb, gpu_ctx, ranks, sc, root, max_values=T, partial=True, label="after-cap")
            got = check(bydb, gpu_ctx, ranks, sc, root, label="rank1-empty", sids=[1, 2, 3, 7, 8, 9])
            assert b"only1" not in got.key_tables[0]
            got = check(bydb, gpu_ctx, ranks, sc, root, keys=FOUR, label="all-empty", tmin=T0 + 10**6 * STEP, tmax=T0 + 2 * 10**6 * STEP)
            assert got.n_tuples == 0 and got.group_id.size == 0 and got.key_tables == [[], [], [], []]
    finally:
        ranks.close()


@gpu
def test_65536_tuples_and_a_tag_of_65536_values(bydb, gpu_ctx, quiet):
    """256 series of 256 rows sharded by series range: b = a value per row (65,536 int64 values, each rank a third of them), a =
    the series' parity, so 65,536 union tuples, all 16 bits of b's union ids in use; at max_values 65,535 the root refuses
    (ENOMEM) although every rank alone is far under it"""
    def cells(rank, sid, x):
        b = (sid - 1) * 256 + x - 30000
        return {"a": b"p%d" % (sid % 2), "b": b, "d": b"d", "e": 0, "z": b"z%d" % (x % 4)}
    pieces = [(min(R - 1, (sid - 1) // 86), sid, 0, 256) for sid in range(1, 257)]
    case = build_case(pieces, {sid: sid % 3 for sid in range(1, 257)}, cells)
    aggs = [("i", SUM), ("i", COUNT), ("f", MAX)]
    ranks = Ranks(bydb, tuple_slot(bydb, case, PAIR, 65536, 65536, aggs=aggs), case.shards)
    try:
        got = check(bydb, gpu_ctx, ranks, case, 0, max_values=65536, label="65536", aggs=aggs)
        assert got.n_tuples == 65536 == got.group_id.size and len(got.key_tables[1]) == 65536 and len(got.key_tables[0]) == 2
        assert got.key == [(b"p%d" % (s % 2), le((s - 1) * 256 + x - 30000)) for s in range(1, 257) for x in range(256)]
        check(bydb, gpu_ctx, ranks, case, 2, max_values=65536, partial=True, label="65536-partial", aggs=aggs)
        refused(bydb, ranks, case, 1, [0, ENOMEM, 0], max_values=65535, aggs=aggs)
        check(bydb, gpu_ctx, ranks, case, 1, max_values=65536, label="65536-after", twin_check=False, aggs=aggs)
    finally:
        ranks.close()


@gpu
def test_slot_filled_exactly(bydb, gpu_ctx, quiet):
    """a rank whose tag values, tuples and composite groups fill the exported slot to its last byte answers; one composite group
    more is refused on that rank and at the root (BYDB_EINVAL), and the ranks stay in step"""
    k = 32  # 32 tuple codes are 256 bytes: the slot at (k, k) ends on a 256-byte boundary, so the export adds no slack
    aggs = [("i", SUM), ("f", SUM)]

    def cells(rank, sid, x):
        v = x % k if sid == 1 else 0 if sid == 4 else (x + sid) % 3
        return {"a": b"k%02d" % v, "b": v, "d": b"d", "e": 0, "z": b"z"}
    fits = build_case([(1, 1, 0, 3 * k), (0, 2, 0, 15), (2, 3, 0, 15)], {1: 0, 2: 0, 3: 1}, cells)
    over = build_case([(1, 1, 0, 3 * k), (1, 4, 0, 5), (0, 2, 0, 15), (2, 3, 0, 15)], {1: 0, 2: 0, 3: 1, 4: 1}, cells)
    slot = tuple_slot(bydb, fits, PAIR, k, k, aggs=aggs)
    assert slot % 256 == 0
    assert tuple_slot(bydb, over, PAIR, k, k + 1, aggs=aggs) > slot
    ranks = Ranks(bydb, slot, fits.shards)
    try:
        check(bydb, gpu_ctx, ranks, fits, 0, max_values=k, label="fits", aggs=aggs)
        ranks.register(over.shards)
        qs = [to_gpu_query(bydb, ranks.hs[r], over.oquery(over.shards[r], aggs=aggs)) for r in range(R)]
        refused(bydb, ranks, over, 0, [EINVAL, EINVAL, 0], qs=qs, max_values=k)
        refused(bydb, ranks, over, 1, [0, EINVAL, 0], qs=qs, max_values=k)
        ranks.register(fits.shards)
        check(bydb, gpu_ctx, ranks, fits, 2, max_values=k, partial=True, label="fits-after", aggs=aggs)
    finally:
        ranks.close()


@gpu
def test_refusals_keep_the_epochs_in_step(bydb, gpu_ctx, quiet):
    """another key order on one rank, a one-key wide call in the same round, intersecting spans, overlapping parts on one rank,
    a block with 257 tuples and a 65-byte tag value: each refused, and each followed by a plain and a tuple collective"""
    sc = series_case()
    ranks = Ranks(bydb, slot_of(bydb, sc), sc.shards)
    try:
        def after(root):
            ranks.register(sc.shards)
            plain_ok(bydb, gpu_ctx, ranks, sc, root)
            check(bydb, gpu_ctx, ranks, sc, root, label="after", twin_check=False, **QUERIES[1])
        qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])) for r in range(R)]
        # rank 1 passes the same tags in another order
        _, codes = ranks.run(lambda r: call(ranks, r, qs[r], 0, PAIR[::-1] if r == 1 else PAIR, 256, False))
        assert codes == [EINVAL, 0, 0], codes
        after(0)
        # rank 2 calls the one-key wide collective on the twin in the same round
        _, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed_wide(qs[r], FAM, "c", root=1, max_values=256) if r == 2
                             else call(ranks, r, qs[r], 1, PAIR, 256, False))
        assert codes == [0, EINVAL, 0], codes
        after(1)
        # series 1 also on rank 1, over times that intersect its rows on rank 0
        inter = build_case([(0, 1, 0, 50), (1, 1, 49, 50), (1, 2, 0, 50), (2, 3, 0, 50)], {1: 0, 2: 0, 3: 0})
        ranks.register(inter.shards)
        refused(bydb, ranks, inter, 0, [ENOTSUP, 0, 0])
        after(0)
        # two parts of rank 2 that overlap in time
        ranks.register(sc.shards)
        cs = [std_cells(2, 8, x) for x in range(20)]
        extra = build_keyed([Series(8, std_fields(8, 20), tag_columns(cs))])
        ranks.hs[2].append(ranks.ctxs[2].register_part(_next_pid(), extra.files()))
        refused(bydb, ranks, sc, 1, [0, ENOTSUP, ENOTSUP])
        after(1)
        # a block with 257 distinct tuples on rank 2, and a 65-byte value of tag a on rank 0
        def many(rank, sid, x):
            c = std_cells(rank, sid, x)
            if rank == 2 and sid == 3:
                c["a"], c["b"] = b"m%d" % (x // 17), x % 17
            if rank == 0 and sid == 1 and x == 4:
                c["a"] = b"x" * 65
            return c
        bad = build_case([(0, 1, 0, 100), (1, 2, 0, 100), (2, 3, 0, 257 + 17)], {1: 0, 2: 0, 3: 0}, many)
        ranks.register(bad.shards)
        refused(bydb, ranks, bad, 2, [ENOTSUP, 0, ENOTSUP], aggs=[("i", COUNT)])
        after(2)
    finally:
        ranks.close()


@gpu
def test_forms_mixed_over_rotating_roots(bydb, gpu_ctx, quiet):
    """the finalised and the partial call mixed in one collective (the root's call decides its answer); plain, wide keyed and tuple
    collectives alternating over rotating roots"""
    sc = series_case()
    slot = max(slot_of(bydb, sc), bydb.keyed_wide_reduce_slot_bytes(to_gpu_query(bydb, [], sc.oquery([])), FAM, "c", 256, 256))
    ranks = Ranks(bydb, slot, sc.shards)
    try:
        for it in range(9):
            root = it % R
            if it % 3 == 1:
                plain_ok(bydb, gpu_ctx, ranks, sc, root)
            elif it % 3 == 2:
                qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])) for r in range(R)]
                res, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed_wide(qs[r], FAM, "c", root=root, max_values=256))
                assert codes == [0] * R and res[root].group_id.size > 0, codes
            else:
                forms = [(r + it) % 2 == 1 for r in range(R)]
                check(bydb, gpu_ctx, ranks, sc, root, keys=PAIR if it % 2 else THREE, forms=forms, max_values=512, label=f"mixed{it}",
                      **QUERIES[it % len(QUERIES)])
    finally:
        ranks.close()

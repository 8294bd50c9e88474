"""Group-by on a stored tag with up to 65,536 values across ranks (bydb_scan_reduce_keyed_wide / _partials, DESIGN.md 5): R = 3
ranks as threads, one context each on device r % device_count (a one-GPU box exercises the host-polled shared-device waits, a
multi-GPU box the device-side waits).  Every rank passes the same query but its parts.  Each answer of the root is checked
  - against the oracle with group_key over all ranks' parts (an int64 key through its string twin);
  - against bydb_scan_agg_keyed_wide / bydb_scan_partials_keyed_wide on one context, over one part holding every rank's rows
    (series shards) or over the ranks' parts themselves (time shards): group ids, key bytes, rows, int64 values and min / max
    exactly and in order, floats within 1e-9 relative;
  - on n_keys, on rows_matched summed over the ranks, on every other rank's empty answer and own counters, and on d2h_bytes /
    kernel_launches against the header's formulas.
"""
import dataclasses

import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0, assert_parity, to_gpu_query
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM
from tests.test_gpu_keyed import FAM, KT, build_keyed, mk
from tests.test_gpu_keyed_int64 import KX
from tests.test_gpu_keyed_reduce import (EINVAL, ENOMEM, ENOTSUP, QUERIES, R, S_TAG, Case, Ranks, _next_pid, order_case, plain_ok,  # noqa: F401
                                         quiet, series_case, split, time_case)
from tests.test_gpu_keyed_wide import identical, int_series, le, same_result, same_rows, string_fixture

gpu = pytest.mark.gpu


def sort_launches(n):
    """bitonic launches past the first tile for n keys (the header's sort(N)), N = pow2(max(n, 2048))"""
    N = 2048
    while N < n:
        N *= 2
    total, size = 0, 4096
    while size <= N:
        total += size.bit_length() - 1 - 10
        size *= 2
    return total


def wide_slot(bydb, case, max_values, max_present, **kw):
    q = to_gpu_query(bydb, [], case.oquery([], **kw))
    return bydb.keyed_wide_reduce_slot_bytes(q, FAM, KT, max_values, max_present)


def call(ranks, r, q, root, key, max_values, vt, partial):
    fn = ranks.ctxs[r].scan_reduce_keyed_wide_partials if partial else ranks.ctxs[r].scan_reduce_keyed_wide
    return fn(q, FAM, key, root=root, max_values=max_values, value_type=vt)


def stats_of(x):
    return x["stats"] if isinstance(x, dict) else x.stats


def n_rows_of(x):
    return len(x["group_id"]) if isinstance(x, dict) else x.group_id.size


def n_keys_of(x):
    return x["n_keys"] if isinstance(x, dict) else x.n_keys


def whole_answer(bydb, gpu_ctx, case, key, max_values, vt, partial, **kw):
    pid = _next_pid()
    whole = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(case.whole)]
    try:
        q = to_gpu_query(bydb, whole, case.oquery(case.whole, **kw))
        fn = gpu_ctx.scan_partials_keyed_wide if partial else gpu_ctx.scan_agg_keyed_wide
        return fn(q, FAM, key, max_values, vt)
    finally:
        for h in whole:
            gpu_ctx.release_part(h)


def check(bydb, gpu_ctx, ranks, case, root, key=KT, vt=0, twin=None, max_values=256, partial=False, forms=None, oracle=True, label="", **kw):
    """one wide keyed collective against the oracle, the single-context wide call and the header's counters; -> the root's answer.
    forms: per rank, True = the partial call (the root's decides the answer), default: every rank `partial`"""
    forms = forms or [partial] * R
    partial = forms[root]
    ctx = f"{label}/root{root}/{'partial' if partial else 'final'}/{kw}"
    qs = [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], **kw)) for r in range(R)]
    res, codes = ranks.run(lambda r: call(ranks, r, qs[r], root, key, max_values, vt, forms[r]))
    assert codes == [0] * R, f"{ctx}: {codes}"
    got = res[root]
    one = whole_answer(bydb, gpu_ctx, case, key, max_values, vt, partial, **kw)
    (same_rows if partial else same_result)(one, got, ctx)
    if oracle and not partial:
        want = O.run_query(dataclasses.replace(case.oquery([p for s in case.shards for p in s], **kw), group_key=(FAM, twin or key)))
        if got.group_id.size or want.group_id.size:
            assert_parity(got, want, kw.get("aggs", K.AGGS), ctx)
        assert got.key == want.key, f"{ctx}: keys vs oracle"
    st = stats_of(got)
    assert sum(stats_of(res[r]).rows_matched for r in range(R)) == stats_of(one).rows_matched, ctx
    # every rank's own counters: its one wide pass, as bydb_scan_partials_keyed_wide over its shard counts it
    width = 8 if vt == bydb.VT_INT64 else 68
    own_d2h, own_launch, sum_v, sum_c = [], [], 0, 0
    for r in range(R):
        alone = ranks.ctxs[r].scan_partials_keyed_wide(qs[r], FAM, key, max_values, vt)
        V, C = alone["n_keys"], len(alone["group_id"])
        sa = alone["stats"]
        sum_v, sum_c = sum_v + V, sum_c + C
        mine = stats_of(res[r])
        assert (mine.rows_scanned, mine.blocks_scanned, mine.rows_matched, mine.page_bytes) == \
            (sa.rows_scanned, sa.blocks_scanned, sa.rows_matched, sa.page_bytes), f"{ctx}: rank {r} counters"
        own_d2h.append(32 + V * width + (264 if V else 0))
        # alone: the pass + the fold + the row kernel when C > 0; in the collective: the pass + fold, spans, first series when C > 0
        own_launch.append(sa.kernel_launches + (1 if V else 0))
        if r != root:
            assert n_rows_of(res[r]) == 0 and n_keys_of(res[r]) == 0, f"{ctx}: rank {r} got rows"
            assert mine.d2h_bytes == own_d2h[r], f"{ctx}: rank {r} d2h {mine.d2h_bytes} vs {own_d2h[r]}"
            assert mine.kernel_launches == own_launch[r], f"{ctx}: rank {r} launches {mine.kernel_launches} vs {own_launch[r]}"
    n_keys = n_keys_of(got)
    Cu = n_rows_of(got)
    # the root: its own pass, then the headers, the union's read-back and the answer
    d2h = own_d2h[root] + 16 * R + ((16 + n_keys * 68) if sum_v else 0)
    if Cu:
        so = stats_of(one)
        disc = 32 + n_keys * width + 264  # the single-context call's own pass (n_keys = its V)
        d2h += so.d2h_bytes - disc        # the same answer over the same C_u groups
    assert st.d2h_bytes == d2h, f"{ctx}: root d2h {st.d2h_bytes} vs {d2h}"
    if partial:
        launches = own_launch[root] + ((6 + (1 if R > 1 else 0) + (1 if sum_c else 0)) if sum_v else 0)
        if Cu:
            launches += 8 + sort_launches(sum_c) + 1
        assert st.kernel_launches == launches, f"{ctx}: root launches {st.kernel_launches} vs {launches}"
    return got


def refused(bydb, ranks, case, root, want_codes, qs=None, key=KT, max_values=256, vt=0, partial=False):
    qs = qs or [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r])) for r in range(R)]
    _, codes = ranks.run(lambda r: call(ranks, r, qs[r], root, key, max_values, vt, partial))
    assert codes == want_codes, (codes, want_codes)


EIGHT_PREDS = dict(aggs=[("i", SUM), ("f", MAX), ("i", COUNT)],
                   preds=[O.Pred(FAM, S_TAG, O.OP_NE, b"w%d" % j) for j in range(7)] + [O.Pred(FAM, KT, O.OP_GE, b"b")])


# ------------------------------------------------------------------ tests
@gpu
def test_series_and_time_shards(bydb, gpu_ctx, quiet):
    """series shards (string key, nil next to "", values of one rank only) and time shards (int64 key, a value first seen on a
    later rank), every query of the per-value collective's test, eight predicates, both answer forms, roots 0 and 2; three
    identical collectives bit for bit"""
    sc, tc = series_case(), time_case()
    ranks = Ranks(bydb, max(wide_slot(bydb, sc, 256, 256), wide_slot(bydb, tc, 256, 256), 1 << 16))
    try:
        ranks.register(sc.shards)
        for root in (0, 2):
            for kw in QUERIES + [EIGHT_PREDS]:
                check(bydb, gpu_ctx, ranks, sc, root, label="series", **kw)
            check(bydb, gpu_ctx, ranks, sc, root, partial=True, label="series", **QUERIES[3])
        got = [check(bydb, gpu_ctx, ranks, sc, 1, label="repeat", **QUERIES[0]) for _ in range(3)]
        assert identical(got[0], got[1]) and identical(got[0], got[2])
        ranks.register(tc.shards)
        for root in (0, 2):
            for kw in QUERIES:
                check(bydb, gpu_ctx, ranks, tc, root, vt=bydb.VT_INT64, twin=KX, label="time", **kw)
            check(bydb, gpu_ctx, ranks, tc, root, vt=bydb.VT_INT64, partial=True, label="time", **QUERIES[0])
    finally:
        ranks.close()


@gpu
def test_insertion_order_across_ranks(bydb, gpu_ctx, quiet):
    """a value first seen on a later rank in a series' later window, a value on one rank only, a group whose first series is on a
    later rank, and Top-N both ways with ties resolved by the insertion order of the whole scan"""
    case = order_case()
    ranks = Ranks(bydb, wide_slot(bydb, case, 256, 64), case.shards)
    try:
        for root in (0, 2):
            got = check(bydb, gpu_ctx, ranks, case, root, label="order")
            assert list(zip(got.group_id.tolist(), got.key))[:3] == [(0, b"p"), (0, b"q"), (0, b"late")], got.key
            check(bydb, gpu_ctx, ranks, case, root, label="order-top", aggs=[("i", COUNT)], top=(4, 0, True))
            check(bydb, gpu_ctx, ranks, case, root, label="order-top-asc", aggs=[("i", COUNT)], top=(3, 0, False))
            check(bydb, gpu_ctx, ranks, case, root, partial=True, label="order-partial")
    finally:
        ranks.close()


@gpu
def test_union_edges(bydb, gpu_ctx, quiet):
    """values only one rank has, a rank without a selected block, all ranks empty, a union of exactly max_values and one of
    max_values + 1 with every rank under the cap (ENOMEM at the root only)"""
    # rank r: series 2r + 1 and 2r + 2 with 200 values each (a block holds at most 256), v[300r, 300r + 400) together
    big = split([(r, 2 * r + 1 + h, [b"v%04d" % v for v in range(300 * r + 200 * h, 300 * r + 200 * h + 200)], 0) for r in range(R) for h in (0, 1)],
                {1: 0, 2: 1, 3: 0, 4: 2, 5: 1, 6: 0})
    ranks = Ranks(bydb, wide_slot(bydb, big, 1000, 1000))
    try:
        ranks.register(big.shards)
        for root in (0, 2):
            got = check(bydb, gpu_ctx, ranks, big, root, max_values=1000, label="1000")
            assert got.n_keys == 1000
            got = check(bydb, gpu_ctx, ranks, big, root, max_values=1000, label="rank1-empty", sids=[1, 2, 5, 6])
            assert got.n_keys == 800 and b"v0400" not in got.key
            got = check(bydb, gpu_ctx, ranks, big, root, max_values=1000, label="all-empty", tmin=T0 + 10**6 * STEP, tmax=T0 + 2 * 10**6 * STEP)
            assert got.n_keys == 0 and got.group_id.size == 0
            want = [0] * R
            want[root] = ENOMEM
            refused(bydb, ranks, big, root, want, max_values=999)
            check(bydb, gpu_ctx, ranks, big, root, max_values=1000, partial=True, label="after-cap")
    finally:
        ranks.close()


@gpu
def test_thousands_of_values(bydb, gpu_ctx, quiet):
    """4,096 string values (and the nil cells' "") sharded by series range, against the oracle; 65,536 int64 values over 256
    series, every (group, value) present once, against the single-context wide call and a numpy model"""
    part, ss = string_fixture(4096)
    third = len(ss) // R
    shards = [[build_keyed(ss[r * third:(r + 1) * third if r < R - 1 else len(ss)])] for r in range(R)]
    case = Case(shards, [part], {s.sid: s.sid % 5 for s in ss})
    aggs = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("f", SUM), ("f", MEAN)]
    vals = [[(s * 256 + r) * 977 % 65536 - 20000 for r in range(256)] for s in range(256)]
    iss = [int_series(s + 1, vals[s]) for s in range(256)]
    ishards = [[build_keyed(iss[r * 86:min((r + 1) * 86, 256)])] for r in range(R)]
    icase = Case(ishards, [build_keyed(iss)], {s + 1: s % 7 for s in range(256)})
    slot = max(wide_slot(bydb, case, 4097, 4097 * 5, aggs=aggs), wide_slot(bydb, icase, 65536, 65536, aggs=[("i", SUM), ("i", COUNT), ("f", MAX)]))
    ranks = Ranks(bydb, slot)
    try:
        ranks.register(case.shards)
        got = check(bydb, gpu_ctx, ranks, case, 1, max_values=4097, label="4096", aggs=aggs)
        assert got.n_keys == 4097
        check(bydb, gpu_ctx, ranks, case, 0, max_values=4097, label="4096-cut", aggs=aggs, tmin=T0 + 123 * STEP, tmax=T0 + 871 * STEP,
              preds=[O.Pred(FAM, "z", O.OP_NE, b"z3")])
        for desc in (True, False):
            check(bydb, gpu_ctx, ranks, case, 2, max_values=4097, label="4096-top", aggs=[("i", COUNT), ("f", MAX)], top=(17, 0, desc))
        check(bydb, gpu_ctx, ranks, case, 2, max_values=65536, partial=True, label="4096-partial", aggs=aggs)
        ranks.register(icase.shards)
        iaggs = [("i", SUM), ("i", COUNT), ("f", MAX)]
        got = check(bydb, gpu_ctx, ranks, icase, 0, vt=bydb.VT_INT64, max_values=65536, oracle=False, label="65536", aggs=iaggs)
        assert got.n_keys == 65536
        assert list(zip(got.group_id.tolist(), got.key)) == [(s % 7, le(v)) for s in range(256) for v in vals[s]]
        assert got.rows.tolist() == [1] * 65536
        assert got.val_i64[:, 0].tolist() == [v * 3 + s + 1 for s in range(256) for v in vals[s]]
        want = [0] * R
        want[0] = ENOMEM
        qs = [to_gpu_query(bydb, ranks.hs[r], icase.oquery(icase.shards[r], aggs=iaggs)) for r in range(R)]
        refused(bydb, ranks, icase, 0, want, qs=qs, vt=bydb.VT_INT64, max_values=65535)
    finally:
        ranks.close()


@gpu
def test_slot_filled_exactly(bydb, gpu_ctx, quiet):
    """a rank whose V_r values and C_r composite groups fill the exported slot to its last byte answers; one more composite group
    is refused on that rank and at the root (BYDB_EINVAL), and the ranks stay in step"""
    k = 34   # with two fields the slot at (k, k) is a multiple of 256 bytes: the export adds no slack
    aggs = [("i", SUM), ("f", SUM)]
    vals = [b"k%02d" % v for v in range(k)]
    fits = split([(1, 1, vals * 3, 0), (0, 2, vals[:3] * 5, 0), (2, 3, vals[5:9] * 5, 0)], {1: 0, 2: 0, 3: 1})
    over = split([(1, 1, vals * 3, 0), (1, 4, vals[:1] * 5, 0), (0, 2, vals[:3] * 5, 0), (2, 3, vals[5:9] * 5, 0)], {1: 0, 2: 0, 3: 1, 4: 1})
    slot = wide_slot(bydb, fits, k, k, aggs=aggs)
    assert slot % 256 == 0
    assert wide_slot(bydb, over, k, k + 1, aggs=aggs) > slot
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
    """a per-value keyed rank among wide ones, a fingerprint mismatch, intersecting spans, a block with 257 values and overlapping
    parts on one rank: each refused, and each followed by a plain and a wide collective that answer correctly"""
    sc = series_case()
    slot = max(wide_slot(bydb, sc, 256, 256), bydb.keyed_reduce_slot_bytes(to_gpu_query(bydb, [], sc.oquery([])), FAM, KT, 256))
    ranks = Ranks(bydb, slot, sc.shards)
    try:
        def after(root):
            ranks.register(sc.shards)
            plain_ok(bydb, gpu_ctx, ranks, sc, root)
            check(bydb, gpu_ctx, ranks, sc, root, label="after", **QUERIES[1])
        # rank 1 calls the per-value collective: the wide root refuses; a per-value root refuses the wide ranks
        qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])) for r in range(R)]
        for root in (0, 1):
            _, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed(qs[r], FAM, KT, root=root, max_values=256) if r == 1
                                 else call(ranks, r, qs[r], root, KT, 256, 0, False))
            want = [0] * R
            want[root] = EINVAL
            assert codes == want, (root, codes)
            after(root)
        # ranks that disagree on max_values
        _, codes = ranks.run(lambda r: call(ranks, r, qs[r], 2, KT, 128 if r == 0 else 256, 0, False))
        assert codes == [0, 0, EINVAL], codes
        after(2)
        # series 1 also on rank 1, over times that intersect its rows on rank 0
        st = {S_TAG: [b"x"] * 50}
        inter = Case([[build_keyed([mk(1, [b"a"] * 50, tags=st)])], [build_keyed([mk(1, [b"b"] * 50, row0=49, tags=st), mk(2, [b"a"] * 50, tags=st)])],
                      [build_keyed([mk(3, [b"c"] * 50, tags=st)])]], None, {1: 0, 2: 0, 3: 0})
        ranks.register(inter.shards)
        refused(bydb, ranks, inter, 0, [ENOTSUP, 0, 0])
        after(0)
        # an int64 block with 257 distinct values on rank 2
        wide_block = Case([[build_keyed([int_series(1, [5] * 40)])], [build_keyed([int_series(2, [6] * 40)])],
                           [build_keyed([int_series(3, list(range(257)))])]], None, {1: 0, 2: 0, 3: 0})
        ranks.register(wide_block.shards)
        qs = [to_gpu_query(bydb, ranks.hs[r], wide_block.oquery(wide_block.shards[r], aggs=[("i", COUNT)])) for r in range(R)]
        refused(bydb, ranks, wide_block, 0, [ENOTSUP, 0, ENOTSUP], qs=qs, vt=bydb.VT_INT64, max_values=1000)
        after(0)
        # two parts of rank 2 that overlap in time
        ranks.register(sc.shards)
        ranks.hs[2].append(ranks.ctxs[2].register_part(_next_pid(), build_keyed([mk(13, [b"a"] * 20, tags={S_TAG: [b"x"] * 20})]).files()))
        refused(bydb, ranks, sc, 1, [0, ENOTSUP, ENOTSUP])
        after(1)
    finally:
        ranks.close()


@gpu
def test_forms_mixed_over_rotating_roots(bydb, gpu_ctx, quiet):
    """the finalised and the partial call mixed in one collective (the root's call decides its answer), plain, per-value keyed
    and wide collectives alternating over rotating roots"""
    sc = series_case()
    slot = max(wide_slot(bydb, sc, 256, 256), bydb.keyed_reduce_slot_bytes(to_gpu_query(bydb, [], sc.oquery([])), FAM, KT, 256))
    ranks = Ranks(bydb, slot, sc.shards)
    try:
        for it in range(9):
            root = it % R
            if it % 3 == 1:
                plain_ok(bydb, gpu_ctx, ranks, sc, root)
            elif it % 3 == 2:
                qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])) for r in range(R)]
                res, codes = ranks.keyed(qs, root)
                assert codes == [0] * R and res[root].group_id.size > 0, codes
            else:
                forms = [(r + it) % 2 == 1 for r in range(R)]
                check(bydb, gpu_ctx, ranks, sc, root, forms=forms, label=f"mixed{it}", **QUERIES[it % len(QUERIES)])
    finally:
        ranks.close()

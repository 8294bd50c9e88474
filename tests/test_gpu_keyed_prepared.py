"""-m gpu: the prepared group-by on a stored tag (bydb_query_prepare_keyed / bydb_scan_agg_keyed_prepared, DESIGN.md 4.6).

Its first execution runs the plain keyed path; the second discovers the key values and captures the V passes, the insertion
order, the finalisation and the row mapping as one CUDA graph; later ones replay that graph.  Every handle here runs at least
five times (plain, capture + replay, replays), and every execution must give what bydb_scan_agg_keyed gives on the same context
for the same query: rows, keys, values bit for bit, the counters, and the same refusals.  The plain answers themselves are checked
against the oracle and the models of test_gpu_keyed.py / test_gpu_keyed_int64.py (KScan / KScan64), so every replay is too.
"""
import dataclasses
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM
from tests.test_gpu_keyed import AGGS, FAM, KT, KScan, ab_parts, build_keyed, lane_series, limit_series, mk, order_series
from tests.test_gpu_keyed_int64 import KScan64, cap_series, kind_series, mk64
from tests.test_gpu_masks import I64_MAX, I64_MIN

pytestmark = pytest.mark.gpu

RUNS = 5
COUNTERS = ("rows_scanned", "rows_matched", "page_bytes", "blocks_scanned", "blocks_slow_lane", "slow_lane_reasons", "blocks_express_lane")
_pid = [9_700_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def assert_same(got, want, what):
    """a prepared execution against the plain keyed call: everything but the timing / transfer stats, floats as bit patterns"""
    assert {k: getattr(got.stats, k) for k in COUNTERS} == {k: getattr(want.stats, k) for k in COUNTERS}, what
    assert got.n_keys == want.n_keys and got.key == want.key, (what, got.n_keys, want.n_keys, got.key[:8], want.key[:8])
    assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), what
    assert got.is_float.tolist() == want.is_float.tolist(), what
    assert got.val_i64.tolist() == want.val_i64.tolist(), what
    assert got.val_f64.view(np.uint64).tolist() == want.val_f64.view(np.uint64).tolist(), what


def a256(x):
    return (x + 255) // 256 * 256


def replay_d2h(want, q):
    """bydb_gpu.h's d2h_bytes of a replay: the result rows over V x G groups, a (group, key) pair per row, a zero page per pass"""
    V, G, A = want.n_keys, (q.n_groups if q.series_group is not None else 1), len(q.aggs)
    R = min(q.top_n, V * G) if q.top_n > 0 else V * G
    return a256(16) + a256(A) + a256(4 * R) + a256(8 * R) + 2 * a256(8 * R * A) + a256(8 * R) + 256 * V


def run_prepared(bydb, ctx, q, key, max_values, value_type, want, what, runs=RUNS):
    """runs a handle `runs` times against the plain answer `want`; replays also against the stats contract"""
    g = ctx.prepare_keyed(q, FAM, key, max_values, value_type)
    try:
        outs = [g.run() for _ in range(runs)]
    finally:
        g.release()
    for i, got in enumerate(outs):
        assert_same(got, want, (what, i))
    assert outs[0].stats.h2d_bytes == want.stats.h2d_bytes and outs[0].stats.kernel_launches == want.stats.kernel_launches, what
    if want.n_keys > 0:
        for i, got in enumerate(outs[1:], 1):
            s = got.stats
            assert s.h2d_bytes == 0 and s.scan_kernel_ms == 0 and s.device_ms > 0, (what, i, s)
            assert s.kernel_launches == want.stats.kernel_launches, (what, i, s.kernel_launches, want.stats.kernel_launches)
            assert s.d2h_bytes == replay_d2h(want, q), (what, i, s.d2h_bytes, replay_d2h(want, q))
    return outs


CAP_TEXT = "more distinct key values than bydb_group_key.max_values"


def refusal(err):
    """(code, text) of a refusal.  The cap error names the block whose value went over the cap first; discovery enters the blocks'
    values from many warps at once, so which block that is varies from one plain call to the next: its number is dropped (and
    required to be there)."""
    text = str(err)
    if CAP_TEXT in text:
        head, sep, block = text.rpartition(" (block #")
        assert sep and block.endswith(")") and block[:-1].isdigit(), text
        text = head
    return err.code, text


def refuses_alike(k, q, key, max_values, value_type, code):
    """the plain keyed call fails with `code`; the prepared form refuses at prepare with the same code and text, or else on every
    execution; afterwards the context still answers a plain query"""
    bydb, ctx = k.bydb, k.ctx
    with pytest.raises(bydb.BydbError) as pe:
        ctx.scan_agg_keyed(q, FAM, key, max_values, value_type)
    assert pe.value.code == code, (code, pe.value)
    try:
        g = ctx.prepare_keyed(q, FAM, key, max_values, value_type)
    except bydb.BydbError as e:
        assert refusal(e) == refusal(pe.value)
    else:
        try:
            for run in range(RUNS):
                with pytest.raises(bydb.BydbError) as e:
                    g.run()
                assert refusal(e.value) == refusal(pe.value), run
        finally:
            g.release()
    oq, pq = k.oquery(AGGS, [], I64_MIN, I64_MAX, None, k.usid[:1], None)
    assert_parity(ctx.scan_agg(pq), O.run_query(oq), AGGS, "plain query after a refusal")


class PScan(KScan):
    """KScan whose every query (checked against the oracle and the model) is also run as a prepared handle"""

    def query(self, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, sids=None, key=KT, max_values=256, order=None, ctx=""):
        want = super().query(aggs, preds, tmin, tmax, top, sids, key, max_values, order, ctx)
        _, q = self.oquery(aggs, list(preds), tmin, tmax, top, sids, order)
        run_prepared(self.bydb, self.ctx, q, key, max_values, 0, want, ctx)
        return want

    def fails(self, code, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, sids=None, key=KT, max_values=256, order=None):
        _, q = self.oquery(aggs, list(preds), tmin, tmax, None, sids, order)
        refuses_alike(self, q, key, max_values, 0, code)


class PScan64(KScan64):
    def query(self, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, sids=None, max_values=256, order=None, ctx=""):
        want = super().query(aggs, preds, tmin, tmax, top, sids, max_values, order, ctx)
        _, q = self.oquery(aggs, list(preds), tmin, tmax, top, sids, order)
        run_prepared(self.bydb, self.ctx, q, KT, max_values, self.bydb.capi.VT_INT64, want, ctx)
        return want

    def fails(self, code, preds=(), sids=None, key=KT, max_values=256, value_type=None, order=None):
        _, q = self.oquery(AGGS, list(preds), I64_MIN, I64_MAX, None, sids, order)
        refuses_alike(self, q, key, max_values, self.bydb.capi.VT_INT64 if value_type is None else value_type, code)


# ------------------------------------------------------------------ string keys
def run_series():
    """runs of 1..40 rows over seven values, nil and "" runs between them, a value that shows only in the last rows; an int64
    tag c, a dictionary tag s and a high-cardinality tag ps (a plain bytes block)"""
    cells = []
    for L in range(1, 41):
        cells += [[b"v0", b"v1", None, b"v2", b"", b"v3", b"v4"][L % 7]] * L
    ss = [mk(900, cells + [b"late"] * 3), mk(901, cells[::-1]), mk(902, cells[100:400], row0=50)]
    for s in ss:
        s.tags["c"] = (np.arange(s.n, dtype=np.int64) % 11, np.zeros(s.n, bool))
        s.tags["s"] = [b"x" if r % 5 else b"y" for r in range(s.n)]
        s.tags["ps"] = [b"p%05d" % (r * 7 % 997) for r in range(s.n)]
    return ss


def test_string_keys(bydb, gpu_ctx):
    """nil and "" as one key, a late value, run lengths 1..40, dictionary / int64 / plain-string predicates, time ranges that cut
    blocks, Top-N both ways, series groups x values"""
    P = O.Pred
    ss = run_series()
    with PScan(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={900: 1, 901: 0, 902: 1}) as k:
        got = k.query(ctx="runs")
        assert b"late" in got.key and b"" in got.key and len(got.key) > got.n_keys
        k.query(preds=[P(FAM, "s", O.OP_EQ, b"x")], ctx="runs: dictionary predicate")
        k.query(preds=[P(FAM, "c", O.OP_LT, 4)], ctx="runs: int64 predicate")
        k.query(preds=[P(FAM, "ps", O.OP_GE, b"p00500")], ctx="runs: plain-string predicate")
        k.query(tmin=T0 + 37 * STEP, tmax=T0 + 700 * STEP, ctx="runs: cut")
        for desc in (True, False):
            k.query(aggs=[("i", COUNT), ("f", MAX)], top=(3, 0, desc), ctx="runs: top")
            k.query(aggs=[("f", SUM), ("i", MIN)], top=(50, 1, desc), ctx="runs: top over all")
    ss = order_series()
    with PScan(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={10: 2, 11: 0, 12: 3, 13: 1, 14: 2}) as k:
        k.query(ctx="order")
        k.query(tmin=T0 + 33 * STEP, tmax=T0 + 8200 * STEP, ctx="order: cut")
        k.query(preds=[P(FAM, "dod", O.OP_GE, 150)], ctx="order: DoD predicate")


def test_row_path_types(bydb, gpu_ctx):
    """BYDB_Q_ROW_PATH_TYPES: the count over a float field comes back float, on the plain call and on every replay"""
    ss = run_series()
    with PScan(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        _, q = k.oquery([("f", COUNT), ("i", COUNT), ("f", MEAN)], [], I64_MIN, I64_MAX, None, None)
        q = dataclasses.replace(q, flags=bydb.capi.Q_ROW_PATH_TYPES)
        want = gpu_ctx.scan_agg_keyed(q, FAM, KT, 256)
        assert want.is_float.tolist() == [True, False, True]
        run_prepared(bydb, gpu_ctx, q, KT, 256, 0, want, "row path types")


def test_parts_lanes_and_absent_tag(bydb, gpu_ctx):
    """two time-disjoint parts in both orders; raw-cell float pages (the slow lane), a binary key, a key tag the part lacks"""
    a, b = ab_parts()
    with PScan(bydb, gpu_ctx, [(build_keyed(a), a), (build_keyed(b), b)], groups={20: 0, 21: 0}) as k:
        for order in ([0, 1], [1, 0]):
            k.query(order=order, ctx=f"parts {order}")
    ss = lane_series()
    with PScan(bydb, gpu_ctx, [(build_keyed(ss, binary=("bk",)), ss)], groups={s.sid: s.sid % 2 for s in ss}) as k:
        got = k.query(aggs=[("i", SUM), ("fx", MAX), ("fx", SUM), ("rn", COUNT)], ctx="lanes")
        assert got.stats.blocks_slow_lane > 0
        k.query(aggs=[("i", SUM), ("f", MEAN)], key="bk", ctx="binary key")
        got = k.query(aggs=[("i", SUM), ("fx", MAX)], key="nosuchtag", ctx="absent tag")
        assert got.key == [b""] * len(got.key) and got.n_keys == 1


# ------------------------------------------------------------------ int64 keys
@pytest.mark.parametrize("kind", ["const", "dc_neg", "d1", "wide", "dod", "raw"])
def test_int64_keys(bydb, gpu_ctx, kind):
    """Const, DeltaConst, Delta (narrow and wide), DoD and raw-cell key pages; nil -> 0 in the raw one and in a part without the key"""
    ss = kind_series(kind)
    with PScan64(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={s.sid: s.sid % 2 for s in ss}) as k:
        k.query(aggs=[("i", SUM), ("i", COUNT), ("f", MAX)], tmin=T0 + 31 * STEP, ctx=kind)
        k.query(aggs=[("i", COUNT), ("f", SUM)], top=(2, 0, True), ctx=kind)


# ------------------------------------------------------------------ refusals
def test_string_key_refusals(bydb, gpu_ctx):
    """test_gpu_keyed.test_cap_and_limits' refusals: above the cap, max_values 257, a 257-value (plain) page, a 65-byte value,
    8 / 9 predicates, overlapping parts"""
    ss = limit_series()
    P, E = O.Pred, bydb.capi
    seven = [P(FAM, "c", O.OP_GE, -5), P(FAM, "c", O.OP_LE, 5), P(FAM, "c", O.OP_NE, 9), P(FAM, "c", O.OP_GT, -9),
             P(FAM, "c", O.OP_LT, 9), P(FAM, "c", O.OP_EQ, 1), P(FAM, "nope", O.OP_NE, b"x")]
    with PScan(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        assert k.query(sids=[40], max_values=0, ctx="cap64").n_keys == 64
        k.fails(E.ENOMEM, sids=[40, 41], max_values=0)
        k.fails(E.ENOMEM, sids=[41, 42], max_values=1)
        k.fails(E.ENOMEM, sids=[41, 43, 44], max_values=256)
        k.fails(E.EINVAL, sids=[40], max_values=257)
        k.fails(E.ENOMEM, sids=[45], preds=[P(FAM, "c", O.OP_EQ, 1)], max_values=8)
        k.fails(E.ENOTSUP, sids=[46])
        k.fails(E.ENOTSUP, sids=[47])
        k.query(sids=[40, 45], preds=seven, ctx="seven predicates")
        k.fails(E.ENOTSUP, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)])
        k.fails(E.EINVAL, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)] * 2)
    over = [mk(40, [b"a00", b"late"] * 20, row0=30)]
    over[0].tags["c"] = (np.ones(40, np.int64), np.zeros(40, bool))
    with PScan(bydb, gpu_ctx, [(build_keyed(ss), ss), (build_keyed(over, 2), over)]) as k:
        k.fails(E.ENOTSUP, sids=[40])


def test_int64_key_refusals(bydb, gpu_ctx):
    """test_gpu_keyed_int64.test_int64_key_cap_and_refusals' refusals: the caps, a page of 8193 values, 8 predicates, the wrong
    key type and unknown value types, overlapping parts"""
    ss = cap_series()
    P, E = O.Pred, bydb.capi
    with PScan64(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        k.fails(E.ENOMEM, sids=[40, 41], max_values=0)
        k.fails(E.ENOMEM, sids=[41, 42], max_values=1)
        k.fails(E.ENOMEM, sids=[41, 43, 44], max_values=256)
        k.fails(E.EINVAL, sids=[40], max_values=257)
        k.fails(E.ENOMEM, sids=[46])
        k.fails(E.ENOMEM, sids=[47], max_values=1)
        k.fails(E.ENOMEM, sids=[48], max_values=3)
        seven = [P(FAM, "c", O.OP_GE, -5), P(FAM, "c", O.OP_LE, 5), P(FAM, "c", O.OP_NE, 9), P(FAM, "c", O.OP_GT, -9),
                 P(FAM, "c", O.OP_LT, 9), P(FAM, "s", O.OP_EQ, b"y"), P(FAM, "nope", O.OP_NE, b"x")]
        k.fails(E.ENOTSUP, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)])
        k.fails(E.EINVAL, sids=[40], key="s")
        for vt in (0, E.VT_STR, E.VT_FLOAT64, 99):
            k.fails(E.EINVAL, sids=[40], value_type=vt)
    over = [mk64(40, [1, 2] * 20, row0=30, tags={"c": (np.ones(40, np.int64), np.zeros(40, bool)), "s": [b"y"] * 40})]
    with PScan64(bydb, gpu_ctx, [(build_keyed(ss), ss), (build_keyed(over, 2), over)]) as k:
        k.fails(E.ENOTSUP, sids=[40])


# ------------------------------------------------------------------ parts coming and going
def _key_part(keys_of):
    ss = [mk(sid, keys) for sid, keys in keys_of.items()]
    return build_keyed(ss), np.array(sorted(keys_of), dtype=np.uint64)


def _q(bydb, h, usid, **kw):
    return bydb.Query([h], usid, [("i", SUM), ("i", COUNT), ("f", MAX)], series_group=(np.arange(usid.size) % 2).astype(np.int32),
                      n_groups=2, **kw)


def test_parts_change_between_executions(bydb, gpu_ctx):
    """Another part registered and released between replays leaves the captured step standing; the handle's own part released
    gives the plain call's ENOENT on every execution; the part id registered again with other data (a key value that did not
    exist before) is answered, by a new handle, with the new key table; a query that selects no block answers with no rows."""
    part, usid = _key_part({1: [b"a", b"b"] * 30, 2: [b"b", None] * 30})
    other, _ = _key_part({1: [b"a", b"new"] * 40, 3: [b"z"] * 10})
    pid = _next_pid()
    h = gpu_ctx.register_part(pid, part.files())
    g = gpu_ctx.prepare_keyed(_q(bydb, h, usid), FAM, KT, 16)
    try:
        want = gpu_ctx.scan_agg_keyed(_q(bydb, h, usid), FAM, KT, 16)
        assert want.n_keys == 3
        for run in range(3):
            assert_same(g.run(), want, run)
        h2 = gpu_ctx.register_part(_next_pid(), other.files())
        assert_same(g.run(), want, "after a registration")
        gpu_ctx.release_part(h2)
        assert_same(g.run(), want, "after a release of another part")
        gpu_ctx.release_part(h)
        with pytest.raises(bydb.BydbError) as pe:
            gpu_ctx.scan_agg_keyed(_q(bydb, h, usid), FAM, KT, 16)
        for _ in range(2):
            with pytest.raises(bydb.BydbError) as e:
                g.run()
            assert e.value.code == pe.value.code == bydb.capi.ENOENT
    finally:
        g.release()
    h = gpu_ctx.register_part(pid, other.files())
    try:
        usid2 = np.array([1, 3], dtype=np.uint64)
        want = gpu_ctx.scan_agg_keyed(_q(bydb, h, usid2), FAM, KT, 16)
        assert b"new" in want.key
        run_prepared(bydb, gpu_ctx, _q(bydb, h, usid2), KT, 16, 0, want, "new data")
        for name, q in (("series the part does not hold", _q(bydb, h, usid2 + 1000)),
                        ("time range before the part", _q(bydb, h, usid2, tmin=T0 - 100 * STEP, tmax=T0 - STEP))):
            want = gpu_ctx.scan_agg_keyed(q, FAM, KT, 16)
            assert want.n_keys == 0 and want.rows.size == 0, name
            for got in run_prepared(bydb, gpu_ctx, q, KT, 16, 0, want, name):
                assert got.key == [] and got.n_keys == 0
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ interleaving
def test_handles_interleaved_and_concurrent(bydb, gpu_ctx):
    """two keyed handles and a plain prepared handle alternating; threads running different handles at once; a handle executed
    behind scan_agg_keyed and scan_partials_keyed calls on the same parts"""
    ss = run_series()
    part = build_keyed(ss)
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        usid = np.array([900, 901, 902], dtype=np.uint64)
        grp = np.array([0, 1, 0], dtype=np.int32)
        qa = bydb.Query([h], usid, [("i", SUM), ("f", MAX)], series_group=grp, n_groups=2)
        qb = bydb.Query([h], usid[1:], [("i", COUNT), ("f", MEAN)], preds=[bydb.Pred(FAM, "s", O.OP_EQ, b"x")], top_n=4)
        qp = bydb.Query([h], usid, [("i", SUM), ("i", COUNT)], series_group=grp, n_groups=2)
        wa, wb = gpu_ctx.scan_agg_keyed(qa, FAM, KT, 64), gpu_ctx.scan_agg_keyed(qb, FAM, "s", 64)
        wp = gpu_ctx.scan_agg(qp)
        ga, gb, gp = gpu_ctx.prepare_keyed(qa, FAM, KT, 64), gpu_ctx.prepare_keyed(qb, FAM, "s", 64), gpu_ctx.prepare_graph(qp)
        try:
            for rnd in range(6):
                assert_same(ga.run(), wa, ("a", rnd))
                pr = gp.run()
                assert pr.val_i64.tolist() == wp.val_i64.tolist() and pr.group_id.tolist() == wp.group_id.tolist(), rnd
                assert_same(gb.run(), wb, ("b", rnd))
            errors = []

            def worker(g, want, name):
                try:
                    for i in range(8):
                        assert_same(g.run(), want, (name, i))
                except Exception as e:   # noqa: BLE001 -- reported by the main thread
                    errors.append(e)
            ths = [threading.Thread(target=worker, args=(g, w, n)) for g, w, n in ((ga, wa, "a"), (gb, wb, "b"))]
            for t in ths:
                t.start()
            for _ in range(8):
                gpu_ctx.scan_agg_keyed(qa, FAM, KT, 64)
            for t in ths:
                t.join()
            assert not errors, errors
            for rnd in range(3):
                gpu_ctx.scan_agg_keyed(qb, FAM, KT, 64)
                gpu_ctx.scan_partials_keyed(qa, FAM, KT, 64)
                assert_same(ga.run(), wa, ("after plain keyed calls", rnd))
                assert_same(gb.run(), wb, ("after plain keyed calls", rnd))
        finally:
            ga.release()
            gb.release()
            gp.close()
    finally:
        gpu_ctx.release_part(h)

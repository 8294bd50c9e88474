"""-m gpu: the prepared group-by on a tuple of 2..4 stored tags (bydb_query_prepare_keys_wide, DESIGN.md 4.6), and the operators
routing two to four stored GroupBy keys to bydb_scan_agg_keys_wide.

A tuple handle's first execution runs the unprepared tuple path; the second runs its discovery, scan and order once with the key
list, captures the reset, tuple scan, order, fold and the form's tail as one CUDA graph and answers from its first replay; later
ones replay.  Every handle here runs at least five times in each form, and every execution must give what bydb_scan_agg_keys_wide /
bydb_scan_partials_keys_wide give on the same context: rows in the same order, series groups and each tag's key bytes per row,
values bit for bit, n_tuples, each tag's value count and the scan counters, one set of key tables across the replays of a capture,
and the replay stats bydb_gpu.h states.  The unprepared answers are held to the oracle in test_gpu_keys_wide*.py and, for the
code-packing fixture, here too, so every replay is.
"""
import ctypes
import dataclasses
import importlib
import re
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM
from tests.test_gpu_keyed_prepared import COUNTERS, a256
from tests.test_gpu_keys_wide import FAM, INT, STR, Parts, grid_series, int_tag, model_parts, pair_parts
from tests.test_gpu_keys_wide_boundaries import PACK_AGGS, PACK_MIX, Tup, against_oracle, gkeys, pack_part, pack_series

pytestmark = pytest.mark.gpu

RUNS = 5
PAIR = [(FAM, "a", STR), (FAM, "b", INT)]


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def parts_of(x):
    """(key, n_tuples, key_tables, stats) of a finalised answer or a partial answer"""
    if isinstance(x, dict):
        return x["key"], x["n_tuples"], x["key_tables"], x["stats"]
    return x.key, x.n_tuples, x.key_tables, x.stats


def assert_same(got, want, what):
    """one execution against the unprepared tuple call: rows, groups, key tuples, values as bit patterns, n_tuples, each tag's
    table (as a set: its order is not part of the contract), counters"""
    if isinstance(want, dict):
        for k in ("group_id", "is_float", "val_i64", "cnt_i64", "val_f64", "cnt_f64"):
            assert _bits(got[k]) == _bits(want[k]), (what, k)
    else:
        assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), what
        assert got.is_float.tolist() == want.is_float.tolist(), what
        assert _bits(got.val_i64) == _bits(want.val_i64) and _bits(got.val_f64) == _bits(want.val_f64), what
    gk, gn, gt, gs = parts_of(got)
    wk, wn, wt, ws = parts_of(want)
    assert gk == wk and gn == wn, (what, gn, wn)
    assert [sorted(t) for t in gt] == [sorted(t) for t in wt], what
    assert {k: getattr(gs, k) for k in COUNTERS} == {k: getattr(ws, k) for k in COUNTERS}, what


def replay_stats(want, q, n_tags, C, partial):
    """bydb_gpu.h's kernel_launches and d2h_bytes of a replay, from the unprepared call's answer `want` (C present composite groups,
    blocks in the parts): discovery's (K + 1) * 2 + 3 launches give way to the reset kernel; the partial tail adds the copy kernel;
    C = 0 launches no fold"""
    plain = parts_of(want)[3].kernel_launches
    disc = (n_tags + 1) * 2 + 3
    if C == 0:
        return plain - disc, 256
    if partial:
        A, F_ = len(q.aggs), len({f for f, _ in q.aggs})
        return plain - disc + 2, a256(8 * C) + 256 + 8 + 8 * F_ + len(want["group_id"]) * (8 + 16 * A)
    A = len(q.aggs)
    R = min(q.top_n, C) if q.top_n > 0 else C
    return plain - disc + 1, a256(16) + a256(A) + a256(4 * R) + a256(8 * R) + 2 * a256(8 * R * A) + 256 + 8 * C


def run_handle(ctx, q, keys, max_values, what="", runs=RUNS, g=None):
    """a tuple handle run `runs` times in each form (finalised, then partial), each execution against a fresh unprepared call; the
    replays also against the stats formulas and one set of key tables.  -> (finalised answers, partial answers)"""
    own = g is None
    g = g or ctx.prepare_keys_wide(q, keys, max_values)
    outs = {}
    try:
        for partial in (False, True):
            plain_fn = ctx.scan_partials_keys_wide if partial else ctx.scan_agg_keys_wide
            C = len(ctx.scan_partials_keys_wide(q, keys, max_values)["group_id"])
            got_all = []
            for i in range(runs):
                got = g.run_partials() if partial else g.run()
                want = plain_fn(q, keys, max_values)
                assert_same(got, want, (what, partial, i))
                got_all.append(got)
                _, n_tuples, _, st = parts_of(got)
                if i == 0 or n_tuples == 0:   # the first execution of a form runs unprepared; T = 0 needs no graph
                    if n_tuples == 0 and i > 0:
                        assert (st.kernel_launches, st.d2h_bytes, st.h2d_bytes) == (0, 0, 0), (what, st)
                    continue
                launches, d2h = replay_stats(want, q, len(keys), C, partial)
                assert st.h2d_bytes == 0 and st.scan_kernel_ms == 0 and st.device_ms > 0, (what, partial, i, st)
                assert (st.kernel_launches, st.d2h_bytes) == (launches, d2h), (what, partial, i, st.kernel_launches, launches, st.d2h_bytes, d2h)
            if runs > 2:   # one set of key tables across the capture's answer and its replays
                assert len({tuple(tuple(t) for t in parts_of(o)[2]) for o in got_all[1:]}) == 1, what
            outs[partial] = got_all
    finally:
        if own:
            g.release()
    return outs[False], outs[True]


def pair_fixture():
    p1, p2 = pair_parts()
    return [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]


# ------------------------------------------------------------------ the query cases of test_gpu_keys_wide.py
def test_pair_queries(bydb, gpu_ctx):
    """(string, int64) over two parts: all rows, a time cut with a predicate, two parts in the other order, Top, eight predicates
    with MEAN, and the row path's typing"""
    with Parts(bydb, gpu_ctx, pair_fixture()) as P:
        fin, _ = run_handle(gpu_ctx, P.q(), PAIR, 4096, "all rows")
        assert fin[-1].n_tuples > 0 and len(fin[-1].key_tables) == 2
        run_handle(gpu_ctx, P.q(tmin=T0 + 100 * STEP, tmax=T0 + 8500 * STEP, preds=[O.Pred(FAM, "z", O.OP_NE, b"z1")]), PAIR, 4096,
                   "time cut")
        run_handle(gpu_ctx, P.q(handles=P.handles[::-1]), PAIR, 4096, "parts reversed")
        run_handle(gpu_ctx, P.q(top=(7, 1, True)), PAIR, 4096, "top")
        eight = [O.Pred(FAM, "z", O.OP_NE, b"zz%d" % j) for j in range(7)] + [O.Pred(FAM, "a", O.OP_GE, b"a1")]
        q = P.q(preds=eight, aggs=[("i", MEAN), ("f", MEAN), ("f", COUNT), ("i", MAX)])
        assert len(q.preds) == 8
        run_handle(gpu_ctx, q, PAIR, 4096, "eight predicates, MEAN")
        run_handle(gpu_ctx, dataclasses.replace(q, flags=bydb.capi.Q_ROW_PATH_TYPES), PAIR, 4096, "row path types")


MODEL_KEYS = [(("a", "b"), (STR, INT)), (("a", "b", "e"), (STR, INT, STR)), (("d", "e", "b", "a"), (INT, STR, INT, STR))]


@pytest.mark.parametrize("keys", MODEL_KEYS, ids=["-".join(k[0]) for k in MODEL_KEYS])
def test_two_three_four_tags(bydb, gpu_ctx, keys):
    """2, 3 and 4 tags of mixed types, over a part whose later part lacks the int64 tags"""
    p1, p2 = model_parts()
    with Parts(bydb, gpu_ctx, [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]) as P:
        gk = [(FAM, t, vt) for t, vt in zip(*keys)]
        fin, _ = run_handle(gpu_ctx, P.q(groups={2: 0, 4: 1, 6: 0, 7: 1, 11: 0, 13: 1}), gk, 4096, f"{keys[0]}")
        assert fin[-1].n_tuples > 0 and len(fin[-1].key_tables) == len(gk)
        assert all(len(k) == len(gk) for k in fin[-1].key)


def test_oracle_tuples_65536_and_top_both_ways(bydb, gpu_ctx):
    """the code-packing fixture (four tags of 65,536 values, 65,536 tuples): every replay against the oracle grouped by the same
    tuple, and Top-N both ways with C > 2048"""
    ss = pack_series()
    gid = {s.sid: s.sid % 3 for s in ss}
    with Tup(bydb, gpu_ctx, [(pack_part(), ss)], gid) as T:
        sids = list(gid)
        oq, q = T.oquery(PACK_MIX, sids, PACK_AGGS)
        fin, rows = run_handle(gpu_ctx, q, gkeys(PACK_MIX), 65536, "65,536 tuples")
        want = O.run_query(oq)
        for got in fin:
            against_oracle(got, want, PACK_AGGS, 0, "prepared 65,536 tuples")
        assert fin[-1].n_tuples == 65536 == fin[-1].group_id.size and len(rows[-1]["group_id"]) == 65536
        for desc in (True, False):
            oq, q = T.oquery(PACK_MIX, sids, PACK_AGGS, top=(17, 1, desc))
            fin, _ = run_handle(gpu_ctx, q, gkeys(PACK_MIX), 65536, f"top desc={desc}")
            assert fin[-1].group_id.size == 17
            against_oracle(fin[-1], O.run_query(oq), PACK_AGGS, 0, f"prepared top desc={desc}")


# ------------------------------------------------------------------ T = 0, C = 0, C = 1
def test_empty_and_single_answers(bydb, gpu_ctx):
    """no block selected (T = 0: no graph, no tuples, zero stats); blocks selected but no row survives (C = 0: a graph that answers
    no rows, the key tables all the same); one composite group (C = 1)"""
    ss = [grid_series(1, {"a": [b"k%d" % (x % 3) for x in range(300)], "b": int_tag([x % 2 for x in range(300)]), "z": [b"z"] * 300}),
          grid_series(2, {"a": [b"k1"] * 300, "b": int_tag([5] * 300), "z": [b"y"] * 300})]
    with Parts(bydb, gpu_ctx, [(K.build_keyed(ss), ss)]) as P:
        base = P.q(aggs=[("i", SUM), ("f", MAX)])
        for name, q in (("series the part does not hold", P.q(aggs=[("i", SUM)], sids=[7, 8])),
                        ("time range before the part", dataclasses.replace(base, tmin=T0 - 100 * STEP, tmax=T0 - STEP))):
            fin, rows = run_handle(gpu_ctx, q, PAIR, 1000, name)
            for got in fin:
                assert got.n_tuples == 0 and got.key == [] and got.group_id.size == 0 and got.key_tables == [[], []], name
            for got in fin[1:] + rows[1:]:
                assert parts_of(got)[3] == bydb.capi.Stats(), name
        fin, rows = run_handle(gpu_ctx, dataclasses.replace(base, preds=[bydb.Pred(FAM, "z", O.OP_EQ, b"none")]), PAIR, 1000, "C = 0")
        assert all(g.n_tuples == 7 and g.group_id.size == 0 for g in fin) and all(len(r["group_id"]) == 0 for r in rows)
        fin, rows = run_handle(gpu_ctx, P.q(sids=[2]), PAIR, 1000, "C = 1")
        assert fin[-1].key == [(b"k1", (5).to_bytes(8, "little"))] and len(rows[-1]["group_id"]) == 1


# ------------------------------------------------------------------ refusals
def refusal(err):
    """(code, text) of a refusal, without the number of the block a device error names (it varies between unprepared calls too)"""
    return err.code, re.sub(r" \(block #\d+\)", " (block #)", str(err))


def refuses_alike(bydb, ctx, q, keys, max_values, code, sane):
    """the unprepared tuple call fails with `code`; the prepared form refuses at prepare with the same code and text, or else on
    every execution in both forms; afterwards the context still answers the plain query `sane`"""
    with pytest.raises(bydb.BydbError) as pe:
        ctx.scan_agg_keys_wide(q, keys, max_values)
    assert pe.value.code == code, (code, pe.value)
    try:
        g = ctx.prepare_keys_wide(q, keys, max_values)
    except bydb.BydbError as e:
        assert refusal(e) == refusal(pe.value)
        return "prepare"
    try:
        for run in range(RUNS):
            with pytest.raises(bydb.BydbError) as e:
                g.run_partials() if run % 2 else g.run()
            assert refusal(e.value) == refusal(pe.value), run
    finally:
        g.release()
    assert ctx.scan_agg(sane).group_id.size > 0
    return "execution"


def test_refusals(bydb, gpu_ctx):
    """every argument refusal at prepare, in the unprepared call's order and with its codes; the cap (ENOMEM), a tag of the wrong
    type (EINVAL), 257 tuples in a block, a plain string page, a 65-byte value, an int64 column of 300 values in a block and parts
    that overlap in time (ENOTSUP) at every execution, alike with the unprepared call"""
    E = bydb.capi
    with Parts(bydb, gpu_ctx, pair_fixture()) as P:
        q = P.q()
        for keys, cap in ((PAIR[:1], 4096), (PAIR + [(FAM, "c", STR), (FAM, "z", STR), (FAM, "k0", STR)], 4096),
                          (PAIR + [(FAM, "a", STR)], 4096), (PAIR, 65537), ([(FAM, "a", 9), (FAM, "b", INT)], 4096)):
            assert refuses_alike(bydb, gpu_ctx, q, keys, cap, E.EINVAL, q) == "prepare", keys
        nine = P.q(preds=[O.Pred(FAM, "z", O.OP_NE, b"q%d" % j) for j in range(9)])
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg_keys_wide(nine, PAIR, 4096)
        assert refuses_alike(bydb, gpu_ctx, nine, PAIR, 4096, e.value.code, q) == "prepare"
        # a key's own max_values: the binding passes 0, so go through the structures
        capi = importlib.import_module(bydb.__name__ + ".capi")
        keep = []
        gks = capi._group_keys(PAIR, 4096, keep)
        gks.keys[1].max_values = 8
        h = ctypes.c_void_p()
        assert capi.load_library().bydb_query_prepare_keys_wide(gpu_ctx._h, ctypes.byref(capi._mk_query(q, keep)), ctypes.byref(gks),
                                                                 ctypes.byref(h)) == E.EINVAL and not h.value
        assert refuses_alike(bydb, gpu_ctx, q, PAIR, 10, E.ENOMEM, q) == "execution"
        assert refuses_alike(bydb, gpu_ctx, q, [(FAM, "a", INT), (FAM, "b", INT)], 4096, E.EINVAL, q) == "execution"
    xs = [b"x%02d" % (i // 16) for i in range(256)]
    ys = [b"y%02d" % (i % 16) for i in range(256)]
    cases = [("257 tuples", [grid_series(1, {"a": xs + [b"x00"], "b": int_tag([i % 16 for i in range(256)] + [99])})]),
             ("plain page", [grid_series(1, {"a": [b"p%03d" % i for i in range(300)], "b": int_tag([0] * 300)})]),
             ("65-byte value", [grid_series(1, {"a": [b"x" * 65, b"y"] * 10, "b": int_tag(list(range(20)))})]),
             ("int64 column of 300 values", [grid_series(1, {"a": [b"q"] * 300, "b": int_tag(list(range(300)))})])]
    assert len(set(zip(xs, ys))) == 256
    with Parts(bydb, gpu_ctx, pair_fixture()) as S:
        sane = S.q()
        for name, ss in cases:
            with Parts(bydb, gpu_ctx, [(K.build_keyed(ss), ss)]) as P:
                assert refuses_alike(bydb, gpu_ctx, P.q(aggs=[("i", COUNT)]), PAIR, 4096, E.ENOTSUP, sane) == "execution", name
        overlap = [grid_series(3, {"a": [b"o"] * 10, "b": int_tag([1] * 10), "z": [b"z"] * 10})]
        with Parts(bydb, gpu_ctx, [S.parts[0], (K.build_keyed(overlap, 3), overlap)]) as P:
            assert refuses_alike(bydb, gpu_ctx, P.q(), PAIR, 4096, E.ENOTSUP, sane) == "execution"


def test_cross_form_calls(bydb, gpu_ctx):
    """a one-key executor on a tuple handle, and a tuple executor on a one-key handle: BYDB_EINVAL naming the executor to use; the
    handles still answer in their own form afterwards"""
    capi = importlib.import_module(bydb.__name__ + ".capi")
    L = capi.load_library()
    with Parts(bydb, gpu_ctx, pair_fixture()) as P:
        q = P.q()
        gt = gpu_ctx.prepare_keys_wide(q, PAIR, 4096)
        g1 = gpu_ctx.prepare_keyed_wide(q, FAM, "a", 4096)
        try:
            for fn, h, out, name in ((L.bydb_scan_agg_keyed_prepared, gt, capi._KeyedResult(), "bydb_scan_agg_keys_prepared"),
                                     (L.bydb_scan_partials_keyed_prepared, gt, capi._KeyedPartialRows(), "bydb_scan_partials_keys_prepared"),
                                     (L.bydb_scan_agg_keys_prepared, g1, capi._KeysResult(), "bydb_scan_agg_keyed_prepared"),
                                     (L.bydb_scan_partials_keys_prepared, g1, capi._KeysPartialRows(), "bydb_scan_partials_keyed_prepared")):
                for _ in range(2):
                    assert fn(gpu_ctx._h, h._h, ctypes.byref(out)) == capi.EINVAL
                    assert name in L.bydb_last_error().decode(), L.bydb_last_error()
            run_handle(gpu_ctx, q, PAIR, 4096, "tuple handle after refused calls", g=gt)
            assert g1.run().key == gpu_ctx.scan_agg_keyed_wide(q, FAM, "a", 4096).key
        finally:
            gt.release()
            g1.release()


# ------------------------------------------------------------------ parts changing under a handle
def test_parts_change_between_executions(bydb, gpu_ctx):
    """another part registered and released leaves the step standing; the handle's own part released gives the plain call's
    ENOENT on every execution; the part id registered again with a new tuple is discovered and captured by a new handle"""
    mk = lambda sid, a, b: grid_series(sid, {"a": a, "b": int_tag(b)})   # noqa: E731
    part = K.build_keyed([mk(1, [b"a", b"b"] * 300, [1, 2] * 300), mk(2, [b"b", None] * 300, [None, 3] * 300)])
    other = K.build_keyed([mk(1, [b"a", b"new"] * 400, [1, 9] * 400), mk(3, [b"z"] * 100, [0] * 100)])
    pid = K._next_pid()
    usid = np.array([1, 2, 3], np.uint64)
    qf = lambda hh: bydb.Query([hh], usid, [("i", SUM), ("i", COUNT), ("f", MAX)], series_group=np.array([0, 1, 0], np.int32), n_groups=2)  # noqa: E731
    h = gpu_ctx.register_part(pid, part.files())
    g = gpu_ctx.prepare_keys_wide(qf(h), PAIR, 1000)
    try:
        want = gpu_ctx.scan_agg_keys_wide(qf(h), PAIR, 1000)
        assert want.n_tuples == 4
        for run in range(3):
            assert_same(g.run(), want, run)
        h2 = gpu_ctx.register_part(K._next_pid(), other.files())
        assert_same(g.run(), want, "after a registration")
        gpu_ctx.release_part(h2)
        got = g.run()
        assert_same(got, want, "after a release of another part")
        assert got.stats.h2d_bytes == 0, "the step stands"
        gpu_ctx.release_part(h)
        with pytest.raises(bydb.BydbError) as pe:
            gpu_ctx.scan_agg_keys_wide(qf(h), PAIR, 1000)
        for partial in (False, True, False):
            with pytest.raises(bydb.BydbError) as e:
                g.run_partials() if partial else g.run()
            assert e.value.code == pe.value.code == bydb.capi.ENOENT
        h_old, h = h, gpu_ctx.register_part(pid, other.files())
        assert h != h_old
        with pytest.raises(bydb.BydbError) as e:   # a handle names a part object, not its id
            g.run()
        assert e.value.code == bydb.capi.ENOENT
        fin, _ = run_handle(gpu_ctx, qf(h), PAIR, 1000, "new data under the same id")
        assert (b"new", (9).to_bytes(8, "little")) in fin[-1].key
    finally:
        g.release()
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ forms and threads
def test_forms_alternating_and_threads(bydb, gpu_ctx):
    """one handle alternating its two forms (each switch drops the step and captures the other); two tuple handles and a one-key
    wide handle run from threads at once, next to unprepared calls"""
    with Parts(bydb, gpu_ctx, pair_fixture()) as P:
        qa = P.q(aggs=[("i", SUM), ("f", MEAN)], groups={3: 0, 5: 1, 8: 2, 9: 0, 12: 1, 20: 2, 30: 0})
        qb = P.q(aggs=[("i", COUNT), ("f", MIN)], preds=[O.Pred(FAM, "z", O.OP_NE, b"z1")], top=(40, 0, True))
        kb = [(FAM, "b", INT), (FAM, "z", STR), (FAM, "a", STR)]
        ga = gpu_ctx.prepare_keys_wide(qa, PAIR, 2000)
        gb = gpu_ctx.prepare_keys_wide(qb, kb, 2000)
        gn = gpu_ctx.prepare_keyed_wide(qa, FAM, "a", 2000)
        try:
            wa, wb = gpu_ctx.scan_agg_keys_wide(qa, PAIR, 2000), gpu_ctx.scan_agg_keys_wide(qb, kb, 2000)
            pa = gpu_ctx.scan_partials_keys_wide(qa, PAIR, 2000)
            wn = gpu_ctx.scan_agg_keyed_wide(qa, FAM, "a", 2000)
            for rnd in range(6):
                for partial in ((False, True) if rnd % 2 else (True, False)):
                    if partial:
                        assert_same(ga.run_partials(), pa, ("a partial", rnd))
                    else:
                        assert_same(ga.run(), wa, ("a", rnd))
            errors = []

            def worker(g, check, name):
                try:
                    for i in range(8):
                        check(g, i)
                except Exception as e:   # noqa: BLE001 -- reported by the main thread
                    errors.append((name, e))

            def one_key(g, i):
                got = g.run()
                assert got.key == wn.key and _bits(got.val_i64) == _bits(wn.val_i64) and _bits(got.val_f64) == _bits(wn.val_f64), i
            ths = [threading.Thread(target=worker, args=a) for a in ((ga, lambda g, i: assert_same(g.run(), wa, ("a", i)), "a"),
                                                                     (gb, lambda g, i: assert_same(g.run(), wb, ("b", i)), "b"),
                                                                     (gn, one_key, "one key"))]
            for t in ths:
                t.start()
            for _ in range(4):
                gpu_ctx.scan_agg_keys_wide(qa, PAIR, 2000)
                gpu_ctx.scan_partials_keys_wide(qb, kb, 2000)
            for t in ths:
                t.join()
            assert not errors, errors
            run_handle(gpu_ctx, qb, kb, 2000, "b after threads", g=gb)
        finally:
            ga.release()
            gb.release()
            gn.release()


# ------------------------------------------------------------------ the Python operator
def _operator(bydb, P, key_cols, max_key_values, batch, top=None, limit=None, order_desc=False):
    """GPUScanAgg over the pair fixture: input columns svc (per series), a (string), b (int64), z (string), k0 (string), c (string),
    i, f; series in index order 3, 5, 8, ... with svc cycling over three values"""
    T = bydb.ColumnType
    cols = [bydb.ColumnDef("svc", bydb.ColumnRole.RoleTag, T.ColumnTypeString, FAM),
            bydb.ColumnDef("a", bydb.ColumnRole.RoleTag, T.ColumnTypeString, FAM),
            bydb.ColumnDef("b", bydb.ColumnRole.RoleTag, T.ColumnTypeInt64, FAM),
            bydb.ColumnDef("z", bydb.ColumnRole.RoleTag, T.ColumnTypeString, FAM),
            bydb.ColumnDef("k0", bydb.ColumnRole.RoleTag, T.ColumnTypeString, FAM),
            bydb.ColumnDef("c", bydb.ColumnRole.RoleTag, T.ColumnTypeString, FAM),
            bydb.ColumnDef("i", bydb.ColumnRole.RoleField, T.ColumnTypeInt64),
            bydb.ColumnDef("f", bydb.ColumnRole.RoleField, T.ColumnTypeFloat64)]
    aggs = [bydb.AggSpec("s", bydb.AggSum, 6), bydb.AggSpec("n", bydb.AggCount, 6), bydb.AggSpec("m", bydb.AggMax, 7)]
    sids = [int(s) for s in P.usid]
    scan = bydb.ScanSpec(parts=P.handles, series_ids=sids, series_tags={(FAM, "svc"): ["svc%d" % (j % 3) for j in range(len(sids))]},
                         max_key_values=max_key_values, order_desc=order_desc)
    op = bydb.GPUScanAgg(P.ctx, bydb.BatchSchema(cols), key_cols, aggs, scan, batch_size=batch, top=top, limit=limit)
    op.Init()
    return op, sids


def _drain(op):
    rows, n_batches = [], 0
    while True:
        b = op.NextBatch()
        if b is None:
            break
        n_batches += 1
        rows += [tuple(c[i] for c in b.Columns[:6]) + tuple(int(x) if not isinstance(x, float) else x for x in (c[i] for c in b.Columns[6:]))
                 for i in range(b.Len)]
    op.Close()
    return rows, n_batches


def test_operator_routes_stored_key_tuples(bydb, gpu_ctx):
    """a per-series key plus (string, int64) stored keys at max_key_values = 1000, in batches of 2, under Top and an offset / limit
    window, row by row against scan_agg_keys_wide called directly; four stored keys; a fifth stored key and order_desc refused"""
    with Parts(bydb, gpu_ctx, pair_fixture()) as P:
        svc_gid = {}
        for j in range(len(P.usid)):
            svc_gid.setdefault(j % 3, len(svc_gid))

        def direct(keys, per_series, top):
            groups = {int(s): (svc_gid[j % 3] if per_series else 0) for j, s in enumerate(P.usid)}
            q = P.q(aggs=[("i", SUM), ("i", COUNT), ("f", MAX)], groups=groups, top=top or (0, 0, True))
            return gpu_ctx.scan_agg_keys_wide(q, keys, 1000)

        def expect(r, key_cols, per_series, lo, hi):
            """the operator's rows [lo, hi) from the direct answer r: svc of the group's first series, the stored key columns
            decoded, null for a stored tag that is not a key, then the aggregates"""
            out = []
            for i in range(lo, min(hi, r.group_id.size)):
                cells = ["svc%d" % [j for j in range(3) if svc_gid[j] == r.group_id[i]][0] if per_series else "svc0"]
                for col in (1, 2, 3, 4, 5):
                    if col not in key_cols:
                        cells.append(None)
                        continue
                    k = r.key[i][key_cols.index(col)]
                    cells.append(int.from_bytes(k, "little", signed=True) if col == 2 else k.decode("utf-8", "surrogateescape"))
                out.append(tuple(cells) + (int(r.val_i64[i, 0]), int(r.val_i64[i, 1]), float(r.val_f64[i, 2])))
            return out

        op, _ = _operator(bydb, P, [0, 1, 2], 1000, 2)
        rows, nb = _drain(op)
        want = direct(PAIR, True, None)
        assert rows == expect(want, [1, 2], True, 0, want.group_id.size) and nb == (len(rows) + 1) // 2 and len(rows) > 2
        top = bydb.TopSpec(N=40, AggIndex=1, Desc=True)
        op, _ = _operator(bydb, P, [0, 1, 2], 1000, 2, top=top, limit=bydb.LimitSpec(Offset=5, Limit=20))
        rows, _ = _drain(op)
        want = direct(PAIR, True, (40, 1, True))
        assert len(rows) == 20 and rows == expect(want, [1, 2], True, 5, 25)
        four = [(FAM, "a", STR), (FAM, "b", INT), (FAM, "z", STR), (FAM, "k0", STR)]
        op, _ = _operator(bydb, P, [1, 2, 3, 4], 1000, 64)
        rows, _ = _drain(op)
        want = direct(four, False, None)
        assert rows == expect(want, [1, 2, 3, 4], False, 0, want.group_id.size) and len(rows) > 0
        for cols, kw, text in (([1, 2, 3, 4, 5], {}, f"{FAM}/c"), ([1, 2], dict(order_desc=True), "order_desc"),
                               ([1, 2], dict(), None)):
            op, _ = _operator(bydb, P, cols, 1000 if text else 256, 8, **kw)
            with pytest.raises(bydb.BydbError) as e:
                op.NextBatch()
            assert e.value.code == bydb.capi.ENOTSUP and (text or f"{FAM}/b") in str(e.value), e.value
            with pytest.raises(bydb.BydbError):   # sticky
                op.NextBatch()

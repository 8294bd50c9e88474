"""-m gpu: the prepared wide group-by on a stored tag (bydb_query_prepare_keyed_wide, DESIGN.md 4.6).

Its first execution runs the unprepared wide path; the second runs discovery, the scan and the order once, captures the reset,
scan, order, fold and the form's tail as one CUDA graph and answers from its first replay; later ones replay.  Every handle here
runs at least five times, in both forms, and every execution must give what bydb_scan_agg_keyed_wide /
bydb_scan_partials_keyed_wide give on the same context: rows in the same order, series groups and key bytes per row, values bit
for bit, n_keys and the scan counters, one key table across the replays of a capture, and the replay stats bydb_gpu.h states.
The unprepared answers are held to the oracle here (oracle_check) and in test_gpu_keyed_wide.py, so every replay is too.
"""
import dataclasses
import re
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, F, I, Series
from tests.test_gpu_keyed_prepared import COUNTERS, a256
from tests.test_gpu_keyed_wide import AGGS, FAM, KT, int_series, le, oracle_check, string_fixture, wide_fields

pytestmark = pytest.mark.gpu

RUNS = 5


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if np.asarray(a).dtype == np.float64 else np.asarray(a).dtype).tolist()


def assert_same(got, want, what):
    """one execution against the unprepared wide call: rows, groups, key bytes, values as bit patterns, n_keys, counters"""
    if isinstance(want, dict):
        for k in ("group_id", "is_float", "val_i64", "cnt_i64", "val_f64", "cnt_f64"):
            assert _bits(got[k]) == _bits(want[k]), (what, k)
        assert got["key"] == want["key"] and got["n_keys"] == want["n_keys"], what
        assert sorted(got["key_table"]) == sorted(want["key_table"]), what
        gs, ws = got["stats"], want["stats"]
    else:
        assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), what
        assert got.key == want.key and got.n_keys == want.n_keys, (what, got.n_keys, want.n_keys)
        assert got.is_float.tolist() == want.is_float.tolist(), what
        assert _bits(got.val_i64) == _bits(want.val_i64) and _bits(got.val_f64) == _bits(want.val_f64), what
        gs, ws = got.stats, want.stats
    assert {k: getattr(gs, k) for k in COUNTERS} == {k: getattr(ws, k) for k in COUNTERS}, what


def replay_stats(want, q, C, partial):
    """bydb_gpu.h's kernel_launches and d2h_bytes of a replay, from the unprepared call's answer `want` (C present composite groups):
    discovery's five launches give way to the reset kernel; the partial tail adds the copy kernel; C = 0 launches no fold"""
    plain = (want["stats"] if partial else want.stats).kernel_launches
    if C == 0:
        return plain - 5, 256
    if partial:
        A, F_ = len(q.aggs), len({f for f, _ in q.aggs})
        return plain - 3, a256(8 * C) + 256 + 8 + 8 * F_ + len(want["group_id"]) * (8 + 16 * A)
    A = len(q.aggs)
    R = min(q.top_n, C) if q.top_n > 0 else C
    return plain - 4, a256(16) + a256(A) + a256(4 * R) + a256(8 * R) + 2 * a256(8 * R * A) + 256 + 8 * C


def run_handle(bydb, ctx, q, key=KT, max_values=0, vt=0, what="", runs=RUNS, g=None):
    """a wide handle run `runs` times in each form (finalised, then partial), each execution against a fresh unprepared call;
    the replays also against the stats formulas and one key table.  -> (finalised answers, partial answers)"""
    own = g is None
    g = g or ctx.prepare_keyed_wide(q, FAM, key, max_values, vt)
    outs = {}
    try:
        for partial in (False, True):
            plain_fn = ctx.scan_partials_keyed_wide if partial else ctx.scan_agg_keyed_wide
            C = len(ctx.scan_partials_keyed_wide(q, FAM, key, max_values, vt)["group_id"])
            got_all = []
            for i in range(runs):
                got = g.run_partials() if partial else g.run()
                want = plain_fn(q, FAM, key, max_values, vt)
                assert_same(got, want, (what, partial, i))
                got_all.append(got)
                st = got["stats"] if partial else got.stats
                n_keys = want["n_keys"] if partial else want.n_keys
                if i == 0 or n_keys == 0:   # the first execution of a form runs unprepared; V = 0 needs no graph
                    if n_keys == 0 and i > 0:
                        assert (st.kernel_launches, st.d2h_bytes, st.h2d_bytes) == (0, 0, 0), (what, st)
                    continue
                launches, d2h = replay_stats(want, q, C, partial)
                assert st.h2d_bytes == 0 and st.scan_kernel_ms == 0 and st.device_ms > 0, (what, partial, i, st)
                assert (st.kernel_launches, st.d2h_bytes) == (launches, d2h), (what, partial, i, st.kernel_launches, launches, st.d2h_bytes, d2h)
            if partial and runs > 2:   # one key table across the capture's answer and its replays
                assert len({tuple(o["key_table"]) for o in got_all[1:]}) == 1, what
            outs[partial] = got_all
    finally:
        if own:
            g.release()
    return outs[False], outs[True]


# ------------------------------------------------------------------ the query cases of test_gpu_keyed_wide.py
@pytest.mark.parametrize("V", [1000, 4096])
def test_string_values(bydb, gpu_ctx, V):
    """1,000 and 4,096 string values against the oracle; a time cut with a predicate; Top-N both ways with C > 2048; eight
    predicates; the row path's typing"""
    part, ss = string_fixture(V)
    sids = [s.sid for s in ss]
    gid = {s: s % 5 for s in sids}
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        cap = V + 1
        _, q = oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=cap)
        fin, _ = run_handle(bydb, gpu_ctx, q, max_values=cap, what="all rows")
        assert fin[-1].n_keys == V + 1
        _, q = oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=cap, tmin=T0 + 123 * STEP, tmax=T0 + 871 * STEP,
                            preds=[O.Pred(FAM, "z", O.OP_NE, b"z3")])
        run_handle(bydb, gpu_ctx, q, max_values=cap, what="time cut")
        for desc in (True, False):
            _, q = oracle_check(bydb, gpu_ctx, h, part, sids, gid, [("i", COUNT), ("f", MAX)], max_values=cap, top=(17, 0, desc))
            C = len(gpu_ctx.scan_partials_keyed_wide(q, FAM, KT, cap)["group_id"])
            assert C > 2048, C
            fin, _ = run_handle(bydb, gpu_ctx, q, max_values=cap, what=f"top desc={desc}")
            assert fin[-1].group_id.size == 17
        preds = [O.Pred(FAM, "z", O.OP_NE, b"z%d" % j) for j in range(7)] + [O.Pred(FAM, KT, O.OP_GE, b"val-00100")]
        _, q = oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=cap, preds=preds)
        assert len(q.preds) == 8
        run_handle(bydb, gpu_ctx, q, max_values=cap, what="eight predicates")
        q = dataclasses.replace(q, flags=bydb.capi.Q_ROW_PATH_TYPES)
        run_handle(bydb, gpu_ctx, q, max_values=cap, what="row path types")
    finally:
        gpu_ctx.release_part(h)


def test_int64_values_up_to_the_cap(bydb, gpu_ctx):
    """65,536 int64 values, every (group, value) present once"""
    vals = [[(s * 256 + r) * 977 % 65536 - 20000 for r in range(256)] for s in range(256)]
    part = K.build_keyed([int_series(s + 1, vals[s]) for s in range(256)])
    gid = (np.arange(256) % 7).astype(np.int32)
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        q = bydb.Query(parts=[h], series_ids=np.arange(1, 257, dtype=np.uint64), aggs=[("i", SUM), ("i", COUNT), ("f", MAX)],
                       series_group=gid, n_groups=7)
        fin, rows = run_handle(bydb, gpu_ctx, q, max_values=65536, vt=bydb.capi.VT_INT64, what="65,536 values")
        assert fin[-1].n_keys == 65536
        assert list(zip(fin[-1].group_id.tolist(), fin[-1].key)) == [(int(gid[s]), le(v)) for s in range(256) for v in vals[s]]
        assert fin[-1].val_i64[:, 0].tolist() == [v * 3 + s + 1 for s in range(256) for v in vals[s]]
    finally:
        gpu_ctx.release_part(h)


def test_more_than_2_20_present_composite_groups(bydb, gpu_ctx):
    """4,200 series, each its own group, each showing 256 values of a 4,096-value pool: 1,075,200 composite groups"""
    G, pool = 4200, [b"p%04d" % v for v in range(4096)]
    keys = [[pool[(s * 613 + r * 16) % 4096] for r in range(256)] for s in range(G)]
    part = K.build_keyed([Series(s + 1, wide_fields(s + 1, 256), {KT: keys[s]}) for s in range(G)])
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        q = bydb.Query(parts=[h], series_ids=np.arange(1, G + 1, dtype=np.uint64), aggs=[("i", SUM), ("i", COUNT)],
                       series_group=np.arange(G, dtype=np.int32), n_groups=G)
        fin, rows = run_handle(bydb, gpu_ctx, q, max_values=4096, what="2^20 groups")
        assert fin[-1].group_id.size == 256 * G > 1 << 20 and fin[-1].key == [k for ks in keys for k in ks]
        assert len(rows[-1]["group_id"]) == 256 * G
    finally:
        gpu_ctx.release_part(h)


def test_float_mantissas_of_17_digits(bydb, gpu_ctx):
    """decimal float pages whose mantissas span the int64 range (16-17 significant digits), against the oracle"""
    n = 600
    r = np.arange(n)
    f1 = -(r % 50 + 5) / 3.0
    f2 = np.where(r % 3 == 0, 0.30000000000000004, -1.5 - (r % 7))
    f3 = np.where(r % 2 == 0, (r % 40 + 90) / 7.0, -(r % 11 + 2) / 3.0)
    ss = [Series(1, {"i": (I, r * 3 - 100, None), "f": (F, f1, None)}, {KT: [b"a" if x % 4 else b"b" for x in r]}),
          Series(2, {"i": (I, r * 5 + 7, None), "f": (F, f2, None)}, {KT: [b"pos" if x % 3 == 0 else b"neg" for x in r]}),
          Series(3, {"i": (I, r - 300, None), "f": (F, f3, None)}, {KT: [b"big" if x % 2 == 0 else b"a" for x in r]})]
    assert all(s.kind(("f", "f"), 0, n)[0] != "raw" for s in ss)
    part = K.build_keyed(ss)
    aggs = [("f", MIN), ("f", MAX), ("f", SUM), ("f", MEAN), ("i", MIN), ("i", MAX)]
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        for gid in ({1: 0, 2: 0, 3: 0}, {1: 0, 2: 1, 3: 2}):
            _, q = oracle_check(bydb, gpu_ctx, h, part, [1, 2, 3], gid, aggs, max_values=300)
            run_handle(bydb, gpu_ctx, q, max_values=300, what=f"groups {gid}")
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ V = 0, C = 0, C = 1
def test_empty_and_single_answers(bydb, gpu_ctx):
    """no block selected (V = 0: no graph, no keys, zero stats); blocks selected but no row survives (C = 0: a graph that answers
    no rows, the key table all the same); one composite group (C = 1)"""
    ss = [Series(1, wide_fields(1, 300), {KT: [b"k%d" % (x % 3) for x in range(300)], "z": [b"z"] * 300}),
          Series(2, wide_fields(2, 300), {KT: [b"k1"] * 300, "z": [b"y"] * 300})]
    part = K.build_keyed(ss)
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        base = bydb.Query(parts=[h], series_ids=np.array([1, 2], np.uint64), aggs=[("i", SUM), ("f", MAX)],
                          series_group=np.array([0, 1], np.int32), n_groups=2)
        for name, q in (("series the part does not hold", dataclasses.replace(base, series_ids=np.array([7, 8], np.uint64))),
                        ("time range before the part", dataclasses.replace(base, tmin=T0 - 100 * STEP, tmax=T0 - STEP))):
            fin, rows = run_handle(bydb, gpu_ctx, q, max_values=1000, what=name)
            for got in fin:
                assert got.n_keys == 0 and got.key == [] and got.group_id.size == 0, name
            for got in fin[1:] + rows[1:]:
                st = got["stats"] if isinstance(got, dict) else got.stats
                assert st == bydb.capi.Stats(), (name, st)
        q = dataclasses.replace(base, preds=[bydb.Pred(FAM, "z", O.OP_EQ, b"none")])
        fin, rows = run_handle(bydb, gpu_ctx, q, max_values=1000, what="C = 0")
        assert all(g.n_keys == 3 and g.group_id.size == 0 for g in fin) and all(len(r["group_id"]) == 0 for r in rows)
        q = dataclasses.replace(base, series_ids=np.array([2], np.uint64), series_group=np.array([1], np.int32))
        fin, rows = run_handle(bydb, gpu_ctx, q, max_values=1000, what="C = 1")
        assert fin[-1].group_id.tolist() == [1] and fin[-1].key == [b"k1"] and len(rows[-1]["group_id"]) == 1
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ refusals
def refusal(err):
    """(code, text) of a refusal, without the number of the block a device error names: discovery and the scan meet the blocks
    from many warps at once, so which one meets a type mix or goes over the cap first varies between unprepared calls too"""
    return err.code, re.sub(r" \(block #\d+\)$", " (block #)", str(err))


def refuses_alike(bydb, ctx, q, key, max_values, vt, code, sane):
    """the unprepared wide call fails with `code`; the prepared form refuses at prepare with the same code and text, or else on
    every execution in both forms; afterwards the context still answers the plain query `sane`"""
    with pytest.raises(bydb.BydbError) as pe:
        ctx.scan_agg_keyed_wide(q, FAM, key, max_values, vt)
    assert pe.value.code == code, (code, pe.value)
    try:
        g = ctx.prepare_keyed_wide(q, FAM, key, max_values, vt)
    except bydb.BydbError as e:
        assert refusal(e) == refusal(pe.value)
    else:
        try:
            for run in range(RUNS):
                with pytest.raises(bydb.BydbError) as e:
                    g.run_partials() if run % 2 else g.run()
                assert refusal(e.value) == refusal(pe.value), run
        finally:
            g.release()
    assert ctx.scan_agg(sane).group_id.size > 0


def test_refusals(bydb, gpu_ctx):
    """above 65,536 (EINVAL at prepare), above the cap (ENOMEM), an int64 tag as a string key, a block with 257 int64 values, a
    plain string page, a 65-byte value, parts that overlap in time (ENOTSUP): each alike with the unprepared call"""
    E = bydb.capi
    one = np.array([1], np.uint64)
    parts = {}
    try:
        def reg(name, ss, n=1):
            parts[name] = gpu_ctx.register_part(K._next_pid(), K.build_keyed(ss, n).files())
            return parts[name]
        part, ss = string_fixture(1000)
        h = reg("strings", ss)
        q = bydb.Query(parts=[h], series_ids=np.array([s.sid for s in ss], np.uint64), aggs=[("i", SUM)])
        refuses_alike(bydb, gpu_ctx, q, KT, 65537, 0, E.EINVAL, q)
        refuses_alike(bydb, gpu_ctx, q, KT, 1000, 0, E.ENOMEM, q)
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.prepare_keyed_wide(q, FAM, KT, 65537)
        assert e.value.code == E.EINVAL
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.prepare_keyed_wide(q, FAM, KT, 16, 9)
        assert e.value.code == E.EINVAL
        nine = [bydb.Pred(FAM, "z", O.OP_NE, b"q%d" % j) for j in range(9)]
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.prepare_keyed_wide(dataclasses.replace(q, preds=nine), FAM, KT, 2000)
        refuses_alike(bydb, gpu_ctx, dataclasses.replace(q, preds=nine), KT, 2000, 0, e.value.code, q)
        hi = reg("int64", [int_series(1, list(range(300))[:256]), int_series(2, [5] * 40)])
        qi = bydb.Query(parts=[hi], series_ids=np.array([1, 2], np.uint64), aggs=[("i", COUNT)])
        refuses_alike(bydb, gpu_ctx, qi, KT, 1000, E.VT_STR, E.EINVAL, qi)
        h257 = reg("257", [int_series(1, list(range(257)))])
        refuses_alike(bydb, gpu_ctx, bydb.Query(parts=[h257], series_ids=one, aggs=[("i", COUNT)]), KT, 1000, E.VT_INT64, E.ENOTSUP, qi)
        for name, keys in (("plain page", ["s%03d" % i for i in range(257)]), ("65-byte value", ["x" * 65, "y"])):
            hs = reg(name, [Series(1, wide_fields(1, len(keys)), {KT: [k.encode() for k in keys]})])
            refuses_alike(bydb, gpu_ctx, bydb.Query(parts=[hs], series_ids=one, aggs=[("i", SUM)]), KT, 300, 0, E.ENOTSUP, qi)
        a, b = [Series(1, wide_fields(1, 40), {KT: [b"a"] * 40})], [Series(1, wide_fields(1, 40), {KT: [b"b"] * 40})]
        ha, hb = reg("a", a), reg("b", b)
        refuses_alike(bydb, gpu_ctx, bydb.Query(parts=[ha, hb], series_ids=one, aggs=[("i", SUM)]), KT, 300, 0, E.ENOTSUP, qi)
    finally:
        for hp in parts.values():
            gpu_ctx.release_part(hp)


# ------------------------------------------------------------------ parts changing under a handle
def test_parts_change_between_executions(bydb, gpu_ctx):
    """another part registered and released leaves the step standing; the handle's own part released gives the plain call's
    ENOENT on every execution; the part id registered again with a new key value is discovered and captured by a new handle"""
    mk = lambda sid, keys: Series(sid, wide_fields(sid, len(keys)), {KT: keys})   # noqa: E731
    part = K.build_keyed([mk(1, [b"a", b"b"] * 300), mk(2, [b"b", None] * 300)])
    other = K.build_keyed([mk(1, [b"a", b"new"] * 400), mk(3, [b"z"] * 100)])
    pid = K._next_pid()
    usid = np.array([1, 2, 3], np.uint64)
    qf = lambda hh: bydb.Query([hh], usid, [("i", SUM), ("i", COUNT), ("f", MAX)], series_group=np.array([0, 1, 0], np.int32), n_groups=2)  # noqa: E731
    h = gpu_ctx.register_part(pid, part.files())
    g = gpu_ctx.prepare_keyed_wide(qf(h), FAM, KT, 1000)
    try:
        want = gpu_ctx.scan_agg_keyed_wide(qf(h), FAM, KT, 1000)
        assert want.n_keys == 3
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
            gpu_ctx.scan_agg_keyed_wide(qf(h), FAM, KT, 1000)
        for partial in (False, True, False):
            with pytest.raises(bydb.BydbError) as e:
                g.run_partials() if partial else g.run()
            assert e.value.code == pe.value.code == bydb.capi.ENOENT
        h_old, h = h, gpu_ctx.register_part(pid, other.files())
        assert h != h_old
        with pytest.raises(bydb.BydbError) as e:   # a handle names a part object, not its id
            g.run()
        assert e.value.code == bydb.capi.ENOENT
        fin, _ = run_handle(bydb, gpu_ctx, qf(h), max_values=1000, what="new data under the same id")
        assert b"new" in fin[-1].key
    finally:
        g.release()
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ forms and threads
def test_forms_alternating_and_threads(bydb, gpu_ctx):
    """one handle alternating its two forms (each switch drops the step and captures the other); two wide handles and a narrow
    keyed handle run from threads at once, next to unprepared calls"""
    part, ss = string_fixture(1000)
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        sids = np.array([s.sid for s in ss], np.uint64)
        qa = bydb.Query([h], sids, [("i", SUM), ("f", MEAN)], series_group=(np.arange(sids.size) % 3).astype(np.int32), n_groups=3)
        qb = bydb.Query([h], sids[:10], [("i", COUNT), ("f", MIN)], preds=[bydb.Pred(FAM, "z", O.OP_NE, b"z1")], top_n=40)
        qn = bydb.Query([h], sids, [("i", SUM), ("i", COUNT)])
        ga = gpu_ctx.prepare_keyed_wide(qa, FAM, KT, 2000)
        gb = gpu_ctx.prepare_keyed_wide(qb, FAM, KT, 2000)
        gn = gpu_ctx.prepare_keyed(qn, FAM, "z", 64)
        try:
            wa, wb = gpu_ctx.scan_agg_keyed_wide(qa, FAM, KT, 2000), gpu_ctx.scan_agg_keyed_wide(qb, FAM, KT, 2000)
            pa = gpu_ctx.scan_partials_keyed_wide(qa, FAM, KT, 2000)
            wn = gpu_ctx.scan_agg_keyed(qn, FAM, "z", 64)
            for rnd in range(6):
                for partial in ((False, True) if rnd % 2 else (True, False)):
                    if partial:
                        assert_same(ga.run_partials(), pa, ("a partial", rnd))
                    else:
                        assert_same(ga.run(), wa, ("a", rnd))
            errors = []

            def worker(g, want, name, partial=False):
                try:
                    for i in range(8):
                        assert_same(g.run_partials() if partial else g.run(), want, (name, i))
                except Exception as e:   # noqa: BLE001 -- reported by the main thread
                    errors.append(e)
            ths = [threading.Thread(target=worker, args=a) for a in ((ga, wa, "a"), (gb, wb, "b"), (gn, wn, "narrow"))]
            for t in ths:
                t.start()
            for _ in range(4):
                gpu_ctx.scan_agg_keyed_wide(qa, FAM, KT, 2000)
                gpu_ctx.scan_partials_keyed_wide(qb, FAM, KT, 2000)
            for t in ths:
                t.join()
            assert not errors, errors
            run_handle(bydb, gpu_ctx, qb, max_values=2000, what="b after threads", g=gb)
        finally:
            ga.release()
            gb.release()
            gn.release()
    finally:
        gpu_ctx.release_part(h)

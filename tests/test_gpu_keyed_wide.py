"""Group-by on a stored tag in one scan pass (bydb_scan_agg_keyed_wide / bydb_scan_partials_keyed_wide, DESIGN.md 4.6).

The one-pass form must answer what the per-value passes answer, so the first test runs every query of the keyed test modules
through a context whose scan_agg_keyed / scan_partials_keyed also call the wide form on the same arguments and check, call by
call: the same rows in the same order, the same key bytes per row, the same n_keys, equal int64 values and floats within 1e-9;
three wide calls bit-identical; and rows_scanned / blocks_scanned / rows_matched equal to the plain scan_agg of the query (one
pass, not V).  The narrow answer goes back to the wrapped test, whose own checks run unchanged.  The other tests cover what the
per-value passes cannot answer: thousands of key values against the oracle and an independent model, the caps, the per-block
limits, eight predicates, more than 2^20 present composite groups, and the operator above 256 values.
"""
import dataclasses
import functools

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests import test_gpu_keyed_int64 as K64
from tests import test_gpu_keyed_partials as KP
from tests.helpers import STEP, T0, assert_parity, to_gpu_query
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, F, I, Series
from tests.test_gpu_masks import I64_MAX, I64_MIN

gpu = pytest.mark.gpu
FAM, KT = K.FAM, K.KT
AGGS = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("i", MEAN), ("f", SUM), ("f", MIN), ("f", MAX), ("f", MEAN)]


def _same_floats(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(((a.view(np.uint64) == b.view(np.uint64)) | np.isclose(a, b, rtol=1e-9, atol=0.0)).all())


def same_result(n, w, ctx):
    assert w.group_id.tolist() == n.group_id.tolist(), f"{ctx}: groups {w.group_id[:8]} vs {n.group_id[:8]}"
    assert w.key == n.key, f"{ctx}: keys {w.key[:8]} vs {n.key[:8]}"
    assert w.n_keys == n.n_keys, f"{ctx}: n_keys {w.n_keys} vs {n.n_keys}"
    assert w.rows.tolist() == n.rows.tolist(), f"{ctx}: rows"
    assert w.is_float.tolist() == n.is_float.tolist(), f"{ctx}: output typing"
    assert (w.val_i64 == n.val_i64).all(), f"{ctx}: int64 values"
    assert _same_floats(w.val_f64, n.val_f64), f"{ctx}: float values"


def same_rows(n, w, ctx):
    for k in ("group_id", "is_float", "val_i64", "cnt_i64"):
        assert np.asarray(w[k]).tolist() == np.asarray(n[k]).tolist(), f"{ctx}: {k}"
    assert w["key"] == n["key"] and w["n_keys"] == n["n_keys"], f"{ctx}: keys"
    assert _same_floats(w["val_f64"], n["val_f64"]) and _same_floats(w["cnt_f64"], n["cnt_f64"]), f"{ctx}: float partials"


def identical(a, b):
    if isinstance(a, dict):
        return all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in ("group_id", "val_i64", "val_f64", "cnt_i64", "cnt_f64")) \
            and a["key"] == b["key"]
    return a.group_id.tobytes() == b.group_id.tobytes() and a.val_f64.tobytes() == b.val_f64.tobytes() and \
        a.val_i64.tobytes() == b.val_i64.tobytes() and a.key == b.key


class Both:
    """gpu_ctx, with the keyed calls checked against the wide form (see the module docstring)"""

    def __init__(self, bydb, ctx):
        self._bydb, self._ctx, self.calls = bydb, ctx, 0

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def _check(self, narrow_fn, wide_fn, same, q, family, tag, max_values=0, value_type=0):
        args = (q, family, tag, max_values, value_type)
        try:
            narrow = narrow_fn(*args)
        except self._bydb.BydbError:
            # the per-value passes refuse more than 256 values and an 8th predicate; anything else the wide form refuses too
            if (max_values or 64) <= 256 and len(q.preds) < 8:
                with pytest.raises(self._bydb.BydbError):
                    wide_fn(*args)
            raise
        ctx = f"{tag} cap={max_values} preds={len(q.preds)} top={q.top_n}"
        wide = [wide_fn(*args) for _ in range(3)]
        same(narrow, wide[0], ctx)
        assert identical(wide[0], wide[1]) and identical(wide[0], wide[2]), f"{ctx}: repeated wide calls differ"
        st = wide[0]["stats"] if isinstance(wide[0], dict) else wide[0].stats
        try:
            plain = self._ctx.scan_agg(q).stats
        except self._bydb.BydbError:
            plain = None
        if plain is not None:
            assert (st.rows_scanned, st.blocks_scanned, st.rows_matched) == (plain.rows_scanned, plain.blocks_scanned, plain.rows_matched), \
                f"{ctx}: wide stats {(st.rows_scanned, st.blocks_scanned, st.rows_matched)} vs plain " \
                f"{(plain.rows_scanned, plain.blocks_scanned, plain.rows_matched)}"
        self.calls += 1
        return narrow

    def scan_agg_keyed(self, *args):
        return self._check(self._ctx.scan_agg_keyed, self._ctx.scan_agg_keyed_wide, same_result, *args)

    def scan_partials_keyed(self, *args):
        return self._check(self._ctx.scan_partials_keyed, self._ctx.scan_partials_keyed_wide, same_rows, *args)


NARROW_CASES = [
    (K.test_first_row_at_int64_max, {}), (K.test_dictionary_shapes, {}), (K.test_hash_collisions, {}), (K.test_cap_and_limits, {}),
    (K.test_insertion_order, {}), (K.test_composite_table_size_and_top_n, {}), (K.test_lanes_under_the_passes, {}),
    *[(K64.test_int64_key_page_kinds, {"kind": kind}) for kind in K64.INT_KINDS],
    (K64.test_int64_key_values, {}), (K64.test_int64_key_cap_and_refusals, {}), (K64.test_int64_key_insertion_order, {}),
    (KP.test_one_node_against_the_oracle, {"int64": False}), (KP.test_one_node_against_the_oracle, {"int64": True}),
    (KP.test_no_one_and_every_composite_group, {}),
]


@gpu
@pytest.mark.parametrize("case", NARROW_CASES, ids=[f"{fn.__module__.split('.')[-1]}.{fn.__name__}" + "".join(f"-{v}" for v in kw.values())
                                                  for fn, kw in NARROW_CASES])
def test_agrees_with_the_per_value_passes(bydb, gpu_ctx, case):
    fn, kw = case
    both = Both(bydb, gpu_ctx)
    fn(bydb, both, **kw)
    assert both.calls > 0


# ------------------------------------------------------------------ thousands of string values against the oracle
def wide_fields(sid, n):
    r = np.arange(n, dtype=np.int64)
    return {"i": (I, (r * 31 + sid * 7) % 1000 - 300, None), "f": (F, np.round(((r * 53 + sid) % 3000) / 10.0 + 0.1, 1), None)}


@functools.lru_cache(None)
def string_fixture(V, n_series=32, n=1000, window=200):
    """n_series series of n rows (one block each), series s drawing its key from a window of `window` values of a V-value pool
    (so <= 256 per block), the windows spread so that every value occurs; tag z for predicates"""
    pool = [b"val-%05d" % v for v in range(V)]
    step = -(-(V - window) // (n_series - 1))
    out = []
    for j, sid in enumerate(range(1, n_series + 1)):
        keys = [pool[(j * step + (r * 7 + j) % window) % V] if r % 97 != 5 else None for r in range(n)]
        z = [b"z%d" % ((r + j) % 10) for r in range(n)]
        out.append(Series(sid, wide_fields(sid, n), {KT: keys, "z": z}))
    return K.build_keyed(out), out


def oracle_check(bydb, ctx, h, part, sids, gid, aggs, key=KT, max_values=0, vt=0, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=(0, 0, True)):
    groups = np.array([gid[int(s)] for s in sids], np.int32)
    oq = O.Query([part], np.asarray(sids, np.uint64), list(aggs), groups=groups, n_groups=max(gid.values()) + 1, tmin=tmin, tmax=tmax,
                 preds=list(preds), top_n=top[0], top_agg=top[1], top_desc=top[2])
    q = to_gpu_query(bydb, [h], oq)
    got = ctx.scan_agg_keyed_wide(q, FAM, key, max_values, vt)
    want = O.run_query(dataclasses.replace(oq, group_key=(FAM, key)))
    assert_parity(got, want, aggs, f"key={key} preds={len(preds)}")
    assert got.key == want.key
    return got, q


@gpu
@pytest.mark.parametrize("V", [1000, 4096])
def test_string_values_against_the_oracle(bydb, gpu_ctx, V):
    part, ss = string_fixture(V)
    sids = [s.sid for s in ss]
    gid = {s: s % 5 for s in sids}
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        got, q = oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=V + 1)
        assert got.n_keys == V + 1   # the nil cells are the value ""
        plain = gpu_ctx.scan_agg(q).stats
        assert (got.stats.rows_scanned, got.stats.blocks_scanned, got.stats.rows_matched) == \
            (plain.rows_scanned, plain.blocks_scanned, plain.rows_matched)
        # a time range that cuts every block, a predicate, Top-N both ways over ties (COUNT)
        oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=V + 1, tmin=T0 + 123 * STEP, tmax=T0 + 871 * STEP,
                     preds=[O.Pred(FAM, "z", O.OP_NE, b"z3")])
        for desc in (True, False):
            oracle_check(bydb, gpu_ctx, h, part, sids, gid, [("i", COUNT), ("f", MAX)], max_values=V + 1, top=(17, 0, desc))
        # eight predicates: the key takes no predicate slot
        preds = [O.Pred(FAM, "z", O.OP_NE, b"z%d" % j) for j in range(7)] + [O.Pred(FAM, KT, O.OP_GE, b"val-00100")]
        oracle_check(bydb, gpu_ctx, h, part, sids, gid, AGGS, max_values=V + 1, preds=preds)
        # the cap: V + 1 values answer at V + 1, not at V; above 65,536 is refused before anything runs
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, V)
        assert e.value.code == bydb.capi.ENOMEM
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 65537)
        assert e.value.code == bydb.capi.EINVAL
        got2 = gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, V + 1)
        assert identical(got, got2)
        # the partial form: the same composite groups, keys and counts
        rows = gpu_ctx.scan_partials_keyed_wide(q, FAM, KT, 65536)
        assert rows["group_id"].tolist() == got.group_id.tolist() and rows["key"] == got.key
        assert rows["val_i64"][:, 1].tolist() == got.val_i64[:, 1].tolist()
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ decimal float pages with 16-17 significant digits
@gpu
def test_float_mantissas_of_17_digits(bydb, gpu_ctx):
    """Decimal float pages hold shortest round-trip mantissas scaled to the page's smallest exponent, so they span the whole int64
    range: -37/3 is about -1.2e16 at exponent -15, and -1.5 next to 0.30000000000000004 is -1.5e17.  Keys whose values are all
    such negatives (and one whose values are all large positives) keep their MIN / MAX bit for bit, against the oracle and the
    per-value passes, in both answer forms."""
    n = 600
    r = np.arange(n)
    f1 = -(r % 50 + 5) / 3.0                                             # every value negative, 16-17 digits
    f2 = np.where(r % 3 == 0, 0.30000000000000004, -1.5 - (r % 7))        # key "neg": -1.5 .. -7.5 at exponent -17
    f3 = np.where(r % 2 == 0, (r % 40 + 90) / 7.0, -(r % 11 + 2) / 3.0)   # key "big": positives only
    ss = [Series(1, {"i": (I, r * 3 - 100, None), "f": (F, f1, None)}, {KT: [b"a" if x % 4 else b"b" for x in r]}),
          Series(2, {"i": (I, r * 5 + 7, None), "f": (F, f2, None)}, {KT: [b"pos" if x % 3 == 0 else b"neg" for x in r]}),
          Series(3, {"i": (I, r - 300, None), "f": (F, f3, None)}, {KT: [b"big" if x % 2 == 0 else b"a" for x in r]})]
    assert all(s.kind(("f", "f"), 0, n)[0] != "raw" for s in ss), "the fixture must give decimal pages, not raw cells"
    part = K.build_keyed(ss)
    aggs = [("f", MIN), ("f", MAX), ("f", SUM), ("f", MEAN), ("i", MIN), ("i", MAX)]
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        for gid in ({1: 0, 2: 0, 3: 0}, {1: 0, 2: 1, 3: 2}):
            got, q = oracle_check(bydb, gpu_ctx, h, part, [1, 2, 3], gid, aggs, max_values=300)
            same_result(gpu_ctx.scan_agg_keyed(q, FAM, KT, 256), got, f"groups {gid}")
            same_rows(gpu_ctx.scan_partials_keyed(q, FAM, KT, 256), gpu_ctx.scan_partials_keyed_wide(q, FAM, KT, 300), f"partials {gid}")
        # the keys' extremes from the fixture itself
        ext = {}
        for s, f in zip(ss, (f1, f2, f3)):
            for k, x in zip(s.tags[KT], f.tolist()):
                lo, hi = ext.get(k, (np.inf, -np.inf))
                ext[k] = (min(lo, x), max(hi, x))
        got = gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 300)
        seen = {}
        for k, mn, mx in zip(got.key, got.val_f64[:, 0].tolist(), got.val_f64[:, 1].tolist()):
            lo, hi = seen.get(k, (np.inf, -np.inf))
            seen[k] = (min(lo, mn), max(hi, mx))
        assert seen == ext, f"per-key extremes {seen} vs the fixture's {ext}"
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ int64 keys up to 65,536 values, against a numpy fold
def le(v):
    return int(v).to_bytes(8, "little", signed=True)


def int_series(sid, values):
    n = len(values)
    return Series(sid, {"i": (I, np.asarray(values, np.int64) * 3 + sid, None), "f": (F, np.round(np.arange(n) / 4.0 + 0.25, 2), None)},
                  {KT: (np.asarray(values, np.int64), np.zeros(n, bool))})


@gpu
def test_int64_values_up_to_the_cap(bydb, gpu_ctx):
    """256 series x 256 distinct values each = 65,536 values, every (group, value) present once"""
    vals = [[(s * 256 + r) * 977 % 65536 - 20000 for r in range(256)] for s in range(256)]
    ss = [int_series(s + 1, vals[s]) for s in range(256)]
    part = K.build_keyed(ss)
    sids = np.arange(1, 257, dtype=np.uint64)
    gid = (np.arange(256) % 7).astype(np.int32)
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        q = bydb.Query(parts=[h], series_ids=sids, aggs=[("i", SUM), ("i", COUNT), ("f", MAX)], series_group=gid, n_groups=7)
        got = gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 65536, bydb.capi.VT_INT64)
        assert got.n_keys == 65536
        want_comp = [(int(gid[s]), le(v)) for s in range(256) for v in vals[s]]
        assert list(zip(got.group_id.tolist(), got.key)) == want_comp
        assert got.rows.tolist() == [1] * 65536
        assert got.val_i64[:, 0].tolist() == [v * 3 + s + 1 for s in range(256) for v in vals[s]]
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 65535, bydb.capi.VT_INT64)
        assert e.value.code == bydb.capi.ENOMEM
        with pytest.raises(bydb.BydbError) as e:   # an int64 tag named as a string key
            gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 65536, bydb.capi.VT_STR)
        assert e.value.code == bydb.capi.EINVAL
    finally:
        gpu_ctx.release_part(h)


@gpu
def test_per_block_limits(bydb, gpu_ctx):
    """an int64 block with 256 distinct values answers, one with 257 is refused naming the block; a 257-value string block is a
    plain page (refused); a 64-byte string value answers, a 65-byte one is refused"""
    for n, ok in ((256, True), (257, False)):
        part = K.build_keyed([int_series(1, list(range(n))), int_series(2, [5] * 40)])
        h = gpu_ctx.register_part(K._next_pid(), part.files())
        try:
            q = bydb.Query(parts=[h], series_ids=np.array([1, 2], np.uint64), aggs=[("i", COUNT)])
            if ok:
                assert gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 1000, bydb.capi.VT_INT64).rows.tolist() == [1] * 5 + [41] + [1] * 250
            else:
                with pytest.raises(bydb.BydbError) as e:
                    gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 1000, bydb.capi.VT_INT64)
                assert e.value.code == bydb.capi.ENOTSUP and "block" in str(e.value)
        finally:
            gpu_ctx.release_part(h)
    cases = ((["s%03d" % i for i in range(257)], False), (["x" * 64, "y"], True), (["x" * 65, "y"], False))
    for keys, ok in cases:
        ss = [Series(1, wide_fields(1, len(keys)), {KT: [k.encode() for k in keys]})]
        part = K.build_keyed(ss)
        h = gpu_ctx.register_part(K._next_pid(), part.files())
        try:
            q = bydb.Query(parts=[h], series_ids=np.array([1], np.uint64), aggs=[("i", SUM)])
            if ok:
                got, _ = oracle_check(bydb, gpu_ctx, h, part, [1], {1: 0}, [("i", SUM)], max_values=300)
                assert len(got.key[0]) == 64
            else:
                with pytest.raises(bydb.BydbError) as e:
                    gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 300)
                assert e.value.code == bydb.capi.ENOTSUP
        finally:
            gpu_ctx.release_part(h)


@gpu
def test_more_than_2_20_present_composite_groups(bydb, gpu_ctx):
    """4,200 series, each its own group, each showing 256 distinct values of a 4,096-value pool: 1,075,200 composite groups"""
    G, pool = 4200, [b"p%04d" % v for v in range(4096)]
    keys = [[pool[(s * 613 + r * 16) % 4096] for r in range(256)] for s in range(G)]
    ss = [Series(s + 1, wide_fields(s + 1, 256), {KT: keys[s]}) for s in range(G)]
    part = K.build_keyed(ss)
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        q = bydb.Query(parts=[h], series_ids=np.arange(1, G + 1, dtype=np.uint64), aggs=[("i", SUM), ("i", COUNT)],
                       series_group=np.arange(G, dtype=np.int32), n_groups=G)
        got = gpu_ctx.scan_agg_keyed_wide(q, FAM, KT, 4096)
        assert got.n_keys == 4096 and got.group_id.size == 256 * G > 1 << 20
        assert got.group_id.tolist() == [s for s in range(G) for _ in range(256)]
        assert got.key == [k for ks in keys for k in ks]
        assert (got.val_i64[:, 1] == 1).all()
        assert got.val_i64[:, 0].tolist() == [int(x) for s in range(G) for x in wide_fields(s + 1, 256)["i"][1]]
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ the operator above 256 values
@gpu
def test_operator_above_256_values(bydb, gpu_ctx):
    so = bydb.scan_operator
    part, ss = string_fixture(999)   # 1,000 values with the nil cells' ""
    sids = [s.sid for s in ss]
    h = gpu_ctx.register_part(K._next_pid(), part.files())
    try:
        cols = [so.ColumnDef(KT, so.ColumnRole.RoleTag, so.ColumnType.ColumnTypeString, FAM),
                so.ColumnDef("i", so.ColumnRole.RoleField, so.ColumnType.ColumnTypeInt64),
                so.ColumnDef("f", so.ColumnRole.RoleField, so.ColumnType.ColumnTypeFloat64)]
        specs = [so.AggSpec("a0", so.AggSum, 1), so.AggSpec("a1", so.AggCount, 1), so.AggSpec("a2", so.AggMax, 2)]
        scan = so.ScanSpec(parts=[h], series_ids=sids, series_tags={}, max_key_values=1000)
        op = so.GPUScanAgg(gpu_ctx, so.BatchSchema(cols), [0], specs, scan, batch_size=4096)
        op.Init()
        rows = []
        while (b := op.NextBatch()) is not None:
            rows += list(zip(*b.Columns))
        oq = O.Query([part], np.asarray(sids, np.uint64), [("i", SUM), ("i", COUNT), ("f", MAX)], groups=np.zeros(len(sids), np.int32),
                     n_groups=1, group_key=(FAM, KT))
        want = O.run_query(oq)
        assert len(rows) == len(want.key) > 256
        assert [r[0] for r in rows] == [k.decode() for k in want.key]
        assert [(int(r[1]), int(r[2])) for r in rows] == [(int(a), int(b)) for a, b in want.val_i64[:, :2].tolist()]
        assert [float(r[3]) for r in rows] == want.val_f64[:, 2].tolist()
    finally:
        gpu_ctx.release_part(h)

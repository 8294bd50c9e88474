"""Group-by on a tuple of stored tags in one scan pass (bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide, DESIGN.md 4.6).

The tuple form is checked two ways:
  - against the oracle-pinned one-key wide call on a twin tag: every row carries, next to its tags, a string tag whose cell is an
    injective encoding of the row's key tuple with nil taken as the component rule does ("" for a string, 0 for an int64, also in
    blocks without the column).  Grouping by the tuple must then give what bydb_scan_agg_keyed_wide gives on the twin: the same
    rows in the same order, series groups, values bit for bit (the records match one to one, so the fold trees are the same),
    n_tuples == n_keys and the same rows_scanned / rows_matched / blocks_scanned;
  - against `tuple_model`, test_gpu_keyed.key_model over a tuple of the cells (computeKey's component rule), for 2, 3 and 4 tags
    of mixed types: composite groups, rows, int64 values and min / max exact, float sums within the wide form's bound; n_tuples
    and each tag's table against the distinct tuples / values of the selected blocks.
Then the boundaries (256 / 257 tuples in a block, the cap, 65,536 tuples, a tag with 65,536 values), every refusal, call-to-call
identity and the header's d2h_bytes / kernel_launches formulas.
"""
import ctypes
import importlib
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, F, I, Series
from tests.test_gpu_masks import I64_MAX, I64_MIN
from tests.helpers import STEP, T0

gpu = pytest.mark.gpu
FAM = K.FAM
AGGS = K.AGGS
STR, INT = 1, 2          # VT_STR, VT_INT64 of the C ABI
ENOMEM, EINVAL, ENOTSUP = -12, -22, -95


def le(v):
    return struct.pack("<q", v)


def int_tag(cells):
    return (np.array([0 if c is None else c for c in cells], np.int64), np.array([c is None for c in cells]))


def comp(cell, vt):
    """one key component (groupby.go:226-254): a string nil is "", an int64 nil is 0 as 8 little-endian bytes"""
    if vt == INT:
        return le(0 if cell is None else cell)
    return b"" if cell is None else cell


def twin(*cols):
    """an injective encoding of the tuple: each component's length (4 bytes) then its bytes, as computeKey concatenates them"""
    return [b"".join(struct.pack("<I", len(c)) + c for c in t) for t in zip(*cols)]


def series(sid, n, tags, row0=0):
    return Series(sid, K.std_fields(sid, n), tags, row0=row0)


# ------------------------------------------------------------------ the pair (a: string, b: int64) and its twin c
def pair_parts():
    """part 1: 6 series, a from 5 strings with nils, b from 7 int64 values with nils, one series of two blocks; part 2 (later in
    time, no column b: its rows key to b = 0) over three of the series"""
    p1, p2 = [], []
    for j, sid in enumerate([3, 5, 8, 9, 12, 20]):
        n = 9000 if sid == 8 else 300 + 37 * j
        r = np.arange(n)
        a = [None if (x + j) % 11 == 0 else b"a%d" % ((x // 3 + j) % 5) for x in r.tolist()]
        b = [None if (x + 2 * j) % 13 == 0 else [0, -1, 7, I64_MIN, I64_MAX, 3, 42][(x * 5 + j) % 7] for x in r.tolist()]
        z = [b"z%d" % ((x + j) % 4) for x in r.tolist()]
        c = twin([comp(x, STR) for x in a], [comp(x, INT) for x in b])
        p1.append(series(sid, n, {"a": a, "b": int_tag(b), "c": c, "z": z, "k0": [b"const"] * n}))
    for j, sid in enumerate([3, 9, 30]):
        n = 200 + 11 * j
        a = [None if x % 7 == 3 else b"a%d" % ((x + j) % 6) for x in range(n)]
        c = twin([comp(x, STR) for x in a], [le(0)] * n)
        p2.append(series(sid, n, {"a": a, "c": c, "z": [b"z%d" % (x % 4) for x in range(n)], "k0": [b"const"] * n}, row0=20000))
    return p1, p2


class Parts:
    def __init__(self, bydb, ctx, parts):
        self.bydb, self.ctx, self.parts = bydb, ctx, parts
        self.series = [s for _, ss in parts for s in ss]
        self.usid = np.array(sorted({s.sid for s in self.series}), np.uint64)

    def __enter__(self):
        pid = K._next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, (p, _) in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def q(self, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=(0, 0, True), sids=None, groups=None, flags=0, handles=None):
        sids = self.usid if sids is None else np.array(sorted(sids), np.uint64)
        gid = groups or {int(s): i for i, s in enumerate(sids.tolist())}
        g = np.array([gid[int(s)] for s in sids.tolist()], np.int32)
        return self.bydb.Query(parts=handles or self.handles, series_ids=sids, aggs=list(aggs), series_group=g, n_groups=max(gid.values()) + 1,
                               tmin=tmin, tmax=tmax, preds=[self.bydb.Pred(p.family, p.tag, p.op, p.value) for p in preds],
                               top_n=top[0], top_agg=top[1], top_desc=top[2], flags=flags)


def bits(x):
    return np.ascontiguousarray(x).tobytes()


def same_answer(t, w, keys_to_twin, ctx):
    """the tuple answer t equals the one-key answer w on the twin, bit for bit"""
    assert t.group_id.tolist() == w.group_id.tolist(), f"{ctx}: groups"
    assert [keys_to_twin(k) for k in t.key] == w.key, f"{ctx}: keys {t.key[:4]} vs {w.key[:4]}"
    assert t.rows.tolist() == w.rows.tolist(), f"{ctx}: rows"
    assert t.is_float.tolist() == w.is_float.tolist(), f"{ctx}: typing"
    assert bits(t.val_i64) == bits(w.val_i64) and bits(t.val_f64) == bits(w.val_f64), f"{ctx}: values"
    assert (t.stats.rows_scanned, t.stats.rows_matched, t.stats.blocks_scanned) == \
        (w.stats.rows_scanned, w.stats.rows_matched, w.stats.blocks_scanned), f"{ctx}: counters"


def same_partials(t, w, keys_to_twin, ctx):
    for k in ("group_id", "is_float", "val_i64", "cnt_i64", "val_f64", "cnt_f64"):
        assert bits(np.asarray(t[k])) == bits(np.asarray(w[k])), f"{ctx}: {k}"
    assert [keys_to_twin(k) for k in t["key"]] == w["key"], f"{ctx}: keys"
    assert t["n_tuples"] == w["n_keys"], f"{ctx}: n_tuples"


def identical(a, b):
    return bits(a.group_id) == bits(b.group_id) and bits(a.val_i64) == bits(b.val_i64) and bits(a.val_f64) == bits(b.val_f64) and \
        a.key == b.key and a.key_tables == b.key_tables and a.n_tuples == b.n_tuples


def check_stats(t, w, n_tags, ctx):
    """the header's formulas: the tuple call's discovery read-back and launches in place of the one-key call's"""
    st, sw = t.stats, w.stats
    vt = [len(tb) for tb in t.key_tables]
    disc_t = 32 * (n_tags + 1) + sum(v * (8 if ty == INT else 68) for v, ty in zip(vt, t.key_types)) + 8 * t.n_tuples
    disc_w = 32 + w.n_keys * 68
    assert st.d2h_bytes - disc_t == sw.d2h_bytes - disc_w, f"{ctx}: d2h {st.d2h_bytes} vs {sw.d2h_bytes}"
    assert st.kernel_launches - sw.kernel_launches == n_tags * 2, f"{ctx}: launches {st.kernel_launches} vs {sw.kernel_launches}"


def pair_call(ctx, q, types, tags=("a", "b"), max_values=0, partial=False):
    keys = [(FAM, tg, ty) for tg, ty in zip(tags, types)]
    r = (ctx.scan_partials_keys_wide if partial else ctx.scan_agg_keys_wide)(q, keys, max_values)
    if not partial:
        r.key_types = list(types)
    return r


PAIR_QUERIES = [
    dict(),
    dict(tmin=T0 + 100 * STEP, tmax=T0 + 8500 * STEP),
    dict(preds=[O.Pred(FAM, "z", O.OP_NE, b"z1")]),
    dict(preds=[O.Pred(FAM, "a", O.OP_GE, b"a2"), O.Pred(FAM, "z", O.OP_LE, b"z2")], tmin=T0 + 50 * STEP),
    dict(top=(7, 1, True)),
    dict(top=(9, 2, False)),
    dict(top=(5, 3, True), groups={3: 0, 5: 1, 8: 0, 9: 1, 12: 0, 20: 1, 30: 1}),
    dict(groups={3: 0, 5: 0, 8: 0, 9: 0, 12: 0, 20: 0, 30: 0}, flags=2),
    dict(sids=[5, 9, 30], aggs=[("i", MEAN), ("f", MEAN), ("f", COUNT)], flags=2),
]


@gpu
@pytest.mark.parametrize("i", range(len(PAIR_QUERIES)))
def test_pair_equals_the_one_key_twin(bydb, gpu_ctx, i):
    p1, p2 = pair_parts()
    parts = [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]
    kw = PAIR_QUERIES[i]
    ctx = f"pair {kw}"
    to_twin = lambda k: twin([k[0]], [k[1]])[0]   # noqa: E731
    with Parts(bydb, gpu_ctx, parts) as P:
        for order in (None, [1, 0]):
            q = P.q(**kw, handles=None if order is None else [P.handles[j] for j in order])
            w = gpu_ctx.scan_agg_keyed_wide(q, FAM, "c", 4096)
            t = pair_call(gpu_ctx, q, (STR, INT), max_values=4096)
            same_answer(t, w, to_twin, ctx)
            assert t.n_tuples == w.n_keys, f"{ctx}: n_tuples {t.n_tuples} vs n_keys {w.n_keys}"
            assert identical(t, pair_call(gpu_ctx, q, (STR, INT), max_values=4096)), f"{ctx}: repeated calls differ"
            check_stats(t, w, 2, ctx)
            wp = gpu_ctx.scan_partials_keyed_wide(q, FAM, "c", 4096)
            tp = pair_call(gpu_ctx, q, (STR, INT), max_values=4096, partial=True)
            same_partials(tp, wp, to_twin, ctx)
            assert tp["stats"].kernel_launches - wp["stats"].kernel_launches == 2 * 2


@gpu
def test_constant_second_tag(bydb, gpu_ctx):
    """(a, a tag with one value everywhere) answers what the one-key call on a answers, bit for bit"""
    p1, p2 = pair_parts()
    parts = [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]
    with Parts(bydb, gpu_ctx, parts) as P:
        for kw in PAIR_QUERIES:
            q = P.q(**kw)
            w = gpu_ctx.scan_agg_keyed_wide(q, FAM, "a", 4096)
            t = pair_call(gpu_ctx, q, (STR, STR), tags=("a", "k0"), max_values=4096)
            same_answer(t, w, lambda k: k[0], f"constant {kw}")
            assert all(k[1] == b"const" for k in t.key) and t.key_tables[1] == [b"const"]
            assert t.n_tuples == w.n_keys and len(t.key_tables[0]) == w.n_keys


# ------------------------------------------------------------------ the model: 2, 3 and 4 tags of mixed types
def model_parts():
    rng = np.random.default_rng(7)
    p1 = []
    for j, sid in enumerate([2, 4, 6, 7, 11]):
        n = 8193 + 5 if sid == 6 else 400 + 50 * j
        s = rng.integers(0, 1 << 30, size=(4, n))
        a = [None if v % 9 == 0 else b"s%d" % (v % 4) for v in s[0].tolist()]
        b = [None if v % 10 == 0 else (v % 3) - 1 for v in s[1].tolist()]
        e = [None if v % 8 == 0 else b"e%d" % (v % 3) for v in s[2].tolist()]
        d = [None if v % 12 == 0 else [5, I64_MIN, 0][v % 3] for v in s[3].tolist()]
        p1.append(series(sid, n, {"a": a, "b": int_tag(b), "e": e, "d": int_tag(d), "z": [b"z%d" % (x % 3) for x in range(n)]}))
    p2 = []
    for sid in (4, 7, 13):   # later in time, without b and d
        n = 150
        a = [b"s%d" % (x % 5) for x in range(n)]
        e = [None if x % 4 == 0 else b"e%d" % (x % 2) for x in range(n)]
        p2.append(series(sid, n, {"a": a, "e": e, "z": [b"z%d" % (x % 3) for x in range(n)]}, row0=30000))
    return p1, p2


def tuple_cells(s, tags, types):
    cols = []
    for tg, ty in zip(tags, types):
        cell = s.tags.get(tg)
        if cell is None:
            cols.append([comp(None, ty)] * s.n)
        elif isinstance(cell, tuple):
            cols.append([comp(None if nl else int(v), INT) for v, nl in zip(cell[0].tolist(), cell[1].tolist())])
        else:
            cols.append([comp(c, STR) for c in cell])
    return list(zip(*cols))


def tuple_model(P, tags, types, q_sids, gid, aggs, preds, tmin, tmax, top):
    for s in P.series:
        s.tags["__tuple"] = tuple_cells(s, tags, types)
    try:
        return K.key_model(P.series, gid, q_sids, aggs, preds, tmin, tmax, "__tuple", top)
    finally:
        for s in P.series:
            del s.tags["__tuple"]


MODEL_KEYS = [(("a", "b"), (STR, INT)), (("b", "d"), (INT, INT)), (("a", "b", "e"), (STR, INT, STR)),
              (("d", "e", "b", "a"), (INT, STR, INT, STR)), (("e", "a", "d"), (STR, STR, INT))]


@gpu
@pytest.mark.parametrize("keys", MODEL_KEYS, ids=["-".join(k[0]) for k in MODEL_KEYS])
def test_tuples_against_the_model(bydb, gpu_ctx, keys):
    tags, types = keys
    p1, p2 = model_parts()
    parts = [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]
    with Parts(bydb, gpu_ctx, parts) as P:
        for kw in (dict(), dict(preds=[O.Pred(FAM, "z", O.OP_EQ, b"z1")], tmin=T0 + 30 * STEP, tmax=T0 + 30100 * STEP),
                   dict(top=(6, 0, False)), dict(groups={2: 0, 4: 1, 6: 0, 7: 1, 11: 0, 13: 1})):
            ctx = f"{tags} {kw}"
            q = P.q(**kw)
            got = pair_call(gpu_ctx, q, types, tags=tags, max_values=4096)
            gid = kw.get("groups") or {int(s): i for i, s in enumerate(P.usid.tolist())}
            tmin, tmax = kw.get("tmin", I64_MIN), kw.get("tmax", I64_MAX)
            preds = kw.get("preds", [])
            exp = tuple_model(P, tags, types, P.usid, gid, AGGS, preds, tmin, tmax, kw.get("top") or None)
            assert list(zip(got.group_id.tolist(), got.key)) == [e[0] for e in exp], f"{ctx}: composite groups"
            assert got.rows.tolist() == [e[1] for e in exp], f"{ctx}: rows"
            for i, (ck, _, vals) in enumerate(exp):
                for a, ((f, fn), (m, x)) in enumerate(zip(AGGS, vals)):
                    where = f"{ctx}: group {ck} agg {a}"
                    if not got.is_float[a]:
                        assert int(got.val_i64[i, a]) == m, where
                    elif fn in (MIN, MAX):
                        assert got.val_f64[i:i + 1, a].view(np.uint64)[0] == np.array([m]).view(np.uint64)[0], where
                    else:
                        tol = 1e-9 * float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1) + 1e-9 * abs(m)
                        assert abs(float(got.val_f64[i, a]) - m) <= tol, where
            blocks = K.selected_blocks(P.series, P.usid, tmin, tmax)
            tuples = {c for s, lo, hi in blocks for c in tuple_cells(s, tags, types)[lo:hi]}
            assert got.n_tuples == len(tuples), f"{ctx}: n_tuples {got.n_tuples} vs {len(tuples)}"
            for t in range(len(tags)):
                assert sorted(got.key_tables[t]) == sorted({c[t] for c in tuples}), f"{ctx}: table of {tags[t]}"


# ------------------------------------------------------------------ boundaries
def grid_series(sid, cols, row0=0):
    n = len(next(iter(cols.values())))
    return series(sid, n, cols, row0=row0)


@gpu
def test_tuples_per_block(bydb, gpu_ctx):
    """exactly 256 tuples in one block (16 x 16 values) is answered; 257 (a third tag adds one) is refused, naming the block"""
    xs = [b"x%02d" % (i // 16) for i in range(256)]
    ys = [b"y%02d" % (i % 16) for i in range(256)]
    ok = [grid_series(1, {"x": xs, "y": ys, "w": [b"w0"] * 256})]
    bad = [grid_series(1, {"x": xs + [b"x00"], "y": ys + [b"y00"], "w": [b"w0"] * 256 + [b"w1"]})]
    with Parts(bydb, gpu_ctx, [(K.build_keyed(ok), ok)]) as P:
        t = pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, STR, STR), tags=("x", "y", "w"), max_values=1024)
        assert t.n_tuples == 256 and t.rows.tolist() == [1] * 256
    with Parts(bydb, gpu_ctx, [(K.build_keyed(bad), bad)]) as P:
        with pytest.raises(bydb.BydbError) as e:
            pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, STR, STR), tags=("x", "y", "w"), max_values=1024)
        assert e.value.code == ENOTSUP and "256 distinct key tuples" in e.value.msg and "block #0" in e.value.msg, e.value
        assert len(pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, STR), tags=("x", "y"), max_values=1024).key) == 256


@gpu
def test_tuple_cap(bydb, gpu_ctx):
    """10 x 10 tuples over two series: max_values = 100 is answered, 99 is ENOMEM while each tag has 10 values"""
    ss = [grid_series(s, {"x": [b"x%d" % (s * 5 + i // 10) for i in range(50)], "y": int_tag([i % 10 for i in range(50)])})
          for s in (1, 2)]
    with Parts(bydb, gpu_ctx, [(K.build_keyed(ss), ss)]) as P:
        t = pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, INT), tags=("x", "y"), max_values=100)
        assert t.n_tuples == 100 and [len(tb) for tb in t.key_tables] == [10, 10]
        with pytest.raises(bydb.BydbError) as e:
            pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, INT), tags=("x", "y"), max_values=99)
        assert e.value.code == ENOMEM, e.value


@gpu
def test_65536_tuples_and_a_tag_of_65536_values(bydb, gpu_ctx):
    """256 series of 256 rows: a = the series (256 values), b = the row (256 int64 values), so 65,536 tuples, 256 per block; and
    v = a value per row (65,536 values) with a constant second tag.  Both against the one-key call on a twin / on v."""
    ss = []
    for s in range(256):
        a = [b"a%03d" % s] * 256
        b = list(range(256))
        ss.append(grid_series(s + 1, {"a": a, "b": int_tag(b), "c": twin(a, [le(x) for x in b]),
                                      "v": [b"v%05d" % (s * 256 + r) for r in range(256)], "k": [b""] * 256}))
    with Parts(bydb, gpu_ctx, [(K.build_keyed(ss), ss)]) as P:
        q = P.q(aggs=[("i", SUM), ("f", MAX), ("f", MEAN)], groups={s + 1: s % 3 for s in range(256)})
        w = gpu_ctx.scan_agg_keyed_wide(q, FAM, "c", 65536)
        t = pair_call(gpu_ctx, q, (STR, INT), max_values=65536)
        same_answer(t, w, lambda k: twin([k[0]], [k[1]])[0], "65,536 tuples")
        assert t.n_tuples == 65536 == len(t.key) and [len(tb) for tb in t.key_tables] == [256, 256]
        with pytest.raises(bydb.BydbError) as e:
            pair_call(gpu_ctx, q, (STR, INT), max_values=65535)
        assert e.value.code == ENOMEM
        w = gpu_ctx.scan_agg_keyed_wide(q, FAM, "v", 65536)
        t = pair_call(gpu_ctx, q, (STR, STR), tags=("v", "k"), max_values=65536)
        same_answer(t, w, lambda k: k[0], "a tag of 65,536 values")
        assert len(t.key_tables[0]) == 65536 and t.key_tables[1] == [b""]


@gpu
def test_refusals(bydb, gpu_ctx):
    p1, p2 = pair_parts()
    parts = [(K.build_keyed(p1), p1), (K.build_keyed(p2, 2), p2)]
    long = [grid_series(1, {"a": [b"x" * 65, b"y"] * 10, "b": int_tag(list(range(20)))})]
    plain = [grid_series(1, {"a": [b"p%03d" % i for i in range(300)], "b": int_tag([0] * 300)})]
    wide_int = [grid_series(1, {"a": [b"q"] * 300, "b": int_tag(list(range(300)))})]
    overlap = [grid_series(3, {"a": [b"o"] * 10, "b": int_tag([1] * 10), "c": [b"c"] * 10, "z": [b"z"] * 10, "k0": [b"const"] * 10})]
    E = bydb.BydbError

    def code(fn):
        with pytest.raises(E) as e:
            fn()
        return e.value.code

    with Parts(bydb, gpu_ctx, parts) as P:
        q = P.q()
        ok = [(FAM, "a", STR), (FAM, "b", INT)]
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, ok[:1])) == EINVAL
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, ok + [(FAM, "c", STR), (FAM, "z", STR), (FAM, "k0", STR)])) == EINVAL
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, ok + [(FAM, "a", STR)])) == EINVAL
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, ok, 65537)) == EINVAL
        assert code(lambda: gpu_ctx.scan_partials_keys_wide(q, [(FAM, "a", STR), (FAM, "b", STR)], 4096)) == EINVAL   # b is int64
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, [(FAM, "a", INT), (FAM, "b", INT)], 4096)) == EINVAL       # a is a string
        assert code(lambda: gpu_ctx.scan_agg_keys_wide(q, ok, 10)) == ENOMEM
        # a key's own max_values: the binding passes 0, so go through the structures
        capi = importlib.import_module(bydb.__name__ + ".capi")
        keep = []
        gks = capi._group_keys(ok, 4096, keep)
        gks.keys[1].max_values = 8
        cq = capi._mk_query(q, keep)
        r = capi._KeysResult()
        assert capi.load_library().bydb_scan_agg_keys_wide(gpu_ctx._h, ctypes.byref(cq), ctypes.byref(gks), ctypes.byref(r)) == EINVAL
        eight = [O.Pred(FAM, "z", O.OP_NE, b"zz%d" % i) for i in range(8)]
        got = pair_call(gpu_ctx, P.q(preds=eight), (STR, INT), max_values=4096)
        assert got.stats.rows_matched == gpu_ctx.scan_agg(P.q(preds=eight)).stats.rows_matched
    for ss, want in ((long, ENOTSUP), (plain, ENOTSUP), (wide_int, ENOTSUP)):
        with Parts(bydb, gpu_ctx, [(K.build_keyed(ss), ss)]) as P:
            assert code(lambda: pair_call(gpu_ctx, P.q(aggs=[("i", COUNT)]), (STR, INT), max_values=4096)) == want
    with Parts(bydb, gpu_ctx, [parts[0], (K.build_keyed(overlap, 3), overlap)]) as P:
        assert code(lambda: pair_call(gpu_ctx, P.q(), (STR, INT), max_values=4096)) == ENOTSUP
    # the context still answers
    with Parts(bydb, gpu_ctx, parts) as P:
        assert pair_call(gpu_ctx, P.q(), (STR, INT), max_values=4096).n_tuples > 0

"""The group-by on a tuple of 2..4 stored tags (bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide and the collective
bydb_scan_reduce_keys_wide / _partials, DESIGN.md 4.6 and 5) against the oracle grouped by the same tuple, at the boundaries of
the tuple machinery in csrc/scan_kernels.cu:
  1. code packing: a tuple is id_0 | id_1 << 16 | id_2 << 32 | id_3 << 48 in the int64-key table, where 0 marks an empty slot and
     the code 0 rides on the table's zero flag.  Four tags of 65,536 values each, every row holding one value in all four: every
     16-bit field of the code takes all its values (bit 63 included), and with four string tags the tuple of the values numbered
     0 has the code 0 without any int64 tag; the order (int64, string, string, int64) puts a 65,536-value component in bits
     48-63.  max_values 65,536 answers, 65,535 is BYDB_ENOMEM;
  2. the component rules: ("ab", "c") vs ("a", "bc") and ("", "x") vs ("x", "") in blocks of their own and mixed in one block;
     nil vs "" and nil vs 0 vs a block without the column in each of the four positions; INT64_MIN, INT64_MAX, -1 and 0; a block
     without any key column; a predicate on a key tag (rows drop, n_tuples still counts the selected blocks' tuples);
  3. tag order: (a, b, c) and its rotations give the same composites in the same order, components permuted, values bit for bit;
  4. tuple_block_keys: 256 tuples from the first tag alone, 16 x 16 in the last two of four tags, 257 refused naming the block, an
     8,193-row block whose tuple changes at rows 8191 and 8192, one 16 x 16 grid in three row orders (the block-local numbering
     differs block to block), and a probe chain of 62 pairs in the 512-slot pair table: a string tag's block-local index is its
     dictionary index, i.e. first-seen order in the block, so the pairs (i, j) a block shows, and with them their pair_home, are
     chosen from the host;
  5. key_tuples_wide_kernel's block walk over 33 and 64 time-disjoint parts in shuffled order; 65 parts and parts that overlap in
     time refused;
  6. merged series groups, a time cut inside blocks, Top-N both ways over COUNT ties and BYDB_Q_ROW_PATH_TYPES;
  7. the collective's root (tuple_union_code recodes each rank's tuples through the tags' union ids): the four-tag fixture split
     over three ranks, union ids up to 65,535 in the top component, against the oracle over all ranks' parts; a tag union at
     max_values answers, one more is refused before any code is packed, and a plain collective answers after it.

Every answer: composite groups and their order, key tuples, rows, int64 values and MIN / MAX / COUNT exactly; float sums within
the wide form's bound, 1e-9 x sum |x| of the composite + 1e-9 x |reference|, which is 2e-9 x |reference| here because every float
field is positive; the partial form against the oracle's rows (test_gpu_keyed_partials.oracle_rows); n_tuples and each tag's
table against the distinct tuples / values of the selected blocks; two calls of each form bit-identical (the order inside a tag's
table is not part of the contract: the concurrent inserts of a large table may place its values differently from call to call).
"""
import dataclasses
import functools

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0, to_gpu_query
from tests.test_gpu_fallback import BLOCK, COUNT, MAX, MIN, SUM, Series
from tests.test_gpu_keyed_partials import check_rows, oracle_rows
from tests.test_gpu_keyed_reduce import R, Case, Ranks, plain_ok, quiet  # noqa: F401 -- quiet is a fixture
from tests.test_gpu_keys_wide import EINVAL, ENOMEM, ENOTSUP, INT, STR, comp, int_tag, le, tuple_cells
from tests.test_gpu_keys_wide_reduce import tuple_slot
from tests.test_gpu_masks import I64_MAX, I64_MIN, str_tag_class

gpu = pytest.mark.gpu
FAM = K.FAM
AGGS = K.AGGS
_pid = [9_100_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def ser(sid, n, tags, row0=0):
    return Series(sid, K.std_fields(sid, n), tags, row0=row0)


def gkeys(keys):
    return [(FAM, t, vt) for t, vt in keys]


# ------------------------------------------------------------------ the checks
def against_oracle(got, want, aggs, flags, ctx):
    assert list(zip(got.group_id.tolist(), got.key)) == list(zip(want.group_id.tolist(), want.key)), \
        f"{ctx}: composites {list(zip(got.group_id.tolist(), got.key))[:4]} vs oracle {list(zip(want.group_id.tolist(), want.key))[:4]}"
    assert got.rows.tolist() == want.rows.tolist(), f"{ctx}: rows"
    for a, (f, fn) in enumerate(aggs):
        gf, wf = bool(got.is_float[a]), bool(want.is_float[a])
        g = got.val_f64[:, a] if gf else got.val_i64[:, a]
        w = want.val_f64[:, a] if wf else want.val_i64[:, a]
        where = f"{ctx}: agg {a} ({f},{fn})"
        if gf != wf:   # BYDB_Q_ROW_PATH_TYPES: COUNT over a float field is typed like the field
            assert flags and fn == COUNT and gf, f"{where}: typing"
            assert g.tolist() == w.astype(np.float64).tolist(), where
        elif not gf or fn in (MIN, MAX, COUNT):
            assert g.view(np.uint64 if gf else np.int64).tolist() == w.view(np.uint64 if gf else np.int64).tolist(), where
        else:
            bad = np.nonzero(np.abs(g - w) > 2e-9 * np.abs(w))[0]
            assert bad.size == 0, f"{where}: row {bad[:1]}: {g[bad[:1]]} vs oracle {w[bad[:1]]}"


def same_call(a, b):
    return a.group_id.tobytes() == b.group_id.tobytes() and a.rows.tobytes() == b.rows.tobytes() and a.key == b.key and \
        a.val_i64.tobytes() == b.val_i64.tobytes() and a.val_f64.tobytes() == b.val_f64.tobytes() and a.n_tuples == b.n_tuples and \
        [set(t) for t in a.key_tables] == [set(t) for t in b.key_tables]


def discovery(series, keys, sids, tmin, tmax):
    """the distinct tuples of the selected blocks (before the time trim and the predicates), by the component rule"""
    tags, types = zip(*keys)
    return {c for s, lo, hi in K.selected_blocks(series, sids, tmin, tmax) for c in tuple_cells(s, tags, types)[lo:hi]}


class Tup:
    """Parts registered once; each query through both tuple calls (twice each) against the oracle grouped by the same tuple"""

    def __init__(self, bydb, ctx, parts_series, gid):
        self.bydb, self.ctx, self.gid = bydb, ctx, gid
        self.parts = [p for p, _ in parts_series]
        self.series = [s for _, ss in parts_series for s in ss]

    def __enter__(self):
        pid = _next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, p in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def oquery(self, keys, sids, aggs, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, order=None, flags=0):
        sids = np.array(sorted(int(s) for s in sids), np.uint64)
        tn, ta, td = top or (0, 0, True)
        order = list(range(len(self.parts))) if order is None else order
        oq = O.Query([self.parts[i] for i in order], sids, list(aggs), groups=np.array([self.gid[int(s)] for s in sids], np.int32),
                     n_groups=max(self.gid.values()) + 1, tmin=tmin, tmax=tmax, preds=list(preds), top_n=tn, top_agg=ta, top_desc=td,
                     group_keys=gkeys(keys))
        q = dataclasses.replace(to_gpu_query(self.bydb, [self.handles[i] for i in order], oq), flags=flags)
        return oq, q

    def query(self, keys, sids, cap, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, order=None, flags=0, ctx=""):
        oq, q = self.oquery(keys, sids, aggs, preds, tmin, tmax, top, order, flags)
        ctx = f"{ctx}/keys={[t for t, _ in keys]}/cap={cap}/preds={len(preds)}/top={top}/flags={flags}"
        fin = [self.ctx.scan_agg_keys_wide(q, gkeys(keys), cap) for _ in range(2)]
        got = fin[0]
        assert same_call(got, fin[1]), f"{ctx}: repeated calls differ"
        against_oracle(got, O.run_query(oq), aggs, flags, ctx)
        tuples = discovery(self.series, keys, oq.sids, tmin, tmax)
        assert got.n_tuples == len(tuples), f"{ctx}: n_tuples {got.n_tuples}, {len(tuples)} tuples in the selected blocks"
        for t, (tag, _) in enumerate(keys):
            vals = {c[t] for c in tuples}
            assert len(got.key_tables[t]) == len(vals) and set(got.key_tables[t]) == vals, f"{ctx}: table of {tag}"
        if not flags:
            par = [self.ctx.scan_partials_keys_wide(q, gkeys(keys), cap) for _ in range(2)]
            for k in ("group_id", "val_i64", "cnt_i64", "val_f64", "cnt_f64"):
                assert np.asarray(par[0][k]).tobytes() == np.asarray(par[1][k]).tobytes(), f"{ctx}: repeated partial calls differ ({k})"
            assert par[0]["key"] == par[1]["key"] and par[0]["n_tuples"] == got.n_tuples, f"{ctx}: partial keys / n_tuples"
            check_rows(par[0], oracle_rows(dataclasses.replace(oq, top_n=0), aggs, None), aggs, f"{ctx}/partial", 1e-9)
        return got

    def fails(self, code, keys, sids, cap, text=None, order=None):
        _, q = self.oquery(keys, sids, [("i", COUNT)], order=order)
        for fn in (self.ctx.scan_agg_keys_wide, self.ctx.scan_partials_keys_wide):
            with pytest.raises(self.bydb.BydbError) as e:
                fn(q, gkeys(keys), cap)
            assert e.value.code == code, (code, e.value)
            assert text is None or text in str(e.value), e.value


# ------------------------------------------------------------------ 1. code packing
PACK_STR = [("a", STR), ("b", STR), ("c", STR), ("d", STR)]
PACK_MIX = [("i", INT), ("a", STR), ("b", STR), ("j", INT)]
PACK_AGGS = [("i", SUM), ("i", COUNT), ("f", MAX), ("f", SUM)]


def pack_value(sid, r):
    return (sid - 1) * 256 + r


@functools.lru_cache(None)
def pack_series():
    """256 series of 256 rows; row r of series s holds v = 256 (s - 1) + r in every tag: a..d as b"v%05d", i and j as v - 32768
    (0 included).  65,536 values per tag, 256 per block, one tuple per row."""
    ss = []
    for sid in range(1, 257):
        v = [pack_value(sid, r) for r in range(256)]
        sv = [b"v%05d" % x for x in v]
        ss.append(ser(sid, 256, {"a": sv, "b": list(sv), "c": list(sv), "d": list(sv),
                                 "i": int_tag([x - 32768 for x in v]), "j": int_tag([x - 32768 for x in v])}))
    return ss


@functools.lru_cache(None)
def pack_part():
    return K.build_keyed(pack_series())


@gpu
@pytest.mark.parametrize("order", ["string", "mixed"])
def test_code_packing(bydb, gpu_ctx, order):
    ss = pack_series()
    keys = PACK_STR if order == "string" else PACK_MIX
    gid = {s.sid: s.sid % 3 for s in ss}
    with Tup(bydb, gpu_ctx, [(pack_part(), ss)], gid) as T:
        sids = list(gid)
        got = T.query(keys, sids, 65536, aggs=PACK_AGGS, ctx=f"pack {order}")
        assert got.n_tuples == 65536 == got.group_id.size and [len(t) for t in got.key_tables] == [65536] * 4
        T.fails(ENOMEM, keys, sids, 65535)
        T.query(keys, sids[:5] + sids[-5:], 65536, aggs=PACK_AGGS, top=(9, 1, False), ctx=f"pack {order} top")


# ------------------------------------------------------------------ 2. the component rules
S_POOL = [None, b"", b"x", b"ab", b"\x00", b"c"]
I_POOL = [None, 0, -1, I64_MIN, I64_MAX, 7]
S_TAGS, I_TAGS = ("sa", "sb", "sc", "sd"), ("ia", "ib", "ic", "id")
ALIAS = [(b"ab", b"c"), (b"a", b"bc"), (b"", b"x"), (b"x", b""), (None, b"x"), (b"x", None), (b"abc", b""), (b"", b"abc")]
RULE_ROWS = 200
RULE_KEYS = [list(zip(S_TAGS, [STR] * 4)), list(zip(I_TAGS, [INT] * 4)),
             [("sa", STR), ("ib", INT), ("sc", STR), ("id", INT)], [("ia", INT), ("sb", STR), ("ic", INT), ("sd", STR)]]
ALIAS_KEYS = [[("a", STR), ("b", STR)], [("a", STR), ("b", STR), ("sa", STR), ("ia", INT)], [("ib", INT), ("sc", STR), ("a", STR), ("b", STR)]]
RULE_GID = {1: 0, 2: 1, 3: 0, 10: 1, 11: 2, 12: 2}


def rule_cells(sid, part, x):
    """position k of row x: the pools cycled at strides 1, 6, 36 and 5 (every nil / "" / 0 combination across positions)"""
    idx = [(x + sid) % 6, (x // 6 + part) % 6, (x // 36 + sid) % 6, (5 * x + 1 + part) % 6]
    return [S_POOL[i] for i in idx], [I_POOL[i] for i in idx]


def alias_cells(sid, x):
    if sid == 10:
        return ALIAS[0]
    if sid == 11:
        return ALIAS[1]
    return ALIAS[(x + sid) % len(ALIAS)]


def rule_series(sid, part, drop=(), row0=0):
    rows = [rule_cells(sid, part, x) for x in range(RULE_ROWS)]
    tags = {}
    for k in range(4):
        if k not in drop:
            tags[S_TAGS[k]] = [r[0][k] for r in rows]
            tags[I_TAGS[k]] = int_tag([r[1][k] for r in rows])
    al = [alias_cells(sid, x) for x in range(RULE_ROWS)]
    tags["a"], tags["b"] = [c[0] for c in al], [c[1] for c in al]
    tags["z"] = [b"z%d" % (x % 3) for x in range(RULE_ROWS)]
    return ser(sid, RULE_ROWS, tags, row0=row0)


@functools.lru_cache(None)
def rule_parts():
    """part 0 (rows 0..199): series 1, 2, 3 and the alias series 10 (only ("ab", "c")), 11 (only ("a", "bc")) and 12 (every alias
    pair mixed); part k = 1..4 (rows 1000 k ..): series 1, 2, 3 without the position k - 1 tags; part 5 (rows 6000 ..): series 1, 2
    without any key column (only z)"""
    out = []
    ss = [rule_series(sid, 0) for sid in (1, 2, 3, 10, 11, 12)]
    out.append((K.build_keyed(ss), ss))
    for k in range(4):
        ss = [rule_series(sid, k + 1, drop=(k,), row0=1000 * (k + 1)) for sid in (1, 2, 3)]
        out.append((K.build_keyed(ss), ss))
    ss = [ser(sid, 50, {"z": [b"z%d" % (x % 3) for x in range(50)]}, row0=6000) for sid in (1, 2)]
    out.append((K.build_keyed(ss), ss))
    return out


@gpu
@pytest.mark.parametrize("ki", range(len(RULE_KEYS)))
def test_component_rules(bydb, gpu_ctx, ki):
    keys = RULE_KEYS[ki]
    with Tup(bydb, gpu_ctx, rule_parts(), RULE_GID) as T:
        sids = list(RULE_GID)
        got = T.query(keys, sids, 4096, ctx="rules")
        nil = tuple(comp(None, vt) for _, vt in keys)
        assert any(k == nil for k in got.key), "the block without key columns keys to the all-nil tuple"
        t0, vt0 = keys[0]
        p = O.Pred(FAM, t0, O.OP_NE, b"x" if vt0 == STR else -1)
        got = T.query(keys, sids, 4096, preds=[p], ctx="rules, a predicate on a key tag")
        assert got.n_tuples > len(set(got.key)), "n_tuples counts the tuples before the predicate"
        T.query(keys, [1, 2, 3], 4096, tmin=T0 + 37 * STEP, tmax=T0 + 3150 * STEP, ctx="rules, a time cut inside blocks")


@gpu
def test_alias_tuples(bydb, gpu_ctx):
    with Tup(bydb, gpu_ctx, rule_parts(), RULE_GID) as T:
        for keys in ALIAS_KEYS:
            got = T.query(keys, list(RULE_GID), 4096, ctx="alias")
            ai = [t for t, _ in keys].index("a")
            pairs = {(k[ai], k[ai + 1]) for k in got.key}
            assert {(b"ab", b"c"), (b"a", b"bc"), (b"", b"x"), (b"x", b"")} <= pairs, pairs
            T.query(keys, [10, 11], 4096, ctx="alias, blocks of their own")
            T.query(keys, [12], 4096, top=(3, 1, True), ctx="alias, mixed in one block")


@gpu
def test_order_top_n_and_row_path_types(bydb, gpu_ctx):
    """merged series groups, a time cut inside blocks, Top-N both ways over COUNT ties, BYDB_Q_ROW_PATH_TYPES"""
    merged = {1: 0, 2: 0, 3: 0, 10: 1, 11: 1, 12: 1}
    aggs = [("f", SUM), ("i", COUNT), ("f", COUNT), ("i", MAX), ("f", MIN)]
    with Tup(bydb, gpu_ctx, rule_parts(), merged) as T:
        sids = list(merged)
        for keys in (RULE_KEYS[2], ALIAS_KEYS[1]):
            cut = dict(tmin=T0 + 77 * STEP, tmax=T0 + 4133 * STEP)
            T.query(keys, sids, 4096, aggs=aggs, ctx="merged groups")
            counts = T.query(keys, sids, 4096, aggs=aggs, **cut, ctx="merged groups, cut").val_i64[:, 1].tolist()
            assert len(set(counts)) < len(counts), "COUNT ties"
            for top in ((6, 1, True), (6, 1, False), (40, 2, True)):
                T.query(keys, sids, 4096, aggs=aggs, top=top, **cut, ctx="top")
            T.query(keys, sids, 4096, aggs=aggs, flags=bydb.capi.Q_ROW_PATH_TYPES, ctx="row-path types")
            T.query(keys, sids, 4096, aggs=aggs, top=(5, 2, False), flags=bydb.capi.Q_ROW_PATH_TYPES, ctx="row-path types, top")


# ------------------------------------------------------------------ 3. tag order
ROT = [("sa", STR), ("ib", INT), ("a", STR)]


@gpu
def test_tag_order(bydb, gpu_ctx):
    with Tup(bydb, gpu_ctx, rule_parts(), RULE_GID) as T:
        sids = list(RULE_GID)
        base = T.query(ROT, sids, 4096, ctx="rotation 0")
        for r in (1, 2):
            keys = ROT[r:] + ROT[:r]
            got = T.query(keys, sids, 4096, ctx=f"rotation {r}")
            assert got.group_id.tolist() == base.group_id.tolist()
            assert [k[-r:] + k[:-r] for k in got.key] == base.key, f"rotation {r}: components"
            assert got.rows.tolist() == base.rows.tolist()
            assert got.val_i64.tobytes() == base.val_i64.tobytes() and got.val_f64.tobytes() == base.val_f64.tobytes(), f"rotation {r}"
            assert got.n_tuples == base.n_tuples


# ------------------------------------------------------------------ 4. tuples per block
M = (1 << 64) - 1
CHAIN_M = 180           # values of each chain tag introduced by the preamble rows (k, k)


def pair_home(pr):
    """tuple_block_keys' home of the pair word pr = 1 + (tuple so far << 8 | the tag's local index) in its 512-slot table"""
    return ((pr * 0x9e3779b97f4a7c15) & M) >> 55 & 511


@functools.lru_cache(None)
def chain_pairs():
    """rows (i, j) of the two chain tags: the preamble (k, k), k < CHAIN_M, numbers value k of each tag k (first seen); then every
    (i, j), i != j, whose pair homes at slot 511"""
    return [(k, k) for k in range(CHAIN_M)] + \
        [(i, j) for i in range(CHAIN_M) for j in range(CHAIN_M) if i != j and pair_home(1 + ((i << 8) | j)) == 511]


def probe_lengths(pairs):
    """linear probing of the distinct pairs in row order: the probes each pair takes"""
    table, out = [0] * 512, []
    for i, j in dict.fromkeys(pairs):
        pr = 1 + ((i << 8) | j)
        s, n = pair_home(pr), 0
        while table[s]:
            s, n = (s + 1) & 511, n + 1
        table[s] = pr
        out.append(n)
    return out


def grid_rows(seed):
    rows = [(z, w) for z in range(16) for w in range(16)]
    if seed:
        rows = [rows[i] for i in np.random.default_rng(seed).permutation(256).tolist()]
    return rows


@functools.lru_cache(None)
def block_parts():
    """one part: sid 1: 256 values of x, y / z / w constant; sid 2..4: the 16 x 16 grid of (z, w) (x, y constant) in three row
    orders; sid 5: 8,193 rows, (x, y) = ("a", 0) but ("b", 0) at row 8191 and ("a", 1) at row 8192; sid 6: the probe chain over
    (cx, cy).  A second part (later in time) holds sid 7: the grid plus one more tuple, 257 in its block."""
    def series(sid, n, x, y, z, w, cx=None, cy=None, row0=0):
        return ser(sid, n, {"x": x, "y": int_tag(y), "z": z, "w": w, "cx": cx or [b"c"] * n, "cy": cy or [b"c"] * n}, row0=row0)
    ss = [series(1, 256, [b"x%03d" % r for r in range(256)], [5] * 256, [b"k"] * 256, [b""] * 256)]
    for sid, seed in ((2, 0), (3, 1), (4, 2)):
        g = grid_rows(seed)
        ss.append(series(sid, 256, [b"k"] * 256, [0] * 256, [b"z%02d" % z for z, _ in g], [b"w%02d" % w for _, w in g]))
    n = BLOCK
    x = [b"a"] * n
    y = [0] * n
    x[8191], y[8192] = b"b", 1
    ss.append(series(5, n, x, y, [b"k"] * n, [b"k"] * n))
    ch = chain_pairs()
    ss.append(series(6, len(ch), [b"k"] * len(ch), [0] * len(ch), [b"k"] * len(ch), [b"k"] * len(ch),
                     [b"c%03d" % i for i, _ in ch], [b"c%03d" % j for _, j in ch]))
    g = grid_rows(3) + [(0, 16)]
    bad = [series(7, 257, [b"k"] * 257, [0] * 257, [b"z%02d" % z for z, _ in g], [b"w%02d" % w for _, w in g], row0=20000)]
    return [(K.build_keyed(ss), ss), (K.build_keyed(bad), bad)]


BLOCK_KEYS = [("x", STR), ("y", INT), ("z", STR), ("w", STR)]


@gpu
def test_tuples_per_block(bydb, gpu_ctx):
    ps = block_parts()
    gid = {s.sid: s.sid % 2 for _, ss in ps for s in ss}
    with Tup(bydb, gpu_ctx, ps[:1], gid) as T:
        got = T.query(BLOCK_KEYS, [1], 1024, ctx="256 tuples from the first tag")
        assert got.n_tuples == 256
        got = T.query(BLOCK_KEYS, [2], 1024, ctx="16 x 16 in the last two tags")
        assert got.n_tuples == 256 and [len(t) for t in got.key_tables] == [1, 1, 16, 16]
        got = T.query(BLOCK_KEYS, [2, 3, 4], 1024, ctx="one grid in three row orders")
        assert got.n_tuples == 256 and got.group_id.size == 512
        T.query([("z", STR), ("w", STR)], [3, 4], 1024, ctx="grid, two tags")
        got = T.query(BLOCK_KEYS, [5], 1024, ctx="8,193 rows")
        assert got.key == [(b"a", le(0), b"k", b"k"), (b"b", le(0), b"k", b"k"), (b"a", le(1), b"k", b"k")]
        assert got.rows.tolist() == [BLOCK - 2, 1, 1]
        T.query(BLOCK_KEYS, [5], 1024, tmin=T0 + 8191 * STEP, ctx="8,193 rows, the last two")
        T.query(BLOCK_KEYS, [5], 1024, tmin=T0 + 8000 * STEP, tmax=T0 + 8191 * STEP, ctx="8,193 rows, cut at 8191")
        for keys in ([("cx", STR), ("cy", STR)], [("cx", STR), ("cy", STR), ("y", INT), ("w", STR)], [("z", STR), ("cx", STR), ("cy", STR)]):
            got = T.query(keys, [6], 1024, ctx="probe chain")
            assert got.n_tuples == len(set(chain_pairs()))
        T.query(BLOCK_KEYS, [1, 2, 3, 4, 5, 6], 4096, ctx="every block")
    with Tup(bydb, gpu_ctx, ps[1:], gid) as T:
        T.fails(ENOTSUP, BLOCK_KEYS, [7], 1024, text="256 distinct key tuples")
        T.fails(ENOTSUP, BLOCK_KEYS, [7], 1024, text="block #0")
        got = T.query([("z", STR), ("y", INT)], [7], 1024, ctx="the same block, fewer tags")
        assert got.n_tuples == 16


# ------------------------------------------------------------------ 5. many parts
PART_ROWS = 40


@functools.lru_cache(None)
def many_parts(n_parts):
    """n_parts time-disjoint parts: series s (1..8) in part p unless (5 s + p) % 4 == 0, its tuple (x, y) depending on p; every
    11th part holds only series 99"""
    out = []
    for p in range(n_parts):
        ss = []
        for sid in ([99] if p % 11 == 7 else [s for s in range(1, 9) if (5 * s + p) % 4]):
            x = [b"v%02d" % ((p * 3 + sid + i // 10) % 37) for i in range(PART_ROWS)]
            y = int_tag([None if (i + p) % 9 == 0 else (p + sid + i // 7) % 5 - 2 for i in range(PART_ROWS)])
            ss.append(ser(sid, PART_ROWS, {"x": x, "y": y}, row0=p * PART_ROWS))
        out.append((K.build_keyed(ss), ss))
    return out


def shuffled(n, seed):
    return np.random.default_rng(seed).permutation(n).tolist()


@gpu
@pytest.mark.parametrize("n_parts", [33, 64])
def test_many_parts(bydb, gpu_ctx, n_parts):
    ps = many_parts(n_parts)
    gid = {s: s % 3 for s in list(range(1, 9)) + [99]}
    keys = [("y", INT), ("x", STR)]
    with Tup(bydb, gpu_ctx, ps, gid) as T:
        for seed in (1, 2):
            order = shuffled(n_parts, seed)
            T.query(keys, range(1, 9), 1024, order=order, ctx=f"{n_parts} parts")
            T.query(keys, [1, 4, 7], 1024, order=order, top=(5, 1, True), tmin=T0 + 5 * PART_ROWS * STEP + 7,
                    tmax=T0 + (n_parts - 3) * PART_ROWS * STEP, ctx=f"{n_parts} parts, cut, top")
    if n_parts == 64:
        extra = K.build_keyed([ser(1, 5, {"x": [b"x"] * 5, "y": int_tag([1] * 5)}, row0=64 * PART_ROWS)])
        with Tup(bydb, gpu_ctx, ps + [(extra, [])], gid) as T:
            T.fails(EINVAL, keys, [1, 2], 1024)
    else:
        over = K.build_keyed([ser(2, 5, {"x": [b"x"] * 5, "y": int_tag([1] * 5)}, row0=3 * PART_ROWS + 2)])
        with Tup(bydb, gpu_ctx, ps + [(over, [])], gid) as T:
            T.fails(ENOTSUP, keys, [1, 2], 1024)


# ------------------------------------------------------------------ 7. the collective
COLL_KEYS = [("a", STR), ("i", INT), ("b", STR), ("j", INT)]   # the 65,536-value int64 tag j in bits 48-63


def rank_of(sid):
    return min(R - 1, (sid - 1) // 86)


@functools.lru_cache(None)
def pack_case():
    """the code packing fixture split by series range: series 1..86 on rank 0, 87..172 on rank 1, 173..256 on rank 2"""
    ss = pack_series()
    shards = [[K.build_keyed([s for s in ss if rank_of(s.sid) == r])] for r in range(R)]
    return Case(shards, [pack_part()], {s.sid: s.sid % 3 for s in ss}), ss


@functools.lru_cache(None)
def union_case(n_values, extra):
    """tag u with n_values values over three ranks (a third each, by series), t constant: n_values tuples; `extra` adds series 40
    on rank 2 with one value more"""
    per = -(-n_values // R)
    by_rank, ss = [[] for _ in range(R)], []
    for r in range(R):
        vals = list(range(r * per, min(n_values, (r + 1) * per)))
        for k in range(0, len(vals), 100):
            chunk = vals[k:k + 100]
            s = ser(1 + r * 10 + k // 100, len(chunk), {"u": [b"u%05d" % v for v in chunk], "t": [b"t"] * len(chunk)})
            by_rank[r].append(s)
            ss.append(s)
    if extra:
        s = ser(40, 2, {"u": [b"u%05d" % n_values] * 2, "t": [b"t"] * 2})
        by_rank[2].append(s)
        ss.append(s)
    gid = {s.sid: s.sid % 2 for s in ss}
    return Case([[K.build_keyed(b)] for b in by_rank], [K.build_keyed(ss)], gid), ss


def collective(bydb, ranks, case, series, keys, root, max_values, partial, aggs, ctx, **kw):
    """the root's answer against the oracle over all ranks' parts; every other rank answers nothing"""
    qs = [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], aggs=aggs, **kw)) for r in range(R)]
    fn = (lambda r: ranks.ctxs[r].scan_reduce_keys_wide_partials(qs[r], gkeys(keys), root=root, max_values=max_values)) if partial else \
        (lambda r: ranks.ctxs[r].scan_reduce_keys_wide(qs[r], gkeys(keys), root=root, max_values=max_values))
    res, codes = ranks.run(fn)
    assert codes == [0] * R, f"{ctx}: {codes}"
    oq = dataclasses.replace(case.oquery([p for s in case.shards for p in s], aggs=aggs, **kw), group_keys=gkeys(keys))
    got = res[root]
    if partial:
        check_rows(got, oracle_rows(dataclasses.replace(oq, top_n=0), aggs, None), aggs, f"{ctx}/partial", 1e-9)
        n_tuples, tables = got["n_tuples"], got["key_tables"]
    else:
        against_oracle(got, O.run_query(oq), aggs, 0, ctx)
        n_tuples, tables = got.n_tuples, got.key_tables
    tuples = discovery(series, keys, oq.sids, oq.tmin, oq.tmax)
    assert n_tuples == len(tuples), f"{ctx}: n_tuples {n_tuples} vs {len(tuples)}"
    for t in range(len(keys)):
        assert len(tables[t]) == len({c[t] for c in tuples}) and set(tables[t]) == {c[t] for c in tuples}, f"{ctx}: table {t}"
    for r in range(R):
        if r != root:
            other = res[r]
            assert len(other["group_id"] if partial else other.group_id) == 0, f"{ctx}: rank {r} got rows"
    return got


@gpu
def test_collective_code_packing(bydb, gpu_ctx, quiet):  # noqa: F811
    case, ss = pack_case()
    slot = max(tuple_slot(bydb, case, gkeys(keys), 65536, 65536, aggs=PACK_AGGS) for keys in (COLL_KEYS, PACK_STR))
    ranks = Ranks(bydb, slot, case.shards)
    try:
        got = collective(bydb, ranks, case, ss, COLL_KEYS, 0, 65536, False, PACK_AGGS, "collective")
        assert got.n_tuples == 65536 == got.group_id.size and [len(t) for t in got.key_tables] == [65536] * 4
        collective(bydb, ranks, case, ss, COLL_KEYS, 2, 65536, True, PACK_AGGS, "collective partial")
        collective(bydb, ranks, case, ss, PACK_STR, 1, 65536, False, PACK_AGGS, "collective strings", top=(7, 1, False))
    finally:
        ranks.close()


@gpu
def test_collective_tag_union_cap(bydb, gpu_ctx, quiet):  # noqa: F811
    keys = [("t", STR), ("u", STR)]
    aggs = [("i", SUM), ("f", SUM)]
    at, _ = union_case(600, False)
    over, _ = union_case(600, True)
    ranks = Ranks(bydb, max(tuple_slot(bydb, c, gkeys(keys), 601, 1024, aggs=aggs) for c in (at, over)), at.shards)
    try:
        got = collective(bydb, ranks, at, union_case(600, False)[1], keys, 1, 600, False, aggs, "union at the cap")
        assert [len(t) for t in got.key_tables] == [1, 600]
        ranks.register(over.shards)
        qs = [to_gpu_query(bydb, ranks.hs[r], over.oquery(over.shards[r], aggs=aggs)) for r in range(R)]
        msg = {}

        def call(r):
            try:
                return ranks.ctxs[r].scan_reduce_keys_wide(qs[r], gkeys(keys), root=1, max_values=600)
            except bydb.BydbError as e:
                msg[r] = str(e)
                raise
        _, codes = ranks.run(call)
        assert codes == [0, ENOMEM, 0], codes
        assert "distinct values of the tag default/u" in msg[1], msg
        plain_ok(bydb, gpu_ctx, ranks, over, 0)
        collective(bydb, ranks, over, union_case(600, True)[1], keys, 2, 601, True, aggs, "union one over, raised cap")
    finally:
        ranks.close()


# ------------------------------------------------------------------ the oracle's tuple key, on the CPU
def fold_model(parts_series, keys, gid, sids):
    """a plain fold: rows by series then time; a row's composite is (series group, tuple of components by the component rule);
    -> [((group, key), rows, int64 SUM of i)] in first-seen order"""
    tags, types = zip(*keys)
    sel = set(int(s) for s in sids)
    rows = []
    for _, ss in parts_series:
        for s in ss:
            if s.sid in sel:
                cells = tuple_cells(s, tags, types)
                rows += [(s.sid, int(s.ts[r]), cells[r], int(s.fields["i"][1][r])) for r in range(s.n)]
    out = {}
    for sid, _, key, iv in sorted(rows, key=lambda x: (x[0], x[1])):
        e = out.setdefault((gid[sid], key if len(keys) > 1 else key[0]), [0, 0])
        e[0] += 1
        e[1] = (e[1] + iv + (1 << 63)) % (1 << 64) - (1 << 63)
    return [(k, n, s) for k, (n, s) in out.items()]


def test_oracle_tuples_match_a_plain_fold():
    ps = rule_parts()
    parts = [p for p, _ in ps]
    sids = np.array(sorted(RULE_GID), np.uint64)
    groups = np.array([RULE_GID[int(s)] for s in sids], np.int32)
    for keys in RULE_KEYS + ALIAS_KEYS + [ROT, [("sa", STR)], [("ia", INT)]]:
        oq = O.Query(parts, sids, [("i", COUNT), ("i", SUM)], groups=groups, n_groups=3, group_keys=gkeys(keys))
        r = O.run_query(oq)
        want = fold_model(ps, keys, RULE_GID, sids)
        assert list(zip(r.group_id.tolist(), r.key)) == [w[0] for w in want], keys
        assert r.rows.tolist() == [w[1] for w in want] == r.val_i64[:, 0].tolist(), keys
        assert r.val_i64[:, 1].tolist() == [w[2] for w in want], keys
    # the aliases stay apart, in blocks of their own and mixed in one block; nil is "" and 0 in every position
    oq = O.Query(parts, np.array([10, 11, 12], np.uint64), [("i", COUNT)], groups=np.zeros(3, np.int32), n_groups=1,
                 group_keys=gkeys(ALIAS_KEYS[0]))
    keys = O.run_query(oq).key
    assert keys[:2] == [(b"ab", b"c"), (b"a", b"bc")] and len(keys) == len(set(keys)) == len({(a or b"", b or b"") for a, b in ALIAS})
    assert (b"", b"x") in keys and (b"x", b"") in keys and (b"", b"abc") in keys and (b"abc", b"") in keys
    # a column missing from a block and a nil cell are the same component
    r = O.run_query(O.Query(parts, sids, [("i", COUNT)], groups=groups, n_groups=3, group_keys=gkeys(RULE_KEYS[2])))
    nil = (b"", le(0), b"", le(0))
    assert nil in r.key
    # without the length prefix the four tuples that concatenate to "abc" would be one key: the encoding keeps them apart
    assert len({k for k in keys if k[0] + k[1] == b"abc"}) == 4


def test_oracle_int64_component_is_its_string_twin():
    """an int64 key in the oracle answers what the oracle answers on the string twin (the 8 little-endian bytes, nil as 0)"""
    from tests.test_gpu_keyed_int64 import twin
    ss = []
    for sid in (1, 2, 5):
        c = [[None, 0, -1, I64_MIN, I64_MAX, 7, 1 << 40][(x * 3 + sid) % 7] for x in range(300 + sid)]
        ss.append(ser(sid, len(c), {"n": int_tag(c), "nt": twin(c)}))
    part = K.build_keyed(ss)
    sids = np.array([1, 2, 5], np.uint64)
    base = dict(aggs=[("i", SUM), ("f", MAX), ("i", COUNT)], groups=np.array([0, 1, 0], np.int32), n_groups=2)
    for extra in (dict(), dict(top_n=3, top_agg=2), dict(tmin=T0 + 50 * STEP, tmax=T0 + 250 * STEP)):
        a = O.run_query(O.Query([part], sids, **base, **extra, group_keys=[(FAM, "n", INT)]))
        b = O.run_query(O.Query([part], sids, **base, **extra, group_key=(FAM, "nt")))
        assert a.key == b.key and a.group_id.tolist() == b.group_id.tolist() and a.rows.tolist() == b.rows.tolist()
        assert a.val_i64.tobytes() == b.val_i64.tobytes() and a.val_f64.tobytes() == b.val_f64.tobytes()
        assert le(0) in a.key
    with pytest.raises(RuntimeError, match="group key"):
        O.run_query(O.Query([part], sids, **base, group_keys=[(FAM, "nt", INT)]))
    with pytest.raises(RuntimeError, match="group key"):
        O.run_query(O.Query([part], sids, **base, group_keys=[(FAM, "n", STR)]))
    with pytest.raises(RuntimeError, match="group key"):
        O.run_query(O.Query([part], sids, **base, group_keys=[(FAM, "n", INT)] * 5))


# ------------------------------------------------------------------ the claimed shapes, on the CPU
def test_tuple_case_layouts():
    # code packing: one value per row in every tag, 65,536 values, 256 per block on dictionary pages, 0 among the int64 values
    ss = pack_series()
    assert len(ss) == 256 and all(s.n == 256 and s.chunks() == [(0, 256)] for s in ss)
    vals = [c for s in ss for c in s.tags["a"]]
    assert len(set(vals)) == 65536 and all(s.tags["a"] == s.tags["b"] == s.tags["c"] == s.tags["d"] for s in ss)
    ivals = np.concatenate([s.tags["j"][0] for s in ss])
    assert len(set(ivals.tolist())) == 65536 and 0 in ivals and not any(s.tags["j"][1].any() for s in ss)
    assert all(str_tag_class(s.tags["a"]) == "dict" for s in ss[:2] + ss[-2:])
    assert len(discovery(ss, PACK_MIX, [s.sid for s in ss], I64_MIN, I64_MAX)) == 65536
    # the collective's split: j's 65,536 values over three ranks, every rank alone far under the cap
    case, _ = pack_case()
    per = [sum(1 for s in ss if rank_of(s.sid) == r) * 256 for r in range(R)]
    assert sum(per) == 65536 and max(per) < 32768
    # the component rules: every pool entry in every position, at most 256 tuples per block, the missing columns
    ps = rule_parts()
    for k in range(4):
        assert {c for _, ss in ps[:1] for s in ss for c in s.tags[S_TAGS[k]]} == set(S_POOL)
        assert {None if nl else int(v) for s in ps[0][1] for v, nl in zip(*s.tags[I_TAGS[k]])} == set(I_POOL)
        assert all(S_TAGS[k] not in s.tags and I_TAGS[k] not in s.tags for s in ps[k + 1][1])
        assert all(S_TAGS[j] in s.tags for j in range(4) if j != k for s in ps[k + 1][1])
    assert all(set(s.tags) == {"z"} for s in ps[5][1])
    for keys in RULE_KEYS + ALIAS_KEYS:
        tags, types = zip(*keys)
        for _, ss in ps:
            for s in ss:
                assert all(len(set(tuple_cells(s, tags, types)[lo:hi])) <= 256 for lo, hi in s.chunks())
    spans = [(min(int(s.ts[0]) for s in ss), max(int(s.ts[-1]) for s in ss)) for _, ss in ps]
    assert all(a[1] < b[0] for a, b in zip(spans, spans[1:]))
    assert set(ps[0][1][3].tags["a"]) == {b"ab"} and set(ps[0][1][4].tags["a"]) == {b"a"}
    assert len(set(zip(ps[0][1][5].tags["a"], ps[0][1][5].tags["b"]))) == len(ALIAS)
    # tuples per block
    (p, bs), (_, bad) = block_parts()
    by = {s.sid: s for s in bs}
    tup = lambda s, keys: [c for lo, hi in s.chunks() for c in [set(tuple_cells(s, *zip(*keys))[lo:hi])]]  # noqa: E731
    assert [len(c) for c in tup(by[1], BLOCK_KEYS)] == [256] and len(set(by[1].tags["x"])) == 256
    for sid in (2, 3, 4):
        assert [len(c) for c in tup(by[sid], BLOCK_KEYS)] == [256]
    firsts = [list(dict.fromkeys(by[sid].tags["z"]))[:4] for sid in (2, 3, 4)]
    assert firsts[0] != firsts[1] != firsts[2], "the grid's first-seen order differs block to block"
    s5 = by[5]
    assert s5.n == BLOCK and s5.chunks() == [(0, BLOCK)] and s5.tags["x"].index(b"b") == 8191 and s5.tags["y"][0].tolist().index(1) == 8192
    assert [len(c) for c in tup(bad[0], BLOCK_KEYS)] == [257] and bad[0].chunks() == [(0, 257)]
    # the probe chain: first-seen order numbers value k of each chain tag k; 62 pairs homed at 511, the chain wraps past slot 0
    s6 = by[6]
    for tag in ("cx", "cy"):
        assert list(dict.fromkeys(s6.tags[tag])) == [b"c%03d" % k for k in range(CHAIN_M)]
        assert str_tag_class(s6.tags[tag]) == "dict"
    ch = chain_pairs()
    assert len(set(ch)) == len(ch) <= 256 and s6.chunks() == [(0, len(ch))]
    homed = [pr for pr in ch if pair_home(1 + ((pr[0] << 8) | pr[1])) == 511]
    assert len(homed) == 62
    assert max(probe_lengths(ch)) >= 61
    # many parts: time-disjoint, some select nothing
    for n in (33, 64):
        ps = many_parts(n)
        spans = [(min(int(s.ts[0]) for s in ss), max(int(s.ts[-1]) for s in ss)) for _, ss in ps]
        assert all(a[1] < b[0] for a, b in zip(spans, spans[1:]))
        assert sum(all(s.sid == 99 for s in ss) for _, ss in ps) == len([q for q in range(n) if q % 11 == 7])
    # the tag-union case: 600 values of u over three ranks, 601 with the extra series
    for extra, n in ((False, 600), (True, 601)):
        case, ss = union_case(600, extra)
        assert len({c for s in ss for c in s.tags["u"]}) == n
        assert max(len({c for s in ss if s in case_series(case, r, ss) for c in s.tags["u"]}) for r in range(R)) <= 201
    # every float field positive: the float bound is 2e-9 x |reference|
    for ss in [pack_series(), [s for _, x in rule_parts() for s in x], bs]:
        assert all((s.fields["f"][1] > 0).all() for s in ss)


def case_series(case, r, ss):
    sids = set()
    for p in case.shards[r]:
        sids |= {int(x) for x in O.scan_rows(O.Query([p], np.array(sorted({s.sid for s in ss}), np.uint64), [("i", COUNT)]))["sid"]}
    return [s for s in ss if s.sid in sids]

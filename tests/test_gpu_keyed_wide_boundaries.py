"""The wide group-by on a stored tag (bydb_scan_agg_keyed_wide / bydb_scan_partials_keyed_wide, DESIGN.md 4.6) against the oracle
at the boundaries of its own machinery in csrc/scan_kernels.cu ("Wide group key"):
  1. the value table of pow2(max(2 * cap, 1024)) slots: caps 511 .. 65,536 at V = cap (answers) and V = cap + 1 (BYDB_ENOMEM),
     values homed at the last slot (probes wrap to 0), a chain sharing one home at load 1/2, "" and nil behind a chain, 64-byte
     values that differ in their last byte; the same for int64 keys with INT64_MIN, INT64_MAX, -1, 0 and nil;
  2. the block-local int64 table (512 slots in shared memory, the value 0 on a flag of its own): 256 values homed at local slot
     511 with and without the 0;
  3. the record sort over N = pow2(max(R, 2048)) keys: R = 1, 2047, 2048, 2049, 4096, 4097 and 8193 records, every other record
     empty, one surviving record, none;
  4. one composite of 1, 31, 32, 33, 64, 65 and 1,000 records folded by wide_fold_kernel, over a narrow delta, a decimal float
     and a raw float field with nulls;
  5. scan_rank over 33 and 64 time-disjoint parts passed in shuffled order, series in subsets of the parts, parts that select
     nothing, and 65 parts refused;
  6. the 128-bit block sums: int64 sums that wrap, decimal mantissas near +-2^62 over 8,192-row blocks, MIN / MAX at the int64
     extremes, an 8,193-row block whose key changes at rows 8191 and 8192, and a composite whose values cancel;
  7. the prepared form and the collective over the same fixtures.

Every answer is checked against the oracle keyed on the tag (an int64 key through its string twin) or, where the oracle would be
slow, against key_model, a plain Python fold: composite groups in order, key bytes, rows, counts, int64 values and MIN / MAX bit for
bit; three calls of each form give identical answers, the partial form the same composite groups and keys.

Float sums (the restated contract): the wide path sums a decimal page's block in the exact integer domain and rounds once, where
the reference adds doubles one after another.  For a composite whose values cancel (0.1 + 0.2 - 0.3) the reference gives
5.55e-17 and the exact sum is 0, so no relative bound holds; the bound is 1e-9 x the sum of |x| over the composite's values plus
1e-9 x |reference| (`float_close`).  The per-value passes and the express lane sum decimal pages the same way and give the same 0.
"""
import dataclasses
import functools

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_gpu_keyed as K
from tests.helpers import STEP, T0, to_gpu_query
from tests.test_gpu_fallback import BLOCK, COUNT, MAX, MEAN, MIN, SUM, F, I, Series
from tests.test_gpu_keyed_int64 import KX, int_tag, twin
from tests.test_gpu_keyed_reduce import R as N_RANKS
from tests.test_gpu_keyed_reduce import Case, Ranks, quiet, split  # noqa: F401 -- quiet is a fixture
from tests.test_gpu_keyed_wide import identical, le
from tests.test_gpu_keyed_wide_reduce import check, wide_slot
from tests.test_gpu_masks import I64_MAX, I64_MIN, str_tag_class

gpu = pytest.mark.gpu
FAM, KT = K.FAM, K.KT
HOME_MASK = (1 << 17) - 1     # the largest value table: 131,072 slots (cap 65,536); a home under it is a home under every smaller one
LOCAL_MASK = 511              # kLocalSlots - 1: the block-local int64 table
STR_CAPS = [511, 512, 513, 1024, 1025, 65536]
I64_CAPS = [512, 1025, 65536]
ORACLE_MAX_CAP = 1025         # above it the fixtures are checked against key_model alone
AGGS4 = [("i", SUM), ("i", COUNT), ("f", MAX), ("f", SUM)]
_pid = [7_300_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def table_slots(cap):
    """slots of the wide value table at `cap` (wide_discover's S)"""
    s = 1
    while s < max(2 * cap, 1024):
        s <<= 1
    return s


# ------------------------------------------------------------------ FNV-1a of key_home / key_slot_i64, for any mask
_FNV0, _FNVP = 0xcbf29ce484222325, 0x100000001b3


def fnv_slot(b, mask):
    """home slot of bytes b in a table of mask + 1 slots: FNV-1a over the bytes, (h ^ h >> 32) & mask"""
    h = _FNV0
    for x in b:
        h = ((h ^ x) * _FNVP) & 0xFFFF_FFFF_FFFF_FFFF
    return (h ^ (h >> 32)) & mask


def i64_slot(v, mask):
    """home slot of an int64 value: FNV-1a over its 8 little-endian bytes"""
    return fnv_slot(le(v), mask)


def _fnv_rows(state, cols, mask):
    """vectorised fnv_slot: `state` the hash after a common prefix, cols the remaining bytes, one uint8 column each"""
    h = np.full(cols[0].size, np.uint64(state), np.uint64)
    with np.errstate(over="ignore"):
        for c in cols:
            h = (h ^ c.astype(np.uint64)) * np.uint64(_FNVP)
    return ((h ^ (h >> np.uint64(32))) & np.uint64(mask)).astype(np.int64)


def _prefix_state(prefix):
    h = _FNV0
    for x in prefix:
        h = ((h ^ x) * _FNVP) & 0xFFFF_FFFF_FFFF_FFFF
    return h


def find_str(slot, n, prefix, mask=HOME_MASK, exclude=()):
    """n values prefix + 8 counter bytes (big endian) homed at `slot`"""
    out, start, st = [], 1, _prefix_state(prefix)
    while len(out) < n:
        c = np.arange(start, start + (1 << 20), dtype=np.uint64)
        cols = [((c >> np.uint64(8 * (7 - k))) & np.uint64(0xff)).astype(np.uint8) for k in range(8)]
        for i in np.nonzero(_fnv_rows(st, cols, mask) == slot)[0].tolist():
            v = prefix + int(c[i]).to_bytes(8, "big")
            if v not in exclude and len(out) < n:
                out.append(v)
        start += 1 << 20
    return out


def find_i64(slot, n, mask, start=1, exclude=()):
    """n non-zero int64 values homed at `slot` (the counter times an odd constant, so the values spread over the range)"""
    out = []
    while len(out) < n:
        c = (np.arange(start, start + (1 << 20), dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        cols = [((c >> np.uint64(8 * k)) & np.uint64(0xff)).astype(np.uint8) for k in range(8)]
        for i in np.nonzero(_fnv_rows(_FNV0, cols, mask) == slot)[0].tolist():
            v = int(c[i].astype(np.int64))
            if v != 0 and v not in exclude and v not in out and len(out) < n:
                out.append(v)
        start += 1 << 20
    return out


# ------------------------------------------------------------------ the restated float bound and the checks
def float_close(g, m, x, fn):
    """|got - want| <= 1e-9 * (sum |x| of the composite [/ n for MEAN] + |want|)"""
    s = float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1)
    return abs(float(g) - float(m)) <= 1e-9 * (s + abs(float(m)))


def _bits(x):
    return np.array([x], np.float64).view(np.uint64)[0]


def against_model(got, exp, aggs, ctx):
    assert list(zip(got.group_id.tolist(), got.key)) == [e[0] for e in exp], \
        f"{ctx}: composites {list(zip(got.group_id.tolist(), got.key))[:8]}, model {[e[0] for e in exp][:8]}"
    assert got.rows.tolist() == [e[1] for e in exp], f"{ctx}: rows"
    for i, (ck, _, vals) in enumerate(exp):
        for a, ((f, fn), (m, x)) in enumerate(zip(aggs, vals)):
            where = f"{ctx}: composite {ck} agg {a} ({f},{fn})"
            if not got.is_float[a]:
                assert int(got.val_i64[i, a]) == m, f"{where}: {got.val_i64[i, a]}, model {m}"
            elif fn in (MIN, MAX):
                # the model folds the values written; a 17-digit value on a decimal page reads back within an ulp (bit for bit
                # as the reference reads it: against_oracle)
                g = float(got.val_f64[i, a])
                assert _bits(g) == _bits(m) or abs(g - m) <= 4.5e-16 * abs(m), f"{where}: {g!r}, model {m!r}"
            else:
                assert float_close(got.val_f64[i, a], m, x, fn), f"{where}: {got.val_f64[i, a]!r}, model {m!r}"


def against_oracle(got, want, exp, aggs, ctx):
    """the oracle's answer: groups, keys, rows, int64 values and float MIN / MAX exactly, float sums within float_close (the sum
    of |x| from the model `exp`, whose composites against_model has already matched)"""
    assert got.group_id.tolist() == want.group_id.tolist(), f"{ctx}: groups vs oracle"
    assert got.key == want.key, f"{ctx}: keys {got.key[:8]} vs oracle {want.key[:8]}"
    assert got.rows.tolist() == want.rows.tolist(), f"{ctx}: rows vs oracle"
    assert got.is_float.tolist() == want.is_float.tolist(), f"{ctx}: typing vs oracle"
    for a, (f, fn) in enumerate(aggs):
        if not want.is_float[a]:
            assert got.val_i64[:, a].tolist() == want.val_i64[:, a].tolist(), f"{ctx}: int64 agg {a} ({f},{fn}) vs oracle"
        elif fn in (MIN, MAX):
            assert got.val_f64[:, a].view(np.uint64).tolist() == want.val_f64[:, a].view(np.uint64).tolist(), \
                f"{ctx}: float agg {a} ({f},{fn}) vs oracle (bit-exact)"
        else:
            for i, (_, _, vals) in enumerate(exp):
                assert float_close(got.val_f64[i, a], want.val_f64[i, a], vals[a][1], fn), \
                    f"{ctx}: float agg {a} ({f},{fn}) row {i}: {got.val_f64[i, a]!r} vs oracle {want.val_f64[i, a]!r}"


class Wide:
    """Parts registered once; each query through both wide calls (three times each), against key_model, the oracle, the
    partial form, the discovery count and the plain scan's counters.  key: the device's tag; mkey: the tag key_model and the
    oracle group by (the string twin of an int64 key)."""

    def __init__(self, bydb, ctx, parts_series, gid, key=KT, mkey=None, vt=0):
        self.bydb, self.ctx, self.gid = bydb, ctx, gid
        self.parts = [p for p, _ in parts_series]
        self.series = [s for _, ss in parts_series for s in ss]
        self.key, self.mkey, self.vt = key, mkey or key, vt
        self.handles = []

    def __enter__(self):
        pid = _next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, p in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def oquery(self, sids, aggs, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, order=None):
        sids = np.array(sorted(int(s) for s in sids), np.uint64)
        tn, ta, td = top or (0, 0, True)
        order = list(range(len(self.parts))) if order is None else order
        oq = O.Query([self.parts[i] for i in order], sids, list(aggs), groups=np.array([self.gid[int(s)] for s in sids], np.int32),
                     n_groups=max(self.gid.values()) + 1, tmin=tmin, tmax=tmax, preds=list(preds), top_n=tn, top_agg=ta, top_desc=td)
        return oq, to_gpu_query(self.bydb, [self.handles[i] for i in order], oq)

    def query(self, sids, cap, aggs=AGGS4, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, order=None, oracle=True, ctx=""):
        preds = list(preds)
        oq, q = self.oquery(sids, aggs, preds, tmin, tmax, top, order)
        ctx = f"{ctx}/cap={cap}/preds={len(preds)}/top={top}"
        fin = [self.ctx.scan_agg_keyed_wide(q, FAM, self.key, cap, self.vt) for _ in range(3)]
        par = [self.ctx.scan_partials_keyed_wide(q, FAM, self.key, cap, self.vt) for _ in range(3)]
        got = fin[0]
        assert identical(got, fin[1]) and identical(got, fin[2]), f"{ctx}: repeated finalised calls differ"
        assert identical(par[0], par[1]) and identical(par[0], par[2]), f"{ctx}: repeated partial calls differ"
        exp = K.key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, self.mkey, top)
        against_model(got, exp, aggs, ctx)
        if oracle:
            against_oracle(got, O.run_query(dataclasses.replace(oq, group_key=(FAM, self.mkey))), exp, aggs, ctx)
        # the partial form: every present composite group in insertion order, with its key
        every = exp if not top else K.key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, self.mkey, None)
        assert list(zip(np.asarray(par[0]["group_id"]).tolist(), par[0]["key"])) == [e[0] for e in every], f"{ctx}: partial rows"
        # discovery: the distinct values of the selected blocks; one pass: the plain scan's counters
        blocks = K.selected_blocks(self.series, oq.sids, tmin, tmax)
        V = len({c for s, lo, hi in blocks for c in K.key_cells(s, self.mkey)[lo:hi]})
        assert got.n_keys == V == par[0]["n_keys"], f"{ctx}: n_keys {got.n_keys}, {V} values in the selected blocks"
        st, plain = got.stats, self.ctx.scan_agg(q).stats
        assert (st.rows_scanned, st.blocks_scanned, st.rows_matched) == (plain.rows_scanned, plain.blocks_scanned, plain.rows_matched), \
            f"{ctx}: wide counters {(st.rows_scanned, st.blocks_scanned, st.rows_matched)} vs plain " \
            f"{(plain.rows_scanned, plain.blocks_scanned, plain.rows_matched)}"
        assert st.rows_matched == sum(e[1] for e in every), f"{ctx}: rows_matched"
        return got, q

    def fails(self, code, sids, cap, aggs=AGGS4, order=None, text=None):
        _, q = self.oquery(sids, aggs, order=order)
        for fn in (self.ctx.scan_agg_keyed_wide, self.ctx.scan_partials_keyed_wide):
            with pytest.raises(self.bydb.BydbError) as e:
                fn(q, FAM, self.key, cap, self.vt)
            assert e.value.code == code, (code, e.value)
            assert text is None or text in str(e.value), e.value


# ------------------------------------------------------------------ 1. the value table
@functools.lru_cache(None)
def str_crafted():
    """string values homed for every table size at once (a home under HOME_MASK is the home under each smaller mask):
    wrap: 24 values homed at the last slot; chain: 24 values sharing one home; empty: 8 values of 3, 8, 63 and 64 bytes homed
    where "" is; long: 8 values of 64 bytes that differ only in their last byte"""
    wrap = find_str(HOME_MASK, 24, b"w")
    chain = find_str(0x15555, 24, b"c")
    home0 = fnv_slot(b"", HOME_MASK)
    empty = _find_short(home0, 2, 3)
    for L in (8, 63, 64):
        empty += find_str(home0, 2, b"e" * (L - 8))
    long = [b"L" * 63 + bytes([x]) for x in (0, 1, 2, 0x41, 0x7f, 0x80, 0xfe, 0xff)]
    return dict(wrap=wrap, chain=chain, empty=empty, long=long)


def _find_short(slot, n, L):
    c = np.arange(1, 1 << (8 * L), dtype=np.uint64)
    cols = [((c >> np.uint64(8 * (L - 1 - k))) & np.uint64(0xff)).astype(np.uint8) for k in range(L)]
    hit = np.nonzero(_fnv_rows(_FNV0, cols, HOME_MASK) == slot)[0][:n]
    return [int(c[i]).to_bytes(L, "big") for i in hit.tolist()]


def str_table_values(cap):
    """cap - 1 distinct non-empty values (the crafted ones first) -- with nil / "" they are cap values"""
    cr = str_crafted()
    vals = cr["wrap"] + cr["chain"] + cr["empty"] + cr["long"]
    vals += [b"f%06d" % i for i in range(cap - 1 - len(vals))]
    return vals


@functools.lru_cache(None)
def i64_crafted():
    """int64 values homed for every table size: wrap (24 at the last slot), chains of 8 at the homes of -1, INT64_MIN and
    INT64_MAX, then those three"""
    special = [I64_MIN, I64_MAX, -1]
    wrap = find_i64(HOME_MASK, 24, HOME_MASK, exclude=special)
    chains = []
    for s in special:
        chains += find_i64(i64_slot(s, HOME_MASK), 8, HOME_MASK, start=1 << 24, exclude=special + wrap + chains)
    return dict(wrap=wrap, chain=chains, special=special)


def i64_table_values(cap):
    """cap - 1 distinct non-zero values (crafted first); with 0 / nil they are cap values"""
    cr = i64_crafted()
    vals = cr["wrap"] + cr["chain"] + cr["special"]
    seen = set(vals)
    i = 0
    while len(vals) < cap - 1:
        v = 1_000_003 * (i + 1) + 7
        i += 1
        if v not in seen:
            vals.append(v)
            seen.add(v)
    return vals


def _series(sid, cells, int64, fields=None, row0=0, tags=None):
    tg = {KT: int_tag(cells), KX: twin(cells)} if int64 else {KT: list(cells)}
    return Series(sid, fields or K.std_fields(sid, len(cells)), {**tg, **(tags or {})}, row0=row0)


EXTRA_SID = 9000


@functools.lru_cache(None)
def table_fixture(cap, int64):
    """-> (series, sids without the extra one).  The cap values (the table values plus nil and its "" / 0) spread over series
    of at most 202 values, each value in two series (1..3 rows per occurrence); at cap 65,536: 256 series of 256 values, one row
    each.  Series EXTRA_SID adds one more value next to some of the others: with it the query has cap + 1 values."""
    vals = i64_table_values(cap) if int64 else str_table_values(cap)
    zero = [None, 0] if int64 else [None, b""]
    ss = []
    if cap < 65536:
        n = -(-len(vals) // 100)
        for j in range(n):
            win = [vals[(j * 100 + i) % len(vals)] for i in range(200)] + (zero if j < 2 else [])
            ss.append(_series(j + 1, K._runs(win, 1), int64))
    else:
        vals = vals + [zero[0]]                   # 65,536 cells: nil the last
        for j in range(256):
            ss.append(_series(j + 1, vals[j * 256:(j + 1) * 256], int64))
    extra = [vals[5], (-12345 if int64 else b"zz-extra"), vals[7]]
    ss.append(_series(EXTRA_SID, extra, int64))
    return ss, [s.sid for s in ss if s.sid != EXTRA_SID]


def _table_case(bydb, gpu_ctx, cap, int64):
    ss, sids = table_fixture(cap, int64)
    gid = {s.sid: s.sid % 3 for s in ss}
    part = K.build_keyed(ss)
    E = bydb.capi
    kw = dict(key=KT, mkey=KX, vt=E.VT_INT64) if int64 else {}
    with Wide(bydb, gpu_ctx, [(part, ss)], gid, **kw) as w:
        got, q = w.query(sids, cap, aggs=AGGS4, oracle=cap <= ORACLE_MAX_CAP, ctx=f"table cap={cap} int64={int64}")
        assert got.n_keys == cap
        w.fails(E.ENOMEM, sids + [EXTRA_SID], cap)
        if cap < 65536:
            got, _ = w.query(sids + [EXTRA_SID], cap + 1, aggs=[("i", SUM), ("f", MIN)], oracle=cap <= ORACLE_MAX_CAP,
                             ctx=f"table cap+1={cap + 1}")
            assert got.n_keys == cap + 1
        else:
            w.fails(E.EINVAL, sids, cap + 1)
    return part, ss, sids, gid, q


@gpu
@pytest.mark.parametrize("cap", STR_CAPS)
def test_value_table_string_keys(bydb, gpu_ctx, cap):
    """string keys: S = pow2(max(2 cap, 1024)) slots; values at the last slot, a chain at one home, "" and nil behind a chain of
    3- to 64-byte values, 64-byte values differing in the last byte; V = cap answers, V = cap + 1 is BYDB_ENOMEM"""
    _table_case(bydb, gpu_ctx, cap, False)


@gpu
@pytest.mark.parametrize("cap", I64_CAPS)
def test_value_table_int64_keys(bydb, gpu_ctx, cap):
    """int64 keys: the same table edges, with INT64_MIN, INT64_MAX and -1 behind chains at their homes, and 0 / nil"""
    _table_case(bydb, gpu_ctx, cap, True)


# ------------------------------------------------------------------ 2. the block-local int64 table
@functools.lru_cache(None)
def local_values():
    """256 non-zero values homed at local slot 511 (the probes wrap to slot 0 and on)"""
    return find_i64(LOCAL_MASK, 256, LOCAL_MASK, exclude=[I64_MIN, I64_MAX, -1])


def _scatter(vals, reps, seed):
    cells = [v for v in vals for _ in range(reps)]
    rng = np.random.default_rng(seed)
    return [cells[i] for i in rng.permutation(len(cells)).tolist()]


@functools.lru_cache(None)
def local_series():
    """sid 1: the 256 values and 0 (257 in one block); sid 2: the 256 values; sid 3: 200 of them with INT64_MIN, INT64_MAX,
    -1, 0 and nil; rows scattered"""
    lv = local_values()
    return [_series(1, _scatter(lv + [0], 3, 1), True), _series(2, _scatter(lv, 3, 2), True),
            _series(3, _scatter(lv[:200] + [I64_MIN, I64_MAX, -1, 0, None], 2, 3), True)]


@gpu
def test_block_local_int64_table(bydb, gpu_ctx):
    ss = local_series()
    E = bydb.capi
    with Wide(bydb, gpu_ctx, [(K.build_keyed(ss), ss)], {1: 0, 2: 0, 3: 1}, key=KT, mkey=KX, vt=E.VT_INT64) as w:
        w.fails(E.ENOTSUP, [1], 1000, text="block")
        w.fails(E.ENOTSUP, [1, 2, 3], 1000, text="block")
        got, _ = w.query([2], 1000, aggs=K.AGGS, ctx="256 values at local slot 511")
        assert got.n_keys == 256
        got, _ = w.query([2, 3], 1000, aggs=K.AGGS, ctx="with the extremes, 0 and nil")
        assert got.n_keys == 260


# ------------------------------------------------------------------ 3. the record sort
SORT_POOL = 1000


def sort_keys(j, D):
    return [b"p%03d" % ((j * 131 + i) % SORT_POOL) for i in range(D)]


@functools.lru_cache(None)
def sort_series():
    """series 1..32: 256 distinct values each (every value twice, one block); 33: one value; 34: 255 values.  Tag z is "a" on
    the even values of the pool, "b" on the odd ones; tag u is "one" on a single row of series 5"""
    ss = []
    for sid, D in [(j, 256) for j in range(1, 33)] + [(33, 1), (34, 255)]:
        keys = sort_keys(sid, D)
        cells = keys + keys[::-1]
        z = [b"a" if int(c[1:]) % 2 == 0 else b"b" for c in cells]
        u = [b"one" if (sid == 5 and r == 10) else b"-" for r in range(len(cells))]
        ss.append(_series(sid, cells, False, tags={"z": z, "u": u}))
    return ss


SORT_SIDS = {1: [33], 2047: list(range(1, 8)) + [34], 2048: list(range(1, 9)), 2049: list(range(1, 9)) + [33],
             4096: list(range(1, 17)), 4097: list(range(1, 17)) + [33], 8193: list(range(1, 33)) + [33]}


@functools.lru_cache(None)
def sort_part():
    return K.build_keyed(sort_series())


def records_of(series, sids):
    """R: the distinct values of every selected block, summed"""
    sel = set(sids)
    return sum(len(set(K.key_cells(s, KT)[lo:hi])) for s in series if s.sid in sel for lo, hi in s.chunks())


@gpu
@pytest.mark.parametrize("R", list(SORT_SIDS))
def test_record_sort_sizes(bydb, gpu_ctx, R):
    ss = sort_series()
    P = O.Pred
    with Wide(bydb, gpu_ctx, [(sort_part(), ss)], {s.sid: s.sid % 3 for s in ss}) as w:
        sids = SORT_SIDS[R]
        got, _ = w.query(sids, 2000, ctx=f"R={R}")
        C = got.group_id.size
        w.query(sids, 2000, preds=[P(FAM, "z", O.OP_EQ, b"a")], ctx=f"R={R}, every other record empty")
        if R >= 4096:
            got, _ = w.query(sids, 2000, preds=[P(FAM, "u", O.OP_EQ, b"one")], ctx=f"R={R}, one record")
            assert got.group_id.size == 1
            got, _ = w.query(sids, 2000, preds=[P(FAM, "u", O.OP_EQ, b"none")], ctx=f"R={R}, no record")
            assert got.group_id.size == 0
            assert C > 2048
            for a, desc in ((1, True), (1, False), (0, True)):
                w.query(sids, 2000, top=(C // 2 + 3, a, desc), ctx=f"R={R}, top")


# ------------------------------------------------------------------ 4. records per composite
COMP_RECORDS = [1, 31, 32, 33, 64, 65, 1000]
LONG_BLOCKS = 3


def comp_fields(sid, n):
    """i: a narrow delta int64 page; f: a decimal float page; r: raw float cells with nulls"""
    r = np.arange(n, dtype=np.int64)
    i = 50 + sid + np.cumsum(((r * 13 + sid) % 41) - 20)
    f = np.round(((r * 37 + sid * 11) % 5000) / 100.0 - 20.0, 2)
    rf = np.sin(r * 0.7 + sid) * 1000.0 / 3.0
    return {"i": (I, i, None), "f": (F, f, None), "r": (F, rf, (r + sid) % 7 == 3)}


@functools.lru_cache(None)
def comp_series():
    """series group g holds COMP_RECORDS[g] records of the value "hot": short series [hot, u<sid>, hot, u<sid>] (each also a
    single-record composite of its own), and for 1,000 one series of LONG_BLOCKS blocks of "hot" and "cold" next to 997 short
    ones.  -> (series, gid)"""
    ss, gid, sid = [], {}, 1
    for g, N in enumerate(COMP_RECORDS):
        short = N - LONG_BLOCKS if N == 1000 else N
        for _ in range(short):
            cells = [b"hot", b"u%05d" % sid, b"hot", b"u%05d" % sid]
            ss.append(Series(sid, comp_fields(sid, 4), {KT: cells}))
            gid[sid] = g
            sid += 1
        if N == 1000:
            n = LONG_BLOCKS * BLOCK
            cells = [b"cold" if r % 5 == 2 else b"hot" for r in range(n)]
            ss.append(Series(sid, comp_fields(sid, n), {KT: cells}))
            gid[sid] = g
            sid += 1
    return ss, gid


@functools.lru_cache(None)
def comp_part():
    return K.build_keyed(comp_series()[0])


COMP_AGGS = [(f, fn) for f in ("i", "f", "r") for fn in (SUM, COUNT, MIN, MAX, MEAN)]


@gpu
def test_records_per_composite(bydb, gpu_ctx):
    ss, gid = comp_series()
    with Wide(bydb, gpu_ctx, [(comp_part(), ss)], gid) as w:
        sids = [s.sid for s in ss]
        got, _ = w.query(sids, 4000, aggs=COMP_AGGS, ctx="records per composite")
        hot = {g: r for g, k, r in zip(got.group_id.tolist(), got.key, got.rows.tolist()) if k == b"hot"}
        assert sorted(hot) == list(range(len(COMP_RECORDS)))
        w.query(sids, 4000, aggs=COMP_AGGS, tmin=T0 + 1 * STEP, tmax=T0 + (2 * BLOCK + 5) * STEP, ctx="records per composite, cut")


# ------------------------------------------------------------------ 5. many parts
PART_ROWS = 40


@functools.lru_cache(None)
def parts_series(n_parts):
    """n_parts time-disjoint parts of PART_ROWS rows per series: series s (1..8) is in part p unless (5 s + p) % 4 == 0, and its
    values there depend on p (so the first value a series shows depends on the parts' time order); every 11th part holds only
    series 99, which no query selects.  -> [(part, series)]"""
    out = []
    for p in range(n_parts):
        ss = []
        for sid in ([99] if p % 11 == 7 else [s for s in range(1, 9) if (5 * s + p) % 4]):
            cells = [b"v%02d" % ((p * 3 + sid + i // 10) % 37) for i in range(PART_ROWS)]
            ss.append(Series(sid, K.std_fields(sid + p, PART_ROWS), {KT: cells}, row0=p * PART_ROWS))
        out.append((K.build_keyed(ss), ss))
    return out


def shuffled(n, seed):
    return np.random.default_rng(seed).permutation(n).tolist()


@gpu
@pytest.mark.parametrize("n_parts", [33, 64])
def test_many_parts(bydb, gpu_ctx, n_parts):
    ps = parts_series(n_parts)
    gid = {s: s % 3 for s in list(range(1, 9)) + [99]}
    with Wide(bydb, gpu_ctx, ps, gid) as w:
        sids = list(range(1, 9))
        for seed in (1, 2):
            order = shuffled(n_parts, seed)
            w.query(sids, 100, aggs=K.AGGS, order=order, ctx=f"{n_parts} parts, order {order[:6]}")
            w.query(sids, 100, order=order, tmin=T0 + 5 * PART_ROWS * STEP + 7, tmax=T0 + (n_parts - 3) * PART_ROWS * STEP,
                    ctx=f"{n_parts} parts, a range that selects nothing of some")
            w.query([1, 4, 7], 100, order=order, top=(5, 1, True), ctx=f"{n_parts} parts, top")
    if n_parts == 64:
        extra = K.build_keyed([Series(1, K.std_fields(1, 5), {KT: [b"x"] * 5}, row0=64 * PART_ROWS)])
        with Wide(bydb, gpu_ctx, ps + [(extra, [])], gid) as w:
            w.fails(bydb.capi.EINVAL, [1, 2], 100)


# ------------------------------------------------------------------ 6. exact sums
BIG = 1 << 62
DEC_BIG = 461168601842738.7   # 16 digits: mantissa 4611686018427387000 ~ 2^62 at the page exponent -4 that 0.0001 sets


@functools.lru_cache(None)
def sums_series():
    """sid 1 and 4 (one series group): 8,192 rows of "pos" / "neg" / "mix" runs, int64 values near +-2^62 (every block and
    composite sum leaves the int64 range), decimal mantissas near +-2^62 (0.0001 on the "tiny" row sets the exponent);
    sid 2: the int64 extremes; sid 3: 8,193 rows, the key "a", then "b" at row 8191 and "c" at row 8192; sid 5: 0.1, 0.2, -0.3"""
    n = 8192
    r = np.arange(n, dtype=np.int64)
    out = []
    for sid in (1, 4):
        kind = (r // (7 + sid)) % 3
        sign = np.where(kind == 0, 1, np.where(kind == 1, -1, np.where(r % 2 == 0, 1, -1)))
        iv = sign * (BIG + (r % 1000) * 3 + sid)
        fv = sign * (DEC_BIG - (r % 100))
        keys = [(b"pos", b"neg", b"mix")[k] for k in kind.tolist()]
        fv[100 + sid] = 0.0001
        keys[100 + sid] = b"tiny"
        out.append(Series(sid, {"i": (I, iv, None), "f": (F, fv, None)}, {KT: keys}))
    ext = np.array([I64_MIN, I64_MAX, -1, 0, 1, I64_MIN + 1, I64_MAX - 1] * 10, np.int64)
    out.append(Series(2, {"i": (I, ext, None), "f": (F, np.round(ext / 7.0e12, 3), None)},
                      {KT: [b"ext" if x % 3 else b"ext2" for x in range(ext.size)]}))
    m = BLOCK
    keys = [b"a"] * (m - 2) + [b"b", b"c"]
    rr = np.arange(m, dtype=np.int64)
    out.append(Series(3, {"i": (I, rr * 1000 - 7, None), "f": (F, np.round(rr / 8.0 + 0.125, 3), None)}, {KT: keys}))
    out.append(Series(5, {"i": (I, np.array([1, 2, 3]), None), "f": (F, np.array([0.1, 0.2, -0.3]), None)}, {KT: [b"cancel"] * 3}))
    return out


@gpu
def test_exact_sums(bydb, gpu_ctx):
    ss = sums_series()
    gid = {1: 0, 4: 0, 2: 1, 3: 2, 5: 3}
    aggs = [(f, fn) for f in ("i", "f") for fn in (SUM, COUNT, MIN, MAX, MEAN)]
    with Wide(bydb, gpu_ctx, [(K.build_keyed(ss), ss)], gid) as w:
        got, q = w.query([1, 2, 3, 4, 5], 100, aggs=aggs, ctx="exact sums")
        rows = {(g, k): i for i, (g, k) in enumerate(zip(got.group_id.tolist(), got.key))}
        # the composite whose values cancel: the exact decimal sum is 0, the reference's double sum 5.55e-17, so no bound
        # relative to the reference holds there; float_close (1e-9 x sum |x|) does
        fs = aggs.index(("f", SUM))
        c = rows[(3, b"cancel")]
        assert got.val_f64[c, fs] == 0.0, got.val_f64[c, fs]
        want = O.run_query(dataclasses.replace(w.oquery([5], aggs)[0], group_key=(FAM, KT)))
        assert want.val_f64[0, fs] == (0.1 + 0.2) + -0.3 != 0.0
        assert abs(got.val_f64[c, fs] - want.val_f64[0, fs]) > 1e-9 * abs(want.val_f64[0, fs])
        assert float_close(got.val_f64[c, fs], want.val_f64[0, fs], np.array([0.1, 0.2, -0.3]), SUM)
        # the per-value passes and the express lane sum the decimal page the same way
        _, q5 = w.oquery([5], [("f", SUM)])
        assert gpu_ctx.scan_agg_keyed(q5, FAM, KT, 4).val_f64[0, 0] == 0.0
        plain = gpu_ctx.scan_agg(q5)
        assert plain.val_f64[0, 0] == 0.0 and plain.stats.blocks_express_lane == 1, (plain.val_f64, plain.stats)
        # the 8,193-row block: one row each for "b" and "c"
        assert got.rows[rows[(2, b"b")]] == 1 and got.rows[rows[(2, b"c")]] == 1 and got.rows[rows[(2, b"a")]] == BLOCK - 2
        w.query([3], 100, aggs=aggs, tmin=T0 + (BLOCK - 2) * STEP, ctx="exact sums, the last two rows")
        w.query([1, 4], 100, aggs=aggs, preds=[O.Pred(FAM, KT, O.OP_NE, b"mix")], ctx="exact sums, a predicate on the key")


# ------------------------------------------------------------------ 7. the prepared form and the collective
@gpu
def test_prepared_over_the_boundaries(bydb, gpu_ctx):
    """items 1, 3, 4 and 5 through prepare_keyed_wide: three executions in each form, each equal to the unprepared call bit for
    bit, the replays' counters as the header states"""
    from tests.test_gpu_keyed_wide_prepared import run_handle
    E = bydb.capi
    for cap, int64 in ((1024, False), (65536, False), (1025, True)):
        ss, sids = table_fixture(cap, int64)
        with Wide(bydb, gpu_ctx, [(K.build_keyed(ss), ss)], {s.sid: s.sid % 3 for s in ss}) as w:
            _, q = w.oquery(sids, AGGS4)
            fin, _ = run_handle(bydb, gpu_ctx, q, max_values=cap, vt=E.VT_INT64 if int64 else 0, what=f"table {cap}", runs=3)
            assert fin[-1].n_keys == cap
    ss = sort_series()
    with Wide(bydb, gpu_ctx, [(sort_part(), ss)], {s.sid: s.sid % 3 for s in ss}) as w:
        for R in (2048, 2049, 8193):
            _, q = w.oquery(SORT_SIDS[R], AGGS4)
            run_handle(bydb, gpu_ctx, q, max_values=2000, what=f"R={R}", runs=3)
            _, q = w.oquery(SORT_SIDS[R], AGGS4, preds=[O.Pred(FAM, "z", O.OP_EQ, b"a")])
            run_handle(bydb, gpu_ctx, q, max_values=2000, what=f"R={R}, half empty", runs=3)
    ss, gid = comp_series()
    with Wide(bydb, gpu_ctx, [(comp_part(), ss)], gid) as w:
        _, q = w.oquery([s.sid for s in ss], COMP_AGGS)
        run_handle(bydb, gpu_ctx, q, max_values=4000, what="records per composite", runs=3)
    ps = parts_series(33)
    with Wide(bydb, gpu_ctx, ps, {s: s % 3 for s in list(range(1, 9)) + [99]}) as w:
        _, q = w.oquery(range(1, 9), K.AGGS, order=shuffled(33, 1))
        run_handle(bydb, gpu_ctx, q, max_values=100, what="33 parts", runs=3)


def table_case_ranks(cap):
    """the string table fixture at `cap` as series shards: series j on rank j % 3"""
    ss, sids = table_fixture(cap, False)
    pieces = [(j % N_RANKS, s.sid, s.tags[KT], 0) for j, s in enumerate(ss) if s.sid != EXTRA_SID]
    return split(pieces, {s.sid: s.sid % 3 for s in ss if s.sid != EXTRA_SID})


def parts_case_ranks(n_parts=33):
    """the many-parts fixture: rank r holds a third of the parts in time order, and passes them shuffled"""
    ps = parts_series(n_parts)
    third = -(-n_parts // N_RANKS)
    shards = []
    for r in range(N_RANKS):
        mine = [p for p, _ in ps[r * third:(r + 1) * third]]
        shards.append([mine[i] for i in shuffled(len(mine), r)])
    return Case(shards, [p for p, _ in ps], {s: s % 3 for s in list(range(1, 9))})


@gpu
def test_collective_over_the_boundaries(bydb, gpu_ctx, quiet):  # noqa: F811
    """the value table at S = 2,048 and 131,072 and 33 parts over 3 ranks through scan_reduce_keyed_wide / _partials: the root's
    union table (homed by key_home) and its composite table at the same edges"""
    for cap in (1024, 65536):
        case = table_case_ranks(cap)
        ranks = Ranks(bydb, wide_slot(bydb, case, cap, cap * 2), case.shards)
        try:
            for root in (0, 2):
                got = check(bydb, gpu_ctx, ranks, case, root, max_values=cap, oracle=cap <= ORACLE_MAX_CAP, label=f"table {cap}")
                assert got.n_keys == cap
            check(bydb, gpu_ctx, ranks, case, 1, max_values=cap, partial=True, label=f"table {cap} partial")
        finally:
            ranks.close()
    case = parts_case_ranks()
    ranks = Ranks(bydb, wide_slot(bydb, case, 100, 400), case.shards)
    try:
        for root in (0, 1, 2):
            check(bydb, gpu_ctx, ranks, case, root, max_values=100, label="33 parts")
        check(bydb, gpu_ctx, ranks, case, 2, max_values=100, partial=True, label="33 parts partial")
        check(bydb, gpu_ctx, ranks, case, 0, max_values=100, label="33 parts top", aggs=[("i", COUNT), ("f", SUM)], top=(5, 0, False))
    finally:
        ranks.close()


# ------------------------------------------------------------------ the layout claims above, on the CPU
def test_wide_case_layouts():
    """Every crafted set lands where the GPU tests claim, and the fixtures read back through the oracle's codecs."""
    cr = str_crafted()
    sizes = sorted({table_slots(c) for c in STR_CAPS + I64_CAPS})
    assert sizes == [1024, 2048, 4096, 131072]
    home0 = {S: fnv_slot(b"", S - 1) for S in sizes}
    for S in sizes:
        assert {fnv_slot(v, S - 1) for v in cr["wrap"]} == {S - 1}, S
        assert len({fnv_slot(v, S - 1) for v in cr["chain"]}) == 1, S
        assert {fnv_slot(v, S - 1) for v in cr["empty"]} == {home0[S]}, S
        assert {i64_slot(v, S - 1) for v in i64_crafted()["wrap"]} == {S - 1}, S
        for k, s in enumerate(i64_crafted()["special"]):
            assert {i64_slot(v, S - 1) for v in i64_crafted()["chain"][8 * k:8 * k + 8]} == {i64_slot(s, S - 1)}, S
    assert sorted(len(v) for v in cr["empty"]) == [3, 3, 8, 8, 63, 63, 64, 64]
    assert len(set(cr["long"])) == 8 and {len(v) for v in cr["long"]} == {64} and len({v[:63] for v in cr["long"]}) == 1
    # the table fixtures: cap values without the extra series, cap + 1 with it, at most 256 per block, dictionary pages
    for cap in STR_CAPS + I64_CAPS:
        for int64 in ((False, True) if cap in I64_CAPS else (False,)):
            if int64 and cap not in I64_CAPS:
                continue
            ss, sids = table_fixture(cap, int64)
            key = KX if int64 else KT
            vals = {c for s in ss if s.sid in sids for c in K.key_cells(s, key)}
            assert len(vals) == cap and len(vals | set(K.key_cells(ss[-1], key))) == cap + 1, (cap, int64)
            assert (le(0) if int64 else b"") in vals
            assert all(len(set(K.key_cells(s, key)[lo:hi])) <= 256 for s in ss for lo, hi in s.chunks())
            if not int64 and cap in (511, 65536):
                assert all(str_tag_class(s.tags[KT]) == "dict" for s in ss[:3] + ss[-3:])
            if cap == 65536:   # load 1/2 of the largest table
                assert table_slots(cap) == 2 * len(vals)
    assert set(i64_crafted()["special"]) <= set(i64_table_values(512))
    # the block-local table
    lv = local_values()
    assert len(set(lv)) == 256 and {i64_slot(v, LOCAL_MASK) for v in lv} == {LOCAL_MASK} and 0 not in lv
    ls = local_series()
    assert [len(set(K.key_cells(s, KX))) for s in ls] == [257, 256, 204]
    assert ls[0].tags[KT][0].tolist() != sorted(ls[0].tags[KT][0].tolist())
    # the record sort: R per query, C > 2048 where Top-N runs, every other record emptied by z == "a"
    ss = sort_series()
    for R, sids in SORT_SIDS.items():
        assert records_of(ss, sids) == R, (R, records_of(ss, sids))
        comps = {(s.sid % 3, c) for s in ss if s.sid in sids for c in s.tags[KT]}
        if R >= 4096:
            assert len(comps) > 2048, (R, len(comps))
    z_a = sum(len({c for c, z in zip(s.tags[KT], s.tags["z"]) if z == b"a"}) for s in ss if s.sid in SORT_SIDS[8193])
    assert 0.4 * 8193 < z_a < 0.6 * 8193
    # records per composite: (group, "hot") has COMP_RECORDS[g] records; the long series spans LONG_BLOCKS blocks
    cs, gid = comp_series()
    recs = {}
    for s in cs:
        for lo, hi in s.chunks():
            for v in set(s.tags[KT][lo:hi]):
                recs[(gid[s.sid], v)] = recs.get((gid[s.sid], v), 0) + 1
    assert [recs[(g, b"hot")] for g in range(len(COMP_RECORDS))] == COMP_RECORDS
    assert max(len(s.chunks()) for s in cs) == LONG_BLOCKS
    kinds = {f: {s.kind(("f", f), lo, hi) for s in cs for lo, hi in s.chunks()} for f in ("i", "f", "r")}
    assert kinds["i"] == {("delta", False)} and ("raw", True) in kinds["r"] and all(k[0] != "raw" for k in kinds["f"])
    # many parts: time-disjoint, some parts select nothing, each series in a subset of them
    for n in (33, 64):
        ps = parts_series(n)
        spans = [(min(int(s.ts[0]) for s in ss), max(int(s.ts[-1]) for s in ss)) for _, ss in ps]
        assert all(a[1] < b[0] for a, b in zip(spans, spans[1:]))
        assert sum(all(s.sid == 99 for s in ss) for _, ss in ps) == len([p for p in range(n) if p % 11 == 7])
        for sid in range(1, 9):
            assert 0 < sum(any(s.sid == sid for s in ss) for _, ss in ps) < n
    # exact sums: decimal mantissas near +-2^62 at exponent -4; int64 sums out of range
    ss = sums_series()
    m, e = O.float64_to_decimal_list(ss[0].fields["f"][1])
    assert e == -4 and BIG // 2 < max(abs(int(x)) for x in m) < 1 << 63
    for s in (ss[0], ss[1]):
        pos = [int(v) for v, k in zip(s.fields["i"][1].tolist(), s.tags[KT]) if k == b"pos"]
        assert sum(pos) > I64_MAX and len(s.chunks()) == 1
    s3 = next(s for s in ss if s.sid == 3)
    assert s3.n == BLOCK and s3.chunks() == [(0, BLOCK)] and s3.tags[KT].index(b"b") == 8191 and s3.tags[KT].index(b"c") == 8192
    # the oracle's reading of the fixtures: key_model and the oracle agree on the composites, rows and int64 values
    for series, gidm, sids, aggs, key in ((ls[1:], {2: 0, 3: 1}, [2, 3], [("i", SUM), ("i", COUNT)], KX),
                                           (cs, gid, [s.sid for s in cs], [("i", SUM), ("r", COUNT), ("f", MAX)], KT),
                                           (ss, {1: 0, 4: 0, 2: 1, 3: 2, 5: 3}, [1, 2, 3, 4, 5], [("i", SUM), ("i", MIN), ("f", MAX)], KT)):
        part = K.build_keyed(series)
        sids = np.array(sorted(sids), np.uint64)
        oq = O.Query([part], sids, aggs, groups=np.array([gidm[int(s)] for s in sids], np.int32), n_groups=max(gidm.values()) + 1,
                     group_key=(FAM, key))
        want = O.run_query(oq)
        exp = K.key_model(series, gidm, sids, aggs, [], I64_MIN, I64_MAX, key, None)
        assert list(zip(want.group_id.tolist(), want.key)) == [e_[0] for e_ in exp]
        assert want.rows.tolist() == [e_[1] for e_ in exp]
        assert want.val_i64[:, 0].tolist() == [e_[2][0][0] for e_ in exp]
    # the cancelling composite: the reference adds the page's doubles in row order, so its sum is not the exact 0
    m, e = O.float64_to_decimal_list(np.array([0.1, 0.2, -0.3]))
    assert list(m) == [1, 2, -3] and e == -1
    cancel = [s for s in ss if s.sid == 5]
    oq = O.Query([K.build_keyed(cancel)], np.array([5], np.uint64), [("f", SUM)], groups=np.zeros(1, np.int32), n_groups=1,
                 group_key=(FAM, KT))
    assert O.run_query(oq).val_f64[0, 0] == (0.1 + 0.2) + -0.3 == 5.551115123125783e-17

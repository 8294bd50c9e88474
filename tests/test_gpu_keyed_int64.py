"""Group-by on a stored int64 tag (bydb_scan_agg_keyed with value_type BYDB_VT_INT64, DESIGN.md 4.6) against the oracle and an
independent model, at its boundaries; and the operator (scan_operator.py) routing a stored-tag GroupBy key to that call.

The reference keys a row by the 8 little-endian bytes of the int64 cell (groupby.go:226-254), and a nil cell reaches the key as
the column's zero value (typed_column.go:49-53): nil and 0 are one key.  key_values_i64_kernel enters every value of the
selected blocks' int64 pages (Const, DeltaConst, Delta / DoD through decode_varint_page, raw cells) into a 1024-slot table
(0 = empty slot, the value 0 in a flag word of its own); one scan pass per value v follows with the predicate "tag == v"
(kOpEqOrNil for 0), then the insertion order and the finalisation of the string key.

Every part carries, next to the int64 key tag `k`, a string twin `kx` whose cell is the 8 little-endian bytes of `k` with nil
taken as 0 -- the reference's key bytes, written out by a plain Python fold.  The oracle groups by the twin (its own int64 key
stays refused, tests/test_oracle_query.py), and `key_model` of test_gpu_keyed.py folds over it.  Each query is checked
  - against the oracle keyed on the twin: groups, rows, aggregates and the per-row key bytes;
  - without Top-N, against the oracle's own reading of the int64 column, independent of the twin (`oracle_per_value`): each
    non-zero key equals a plain oracle query with `k == v`, the key 0 holds rows(`k == 0`) plus the nil rows;
  - against key_model: composite groups in first-seen order with the keys decoded from 8 little-endian bytes, rows and folds;
  - on key discovery and the counters: n_keys = distinct values (nil -> 0) over all rows of the selected blocks; rows_matched;
    rows_scanned / blocks_scanned = V passes; no express-lane block; and the slow lane: the key tag's own DoD, wide-delta or
    raw-cell page defers its block (reason 2) in every pass with a row in range, as does a deferring user predicate; otherwise
    a deferring field page defers only the passes whose value survives in the block (test_gpu_keyed.lane_model's rule).
"""
import dataclasses
import functools
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity
from tests.test_gpu_fallback import BLOCK, COUNT, MAX, MEAN, MIN, SUM, Series
from tests.test_gpu_keyed import (AGGS, DEFER_TAG, FAM, KScan, build_keyed, fnv_slot, key_cells, key_model, row_mask,
                                  selected_blocks, std_fields)
from tests.test_gpu_lanes import LIMIT_DELTAS
from tests.test_gpu_masks import I64_MAX, I64_MIN, INT_CLASS, INT_KINDS, int_tag_values, wrap64

gpu = pytest.mark.gpu

KT, KX = "k", "kx"          # the int64 key tag and its string twin (the reference's key bytes)
SIZES = [1, 31, 32, 33, 8192, 8193]
_pid = [160_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def le(v):
    return struct.pack("<q", v)


def unle(b):
    assert len(b) == 8, b
    return struct.unpack("<q", b)[0]


def twin(cells):
    """the key bytes of each cell: nil -> 0 (typed_column.go:49-53), then 8 bytes little-endian (groupby.go:226-254)"""
    return [le(0 if c is None else c) for c in cells]


def int_tag(cells):
    return (np.array([0 if c is None else c for c in cells], np.int64), np.array([c is None for c in cells]))


def mk64(sid, cells, row0=0, tags=None):
    """a series whose int64 key tag holds `cells` (None = nil), with the twin and the other tags given"""
    return Series(sid, std_fields(sid, len(cells)), {KT: int_tag(cells), KX: twin(cells), **(tags or {})}, row0=row0)


def mk_absent(sid, n, row0=0, tags=None):
    """a series of a part without the key column: every cell is nil, so the key is 0"""
    return Series(sid, std_fields(sid, n), {KX: [le(0)] * n, **(tags or {})}, row0=row0)


def lane_model64(series, sids, aggs, preds, tmin, tmax, values):
    """(blocks_slow_lane, slow_lane_reasons) summed over the V passes; the key predicate of every pass is on KT"""
    fields = list(dict.fromkeys(f for f, _ in aggs))
    need = dict.fromkeys(fields, 0)
    for f, fn in aggs:
        need[f] |= 1 if fn in (SUM, MEAN) else 2 if fn in (MIN, MAX) else 0
    slow = reasons = 0
    for s, lo, hi in selected_blocks(series, sids, tmin, tmax):
        if not ((s.ts[lo:hi] >= tmin) & (s.ts[lo:hi] <= tmax)).any():
            continue
        if any(t in s.tags and s.kind(("t", t), lo, hi)[0] in DEFER_TAG for t in [KT] + [p.tag for p in preds]):
            slow += len(values)
            reasons |= 2
            continue
        why = next((4 << c for c, f in enumerate(fields) for k, nl in [s.kind(("f", f), lo, hi)]
                    if (k == "raw" and (need[f] or nl)) or (k == "wide" and need[f])), 0)
        if why:
            keys = key_cells(s, KX)
            m = row_mask(s, preds, tmin, tmax)
            live = {keys[r] for r in range(lo, hi) if m[r]}
            slow += len(live & set(values))
            reasons |= why if live else 0
    return slow, reasons


def _by_group(r):
    return {g: i for i, g in enumerate(r.group_id.tolist())}


def oracle_per_value(oq, preds, got, aggs, ctx):
    """The keyed answer against the oracle's OWN reading of the int64 column, independent of the twin: for every non-zero key
    v, each group's row equals a plain oracle query with the extra int64 predicate `k == v`; for the key 0, each group's rows
    equal rows(k == 0) + nil rows, the nil rows being rows(k != 0) (nil passes NE) minus the rows of every non-zero key."""
    keys = [unle(k) for k in got.key]
    gid = got.group_id.tolist()
    plain = lambda extra: O.run_query(dataclasses.replace(oq, preds=list(preds) + [extra]))   # noqa: E731
    nonzero = {}
    for v in sorted(set(keys) - {0}):
        w = plain(O.Pred(FAM, KT, O.OP_EQ, v))
        wg = _by_group(w)
        mine = {gid[i]: i for i, k in enumerate(keys) if k == v}
        assert sorted(mine) == sorted(wg), f"{ctx}: key {v}: groups {sorted(mine)} vs oracle k == v {sorted(wg)}"
        for g, i in mine.items():
            j = wg[g]
            assert int(got.rows[i]) == int(w.rows[j]), f"{ctx}: key {v} group {g}: rows {got.rows[i]} vs {w.rows[j]}"
            for a, (_, fn) in enumerate(aggs):
                if not got.is_float[a]:
                    assert int(got.val_i64[i, a]) == int(w.val_i64[j, a]), f"{ctx}: key {v} group {g} agg {a}"
                elif fn in (MIN, MAX):
                    assert got.val_f64[i:i + 1, a].view(np.uint64)[0] == w.val_f64[j:j + 1, a].view(np.uint64)[0], f"{ctx}: key {v} agg {a}"
                else:
                    assert abs(float(got.val_f64[i, a]) - float(w.val_f64[j, a])) <= 1e-9 * max(abs(float(w.val_f64[j, a])), 1e-300), \
                        f"{ctx}: key {v} group {g} agg {a}"
        for g, j in wg.items():
            nonzero[g] = nonzero.get(g, 0) + int(w.rows[j])
    eq0, ne0 = plain(O.Pred(FAM, KT, O.OP_EQ, 0)), plain(O.Pred(FAM, KT, O.OP_NE, 0))
    want0 = {g: 0 for g in set(gid) | set(eq0.group_id.tolist()) | set(ne0.group_id.tolist())}
    for r, sign in ((eq0, 1), (ne0, 1)):
        for g, j in _by_group(r).items():
            want0[g] += sign * int(r.rows[j])
    for g, n in nonzero.items():
        want0[g] -= n
    got0 = {gid[i]: int(got.rows[i]) for i, k in enumerate(keys) if k == 0}
    assert {g: n for g, n in want0.items() if n} == got0, f"{ctx}: key 0 rows {got0} vs oracle k == 0 plus nil rows {want0}"


class KScan64(KScan):
    """KScan with the device keyed on the int64 tag, the oracle / model keyed on its twin, and (without Top-N) the oracle's
    own int64 predicates per key value."""

    def query(self, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, sids=None, max_values=256, order=None, ctx=""):
        preds = list(preds)
        oq, q = self.oquery(aggs, preds, tmin, tmax, top, sids, order)
        ctx = f"{ctx}/{[(f, fn) for f, fn in aggs]}/{[(p.tag, p.op, p.value) for p in preds]}" \
              f"/{(tmin - T0) // STEP if tmin > I64_MIN else '-'}..{(tmax - T0) // STEP if tmax < I64_MAX else '-'}/top{top}"
        got = self.ctx.scan_agg_keyed(q, FAM, KT, max_values, self.bydb.capi.VT_INT64)
        want = O.run_query(dataclasses.replace(oq, group_key=(FAM, KX)))
        assert_parity(got, want, aggs, ctx)
        assert got.key == want.key, f"{ctx}: keys {got.key[:8]} vs oracle {want.key[:8]}"
        if top is None:
            oracle_per_value(oq, preds, got, aggs, ctx)
        exp = key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, KX, top)
        got_comp = [(g, unle(k)) for g, k in zip(got.group_id.tolist(), got.key)]
        want_comp = [(g, unle(k)) for (g, k), _, _ in exp]
        assert got_comp == want_comp, f"{ctx}: composite groups {got_comp[:8]}, model {want_comp[:8]}"
        assert got.rows.tolist() == [e[1] for e in exp], f"{ctx}: rows vs model"
        for i, (ck, _, vals) in enumerate(exp):
            for a, ((f, fn), (m, x)) in enumerate(zip(aggs, vals)):
                where = f"{ctx}: group {ck} agg {a} ({f},{fn})"
                if not got.is_float[a]:
                    assert int(got.val_i64[i, a]) == m, f"{where}: {got.val_i64[i, a]}, model {m}"
                elif fn in (MIN, MAX):
                    assert got.val_f64[i:i + 1, a].view(np.uint64)[0] == np.array([m]).view(np.uint64)[0], f"{where}: bit-exact"
                else:
                    tol = 1e-9 * float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1)
                    assert abs(float(got.val_f64[i, a]) - m) <= tol, f"{where}: {got.val_f64[i, a]!r}, model {m!r}"
        blocks = selected_blocks(self.series, oq.sids, tmin, tmax)
        values = {c for s, lo, hi in blocks for c in key_cells(s, KX)[lo:hi]}
        V = len(values)
        st = got.stats
        assert got.n_keys == V and set(want.key) <= values, f"{ctx}: n_keys {got.n_keys}, {V} values in the selected blocks"
        rows = sum(e[1] for e in key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, KX, None))
        assert st.rows_matched == rows, f"{ctx}: rows_matched {st.rows_matched}, model {rows}"
        assert st.rows_scanned == V * sum(hi - lo for _, lo, hi in blocks), f"{ctx}: rows_scanned {st.rows_scanned}"
        assert st.blocks_scanned == V * len(blocks), f"{ctx}: blocks_scanned {st.blocks_scanned}, {V} x {len(blocks)}"
        assert st.blocks_express_lane == 0, f"{ctx}: express-lane blocks {st.blocks_express_lane}"
        lanes = lane_model64(self.series, oq.sids, aggs, preds, tmin, tmax, values)
        assert (st.blocks_slow_lane, st.slow_lane_reasons) == lanes, \
            f"{ctx}: (slow blocks, reasons) {(st.blocks_slow_lane, st.slow_lane_reasons)}, model {lanes}"
        return got

    def fails(self, code, preds=(), sids=None, key=KT, max_values=256, value_type=None, order=None):
        """the keyed call fails with `code`; afterwards the context still answers a plain query"""
        vt = self.bydb.capi.VT_INT64 if value_type is None else value_type
        _, q = self.oquery(AGGS, list(preds), I64_MIN, I64_MAX, None, sids, order)
        with pytest.raises(self.bydb.BydbError) as e:
            self.ctx.scan_agg_keyed(q, FAM, key, max_values, vt)
        assert e.value.code == code, (code, e.value)
        oq, q = self.oquery(AGGS, [], I64_MIN, I64_MAX, None, self.usid[:1], None if order is None else order[:1])
        assert_parity(self.ctx.scan_agg(q), O.run_query(oq), AGGS, "plain query after a keyed error")


# ------------------------------------------------------------------ every int64 page kind as the key page
def key_block(kind, n, rng):
    """int64 key cells of one block of `kind` (test_gpu_masks.INT_KINDS) with at most 64 distinct values: the masks'
    generator up to 33 rows; longer blocks repeat a short run forwards and backwards (same varint widths), DeltaConst takes
    a step of 2^62 / 2^63 (4 / 2 values mod 2^64), DoD climbs in steps every 199 rows, `limits` cycles the zig-zag limits."""
    if n <= 33 or kind in ("const", "wrap"):
        return int_tag_values(kind, n, rng)
    if kind == "dc_neg":
        return [wrap64(1000 - (1 << 62) * r) for r in range(n)]
    if kind == "dc_wrap":
        return [wrap64(I64_MAX - 100 + (1 << 63) * r) for r in range(n)]
    if kind == "dod":
        steps = np.where(np.arange(n - 1) % 199 == 0, rng.integers(1, 100, n - 1), 0)
        return (5000 + np.concatenate([[0], np.cumsum(steps)])).astype(np.int64).tolist()
    if kind == "limits":   # the limits, then two 3-byte steps back to the start: a period of 13 values
        d = np.resize(np.array(LIMIT_DELTAS + [(1 << 20) - 1, 5], dtype=np.int64), n - 1)
        return (500 + np.concatenate([[0], np.cumsum(d)])).astype(np.int64).tolist()
    base = int_tag_values("d1" if kind == "raw" else kind, 32, rng)
    v = ((base + base[::-1]) * (n // 64 + 1))[:n]
    if kind == "raw":      # nil at rows 0, 31, 32 and the last one, a 0 right after the nil of row 32
        for r in (0, 31, 32, n - 1):
            v[r] = None
        v[33] = 0
    return v


def kind_series(kind):
    rng = np.random.default_rng(0x64E0 + INT_KINDS.index(kind))
    return [mk64(1 + j, key_block(kind, n, rng)) for j, n in enumerate(SIZES)]


@gpu
@pytest.mark.parametrize("kind", INT_KINDS)
def test_int64_key_page_kinds(bydb, gpu_ctx, kind):
    """Every int64 tag page kind as the key page, blocks of 1, 31, 32, 33, 8192 and 8193 rows: Const, DeltaConst (negative,
    wrapping, 2^62 / 2^63 steps), narrow and wide Delta, zig-zag limits, a running value that wraps at every row, DoD and raw
    cells with nulls; over every row, behind a time cut at row 31, with a Top-1 over COUNT."""
    ss = kind_series(kind)
    with KScan64(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={s.sid: s.sid % 2 for s in ss}) as k:
        k.query(ctx=kind)
        k.query(aggs=[("i", SUM), ("i", COUNT), ("f", MAX)], tmin=T0 + 31 * STEP, ctx=kind)
        k.query(aggs=[("i", COUNT), ("f", SUM)], top=(1, 0, True), ctx=kind)


# ------------------------------------------------------------------ values: the int64 limits, the empty slot, the hash
@functools.lru_cache(None)
def wrap_values():
    """40 int64 values whose 8 key bytes home at slot 1023 (probes wrap to slot 0)"""
    out, i = [], 1
    while len(out) < 40:
        if fnv_slot(le(i)) == 1023:
            out.append(i)
        i += 1
    return out


TOP_BYTE = [5, (1 << 56) | 5, (2 << 56) | 5, (0x7f << 56) | 5, -(1 << 56) + 5, wrap64((0x80 << 56) | 5)]
SPECIAL = [I64_MIN, I64_MAX, -1, 0, 1, I64_MIN + 1, I64_MAX - 1] + TOP_BYTE


def value_parts():
    """part 1: raw cells with nulls next to every special value, the 40 wrapping values in a delta page, the specials again in
    another order; part 2 (later in time) has no key column: its rows key to 0"""
    sp = SPECIAL
    wv = wrap_values()
    cells = {60: [x for v in sp for x in (None, v, v)] + [0, None], 61: [x for v in wv for x in (v, v)] + wv[::-3],
             62: sp[::-1] * 3 + wv[:5]}
    tags = lambda n: {"c": (np.arange(n, dtype=np.int64) % 5, np.zeros(n, bool))}   # noqa: E731
    p1 = [mk64(sid, c, tags=tags(len(c))) for sid, c in cells.items()]
    p2 = [mk_absent(60, 30, row0=500, tags=tags(30)), mk_absent(63, 20, row0=500, tags=tags(20))]
    return p1, p2


@gpu
def test_int64_key_values(bydb, gpu_ctx):
    """INT64_MIN, INT64_MAX, -1, 0 (the empty-slot pattern: it lives in the flag word), values that differ only in the top
    byte, 40 values homed at slot 1023, nil next to each of them in raw cells, and blocks without the key column (key 0) in a
    second part; one series group and a group per series."""
    p1, p2 = value_parts()
    parts = [(build_keyed(p1), p1), (build_keyed(p2, 2), p2)]
    with KScan64(bydb, gpu_ctx, parts, groups={60: 0, 61: 0, 62: 0, 63: 0}) as k:
        got = k.query(ctx="values")
        assert got.n_keys == len(set(SPECIAL) | set(wrap_values()))
        assert {unle(x) for x in got.key} == set(SPECIAL) | set(wrap_values())
        k.query(aggs=[("i", SUM), ("f", MIN)], sids=[60, 63], ctx="values: raw and absent")
        k.query(preds=[O.Pred(FAM, "c", O.OP_GE, 2)], ctx="values")
    with KScan64(bydb, gpu_ctx, parts) as k:
        k.query(ctx="values, a group per series")
        k.query(top=(3, 1, False), ctx="values, top")


# ------------------------------------------------------------------ the cap and the refusals
def cap_series():
    def t(n):
        return {"c": (np.ones(n, np.int64), np.zeros(n, bool)), "s": [b"y"] * n}
    spec = [(40, [1000 + i for i in range(64) for _ in range(2)]), (41, [7] * 10), (42, [9] * 7),
            (43, [2000 + (i * 37) % 128 for i in range(128)]), (44, [3000 + (i * 41) % 128 for i in range(128)]),
            (46, int_tag_values("dc_neg", BLOCK, None)), (47, [wrap64(11 + (1 << 63) * r) for r in range(BLOCK)]),
            (48, [wrap64(-3 + (1 << 62) * r) for r in range(BLOCK)])]
    return [mk64(sid, cells, tags=t(len(cells))) for sid, cells in spec]


@gpu
def test_int64_key_cap_and_refusals(bydb, gpu_ctx):
    """max_values 0 (64), 1 and 256 at and one past the cap -> ENOMEM, 257 -> EINVAL; an 8193-row DeltaConst block of 8193
    values -> ENOMEM; steps 2^63 / 2^62 over 8193 rows hold 2 / 4 values (one fewer allowed -> ENOMEM); 7 user predicates
    answer and 8 give ENOTSUP; VT_INT64 on a string tag, value_type 0 / VT_STR on the int64 tag and unknown value types ->
    EINVAL; overlapping parts -> ENOTSUP.  The context answers a plain query after each refusal."""
    ss = cap_series()
    P, E = O.Pred, bydb.capi
    with KScan64(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        assert k.query(sids=[40], max_values=0, ctx="cap64").n_keys == 64
        k.fails(E.ENOMEM, sids=[40, 41], max_values=0)
        assert k.query(sids=[42], max_values=1, ctx="cap1").n_keys == 1
        k.fails(E.ENOMEM, sids=[41, 42], max_values=1)
        assert k.query(aggs=[("i", SUM), ("f", MIN)], sids=[43, 44], max_values=256, ctx="cap256").n_keys == 256
        k.fails(E.ENOMEM, sids=[41, 43, 44], max_values=256)
        k.fails(E.EINVAL, sids=[40], max_values=257)
        k.fails(E.ENOMEM, sids=[46])
        assert k.query(sids=[47], max_values=2, ctx="step 2^63").n_keys == 2
        k.fails(E.ENOMEM, sids=[47], max_values=1)
        assert k.query(sids=[48], max_values=4, ctx="step 2^62").n_keys == 4
        k.fails(E.ENOMEM, sids=[48], max_values=3)
        seven = [P(FAM, "c", O.OP_GE, -5), P(FAM, "c", O.OP_LE, 5), P(FAM, "c", O.OP_NE, 9), P(FAM, "c", O.OP_GT, -9),
                 P(FAM, "c", O.OP_LT, 9), P(FAM, "s", O.OP_EQ, b"y"), P(FAM, "nope", O.OP_NE, b"x")]
        k.query(sids=[40, 42], preds=seven, ctx="seven predicates")
        k.fails(E.ENOTSUP, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)])
        k.fails(E.EINVAL, sids=[40], key="s")
        for vt in (0, E.VT_STR, E.VT_BINARY, E.VT_FLOAT64, 5, 99):
            k.fails(E.EINVAL, sids=[40], value_type=vt)
    over = [mk64(40, [1, 2] * 20, row0=30, tags={"c": (np.ones(40, np.int64), np.zeros(40, bool)), "s": [b"y"] * 40})]
    with KScan64(bydb, gpu_ctx, [(build_keyed(ss), ss), (build_keyed(over, 2), over)]) as k:
        k.fails(E.ENOTSUP, sids=[40])


# ------------------------------------------------------------------ insertion order
EDGE_ROWS = [0, 31, 32, 33, 8191, 8192]


def order_series():
    """sid 10: 8193 rows of 7 with value 1000 + r first at row r of EDGE_ROWS; sid 11: two blocks, values first in the second;
    sid 12: -5 at rows 5 and 20, -6 at row 10, nil at row 40; sid 13 only 7; sid 14 repeats values of sid 10.  Tags c
    (int64, -1 at row 5 of sid 12), s (dictionary, "n" there) and dod (a DoD page)."""
    rng = np.random.default_rng(0x0D64)
    k10 = [7] * BLOCK
    for r in EDGE_ROWS:
        k10[r] = 1000 + r
    k11 = [7] * (BLOCK + 40)
    k11[BLOCK - 1] = 21
    k11[BLOCK], k11[BLOCK + 33], k11[BLOCK + 7], k11[BLOCK + 8] = 22, 23, 24, 21
    k12 = [7] * 64
    k12[5] = k12[20] = -5
    k12[10] = -6
    k12[40] = None
    k14 = [9192, 7, 1031, -6, 1000] * 8
    ss = [mk64(10, k10), mk64(11, k11), mk64(12, k12), mk64(13, [7] * 50), mk64(14, k14, row0=3)]
    for s in ss:
        c = np.ones(s.n, np.int64)
        if s.sid == 12:
            c[5] = -1
        s.tags["c"] = (c, np.zeros(s.n, bool))
        s.tags["s"] = [b"n" if (s.sid == 12 and r == 5) else b"y" for r in range(s.n)]
        s.tags["dod"] = ((100 + np.concatenate([[0], np.cumsum(rng.integers(1, 9, s.n - 1))])).astype(np.int64), np.zeros(s.n, bool))
    return ss


def ab_parts():
    """two parts that follow each other in time: values 31 / 30 first show in the second (sid 21 shows 30 earlier than sid 20)"""
    a = [mk64(20, [1, 2] * 50), mk64(21, [1] * 100)]
    kb20 = [2] * 100
    kb20[50], kb20[60] = 31, 30
    kb21 = [1] * 100
    kb21[20] = 30
    return a, [mk64(20, kb20, row0=100), mk64(21, kb21, row0=100)]


@gpu
def test_int64_key_insertion_order(bydb, gpu_ctx):
    """First surviving rows at rows 0, 31, 32, 33, 8191, 8192 of an 8193-row block, in the second block of a series and in a
    second part (parts in both orders); a time cut, an int64 and a dictionary predicate, a DoD predicate, and a predicate on
    the key tag itself (its value's group vanishes while n_keys still counts it); series groups out of first-appearance
    order; Top-N 1 / all over COUNT ties in both directions."""
    ss = order_series()
    P = O.Pred
    with KScan64(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={10: 2, 11: 0, 12: 3, 13: 1, 14: 2}) as k:
        got = k.query(ctx="order")
        assert [unle(x) for x in got.key[:7]] == [1000, 7, 1031, 1032, 1033, 9191, 9192]
        k.query(tmin=T0 + 6 * STEP, ctx="order")
        k.query(tmin=T0 + 33 * STEP, tmax=T0 + (BLOCK + 20) * STEP, ctx="order")
        k.query(preds=[P(FAM, "c", O.OP_GE, 0)], ctx="order")
        k.query(preds=[P(FAM, "s", O.OP_NE, b"n")], ctx="order")
        k.query(preds=[P(FAM, "dod", O.OP_GE, 150)], ctx="order: DoD predicate")
        got = k.query(preds=[P(FAM, KT, O.OP_NE, 7)], ctx="order: predicate on the key")
        assert 7 not in {unle(x) for x in got.key}
        for n in (1, 2048):
            for desc in (True, False):
                k.query(aggs=[("i", COUNT), ("f", MAX)], top=(n, 0, desc), ctx="order: top")
    a, b = ab_parts()
    with KScan64(bydb, gpu_ctx, [(build_keyed(a), a), (build_keyed(b), b)], groups={20: 0, 21: 0}) as k:
        for order in ([0, 1], [1, 0]):
            got = k.query(order=order, ctx=f"parts {order}")
            assert [unle(x) for x in got.key] == [1, 2, 31, 30]
            k.query(order=order, tmin=T0 + 120 * STEP, ctx=f"parts {order}")


# ------------------------------------------------------------------ the operator (scan_operator.py)
SVC = {70: b"svc-a", 71: b"svc-b", 72: b"svc-a", 73: b"svc-c", 74: b"svc-b"}


def operator_series():
    """five series: int64 key k (nil in places), string key z (nil in places), a non-key string tag note"""
    rng = np.random.default_rng(0x0B)
    out = []
    for j, sid in enumerate(SVC):
        n = 40 + 17 * j
        ks = [None if r % 11 == 3 else int(x) for r, x in enumerate(rng.integers(-3, 4, n))]
        z = [None if r % 13 == 5 else b"z%d" % ((r // 4 + j) % 3) for r in range(n)]
        if j == 1:
            z[7] = b"\xffbad"   # not UTF-8: comes back through surrogateescape
        out.append(mk64(sid, ks, tags={"z": z, "note": [b"x"] * n}))
    return out


def _operator(bydb, ctx, handles, keys, series_ids, series_tags, aggs, top=None, limit=None, order_desc=False):
    so = bydb.scan_operator
    cols = [so.ColumnDef("svc", so.ColumnRole.RoleTag, so.ColumnType.ColumnTypeString, FAM),
            so.ColumnDef("z", so.ColumnRole.RoleTag, so.ColumnType.ColumnTypeString, FAM),
            so.ColumnDef(KT, so.ColumnRole.RoleTag, so.ColumnType.ColumnTypeInt64, FAM),
            so.ColumnDef("note", so.ColumnRole.RoleTag, so.ColumnType.ColumnTypeString, FAM),
            so.ColumnDef("i", so.ColumnRole.RoleField, so.ColumnType.ColumnTypeInt64),
            so.ColumnDef("f", so.ColumnRole.RoleField, so.ColumnType.ColumnTypeFloat64)]
    fn = {SUM: so.AggSum, COUNT: so.AggCount, MIN: so.AggMin, MAX: so.AggMax, MEAN: so.AggMean}
    specs = [so.AggSpec(f"a{a}", fn[f], 4 if col == "i" else 5) for a, (col, f) in enumerate(aggs)]
    scan = so.ScanSpec(parts=handles, series_ids=series_ids, series_tags=series_tags, order_desc=order_desc, max_key_values=64)
    op = so.GPUScanAgg(ctx, so.BatchSchema(cols), keys, specs, scan, batch_size=2,
                       top=None if top is None else so.TopSpec(*top), limit=None if limit is None else so.LimitSpec(*limit))
    op.Init()
    rows = []
    while True:
        b = op.NextBatch()
        if b is None:
            return rows
        assert 0 < b.Len <= 2
        rows += list(zip(*b.Columns))


def _vals(exp_vals):
    return [m for m, _ in exp_vals]


@gpu
def test_operator_stored_keys(bydb, gpu_ctx):
    """GPUScanAgg with a per-series key plus a stored string key, and with a stored int64 key alone under Top and an
    offset / limit window, in batches of 2, against key_model; two stored keys and order_desc with a stored key are refused."""
    ss = operator_series()
    part = build_keyed(ss)
    sids = [72, 70, 74, 71, 73]   # index order, not ascending
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        aggs = [("i", SUM), ("i", COUNT), ("f", MAX)]
        svc_tags = {(FAM, "svc"): [SVC[s] for s in sids]}
        # per-series key svc + stored string key z: series groups numbered in the index order's first appearances
        firsts = list(dict.fromkeys(SVC[s] for s in sids))
        gid = {s: firsts.index(SVC[s]) for s in sids}
        rows = _operator(bydb, gpu_ctx, [h], [0, 1], sids, svc_tags, aggs)
        exp = key_model(ss, gid, sorted(sids), aggs, [], I64_MIN, I64_MAX, "z", None)
        want = [(firsts[g], z.decode("utf-8", "surrogateescape"), None, None, *_vals(v)) for (g, z), _, v in exp]
        got = [(r[0], r[1], r[2], r[3], *r[4:]) for r in rows]
        assert [tuple(x) for x in got] == want, f"svc + z: {got[:4]} vs {want[:4]}"
        # stored int64 key alone, Top 3 by COUNT ascending, then an offset / limit window over plain order
        one = {s: 0 for s in sids}
        for top, limit in (((3, 1, False), None), (None, (2, 3)), ((4, 0, True), (1, 2))):
            rows = _operator(bydb, gpu_ctx, [h], [2], sids, {}, aggs, top=top, limit=limit)
            exp = key_model(ss, one, sorted(sids), aggs, [], I64_MIN, I64_MAX, KX, top)
            if limit:
                exp = exp[limit[0]:limit[0] + limit[1]]
            want = [(None, None, unle(k), None, *_vals(v)) for (_, k), _, v in exp]
            assert [tuple(r) for r in rows] == want, f"k top={top} limit={limit}: {rows[:4]} vs {want[:4]}"
        with pytest.raises(bydb.BydbError) as e:
            _operator(bydb, gpu_ctx, [h], [1, 2], sids, {}, aggs)
        assert e.value.code == bydb.capi.ENOTSUP and f"{FAM}/{KT}:" in str(e.value)
        with pytest.raises(bydb.BydbError) as e:
            _operator(bydb, gpu_ctx, [h], [2], sids, {}, aggs, order_desc=True)
        assert e.value.code == bydb.capi.ENOTSUP
        with pytest.raises(ValueError):   # a field column as a key is not a stored tag: it still needs per-series values
            _operator(bydb, gpu_ctx, [h], [4], sids, {}, aggs)
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ the claims above, on the CPU
def test_int64_key_case_layouts():
    """The oracle's codecs and the fold behind the twin: nil and 0 give the same 8 little-endian key bytes; every page kind,
    value set and hash-slot layout the GPU cases claim holds."""
    assert twin([None, 0, -1, 1, I64_MIN]) == [b"\0" * 8, b"\0" * 8, b"\xff" * 8, b"\x01" + b"\0" * 7, b"\0" * 7 + b"\x80"]
    assert all(le(v) == v.to_bytes(8, "little", signed=True) for v in SPECIAL + wrap_values())
    # the oracle's own reading of a stored int64 column: nil and 0 fall into one key, the per-value rule holds
    ss = [mk64(1, [None, 0, 5, None, -1, 0, 5, None]), mk64(2, [7, None, 7, 0])]
    part = build_keyed(ss)
    oq = O.Query([part], np.array([1, 2], np.uint64), [("i", SUM), ("i", COUNT)], groups=np.array([0, 1], np.int32), n_groups=2)
    want = O.run_query(dataclasses.replace(oq, group_key=(FAM, KX)))
    assert [(g, unle(k), int(n)) for g, k, n in zip(want.group_id.tolist(), want.key, want.rows)] == \
        [(0, 0, 5), (0, 5, 2), (0, -1, 1), (1, 7, 2), (1, 0, 2)]
    oracle_per_value(oq, [], want, [("i", SUM), ("i", COUNT)], "oracle int64 reading")
    for kind in INT_KINDS:
        for s in kind_series(kind):
            cells = [None if nl else int(v) for v, nl in zip(*s.tags[KT])]
            assert s.tags[KX] == twin(cells)
            assert len(set(s.tags[KX])) <= 65, (kind, s.n)
            if s.n >= 31:
                assert s.kind(("t", KT), 0, s.n)[0] == INT_CLASS[kind], (kind, s.n, s.kind(("t", KT), 0, s.n))
        assert sum(len(set(s.tags[KX])) for s in kind_series(kind)) <= 256
    raw = kind_series("raw")[-1]
    assert raw.n == BLOCK and [r for r in range(raw.n) if raw.tags[KT][1][r]][:3] == [0, 31, 32] and raw.tags[KT][1][-1]
    assert raw.tags[KT][0][33] == 0 and not raw.tags[KT][1][33]
    assert {s.n for s in kind_series("dc_wrap")} == set(SIZES)
    assert [len(set(kind_series(k)[-1].tags[KX])) for k in ("dc_neg", "dc_wrap")] == [4, 2]
    # values and the hash
    assert len(wrap_values()) == 40 and {fnv_slot(le(v)) for v in wrap_values()} == {1023}
    assert len({le(v)[:7] for v in TOP_BYTE}) == 1 and len(set(TOP_BYTE)) == len(TOP_BYTE)
    p1, p2 = value_parts()
    assert p1[0].kind(("t", KT), 0, p1[0].n)[0] == "raw" and all(KT not in s.tags for s in p2)
    # the cap series
    cs = {s.sid: s for s in cap_series()}
    assert [len(set(cs[s].tags[KX])) for s in (40, 41, 42, 43, 44, 46, 47, 48)] == [64, 1, 1, 128, 128, BLOCK, 2, 4]
    assert not set(cs[43].tags[KX]) & set(cs[44].tags[KX]) and not set(cs[41].tags[KX]) & set(cs[43].tags[KX] + cs[44].tags[KX])
    assert [cs[s].kind(("t", KT), 0, BLOCK)[0] for s in (46, 47, 48)] == ["delta_const"] * 3
    # first appearances
    os_ = order_series()
    k10 = os_[0].tags[KT][0].tolist()
    assert [k10.index(1000 + r) for r in EDGE_ROWS] == EDGE_ROWS and k10.index(7) == 1
    assert os_[1].chunks() == [(0, BLOCK), (BLOCK, BLOCK + 40)] and os_[1].tags[KT][0].tolist().index(21) == BLOCK - 1
    assert {s.kind(("t", "dod"), lo, hi)[0] for s in os_ for lo, hi in s.chunks()} == {"dod"}
    assert any(s.tags[KT][1].any() for s in operator_series())

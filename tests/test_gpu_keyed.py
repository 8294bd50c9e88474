"""Group-by on a stored tag (bydb_scan_agg_keyed, DESIGN.md 4.6) against the oracle and an independent model, at its boundaries.

The keyed path has kernels of its own: key_values_kernel enters the values of every selected block's dictionary page into a
1024-slot FNV-1a open-addressing table (32 values per warp step, the byte offset carried from one window to the next),
key_pack_kernel packs them, one ordinary scan pass per value v runs with the extra predicate "tag is v" (kOpEqOrNil for "": a nil
cell and "" are one key) and records where each series first shows v (Pfirst -> Kts / Krow), key_order_kernel /
key_perm_kernel rank the V x G composite groups into insertion order, and permute_table_kernel hands the table to the ordinary
finalisation and Top-N.

Every query is checked three ways:
  - against the oracle with group_key=(family, tag): parity of groups, rows and aggregates, and the per-row key lists;
  - against `key_model`, a plain Python fold over the generated rows of the selected series in (series id, time) order: a row's
    key is its cell (nil and a missing column give b""); composite groups in first-seen order, their rows, and the fold rules of
    test_gpu_fallback.py (int64 SUM mod 2^64, MEAN quirks, float MIN / MAX bit for bit, float SUM within 1e-9 * sum|x|); Top-N
    is a stable sort of that order, so ties go to the group inserted first;
  - key discovery and the counters: n_keys is the number of distinct values in the dictionaries of the *selected* blocks (series
    in the query, time span meeting the range), which can exceed the keys that survive predicates; rows_matched is the model's
    row count; rows_scanned / blocks_scanned are V times one pass's; no block takes the express lane; and `lane_model` predicts
    blocks_slow_lane / slow_lane_reasons pass by pass: a deferring tag page (DoD, wide delta, raw cells, plain) defers its block
    in every pass in which the block has a row in range (reason 2), a deferring field page only in the passes whose value has a
    surviving row in the block (reason 4 << field, the first such field).
"""
import dataclasses
import functools

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_fallback import BLOCK, COUNT, MAX, MEAN, MIN, SUM, F, I, Series, fold
from tests.test_gpu_lanes import WIDE
from tests.test_gpu_masks import I64_MAX, I64_MIN, dict_layout, str_tag_class
from tests.test_oracle_model_sweep import OPS

gpu = pytest.mark.gpu

FAM, KT = "default", "k"
AGGS = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("i", MEAN), ("f", SUM), ("f", MIN), ("f", MAX), ("f", MEAN)]
DEFER_TAG = ("raw", "dod", "wide", "plain")   # tag page kinds the fast lane hands to the slow lane
KEY_SLOTS = 1024
_pid = [120_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


# ------------------------------------------------------------------ the hash of key_insert
def fnv_slot(b):
    """home slot of a value in key_values_kernel's table: FNV-1a over the bytes, (h ^ h >> 32) & 1023"""
    h = 0xcbf29ce484222325
    for x in b:
        h = ((h ^ x) * 0x100000001b3) & 0xFFFF_FFFF_FFFF_FFFF
    return (h ^ (h >> 32)) & (KEY_SLOTS - 1)


def _find(slot, n, make):
    out, i = [], 0
    while len(out) < n:
        c = make(i)
        if fnv_slot(c) == slot:
            out.append(c)
        i += 1
    return out


@functools.lru_cache(None)
def hash_sets():
    """-> (40 values homed at slot 1023, values of 2..64 bytes homed at the slot of "", values of 1..64 bytes sharing one slot)"""
    wrap = _find(1023, 40, lambda i: b"w%d" % i)
    empty_slot = fnv_slot(b"")
    with_empty = [_find(empty_slot, 1, lambda i, L=L: i.to_bytes(L, "big"))[0] for L in (2, 3, 8, 63, 64)]
    q = b"\x9c"
    same = [q] + [_find(fnv_slot(q), 1, lambda i, L=L: (i + 0x7070).to_bytes(L, "little"))[0] for L in (2, 5, 33, 64)]
    return wrap, with_empty, same


# ------------------------------------------------------------------ series, parts and the models
def std_fields(sid, n):
    """int64 `i` (a narrow delta page) and float64 `f` (short positive decimals) of one series"""
    r = np.arange(n, dtype=np.int64)
    i = 1000 + sid + np.cumsum(((r * 37 + sid) % 63 + 1) * np.where(r % 2 == 0, 1, -1))
    f = np.round(((r * 53 + sid * 7) % 2000) / 10.0 + 0.1, 1)
    return {"i": (I, i, None), "f": (F, f, None)}


def mk(sid, keys, row0=0, tags=None, fields=None):
    return Series(sid, fields or std_fields(sid, len(keys)), {KT: list(keys), **(tags or {})}, row0=row0)


def build_keyed(series, version=1, binary=()):
    """test_gpu_fallback.build, with the tags named in `binary` stored as VT_BINARY"""
    series = sorted(series, key=lambda s: s.sid)
    sids = np.concatenate([np.full(s.n, s.sid, np.uint64) for s in series])
    fields = []
    for name, (vt, _, _) in series[0].fields.items():
        v = np.concatenate([np.where(s.fields[name][2], 0, s.fields[name][1]) for s in series])
        nl = np.concatenate([s.fields[name][2] for s in series]).astype(np.uint8)
        fields.append((name, vt, v, nl if nl.any() else None))
    cols = []
    for name, tag in series[0].tags.items():
        if isinstance(tag, tuple):
            v = np.concatenate([np.where(s.tags[name][1], 0, s.tags[name][0]) for s in series])
            nl = np.concatenate([s.tags[name][1] for s in series]).astype(np.uint8)
            cols.append((name, I, v, nl if nl.any() else None))
        else:
            cols.append((name, O.VT_BINARY if name in binary else O.VT_STR, [x for s in series for x in s.tags[name]], None))
    return build_part(sids, np.concatenate([s.ts for s in series]), np.full(sids.size, version, np.int64), fields, [(FAM, cols)])


def key_cells(s, key):
    cells = s.tags.get(key)
    return [b""] * s.n if cells is None else [b"" if c is None else c for c in cells]


def row_mask(s, preds, tmin, tmax):
    m = s.alive & (s.ts >= tmin) & (s.ts <= tmax)
    for p in preds:
        m &= s.passes(p) if p.tag in s.tags else OPS[p.op](False, 0)   # an absent tag: every cell nil
    return m


def selected_blocks(series, sids, tmin, tmax):
    """(series, lo, hi) of every block the device selects: series in the query, time span meeting [tmin, tmax]"""
    sel = set(int(x) for x in sids)
    return [(s, lo, hi) for s in series if s.sid in sel for lo, hi in s.chunks()
            if tmin <= tmax and not (s.ts[hi - 1] < tmin or s.ts[lo] > tmax)]


class Comp:
    def __init__(self):
        self.rows = 0
        self.parts = []   # (series, row indices)


def key_model(series, gid, sids, aggs, preds, tmin, tmax, key, top):
    """-> [((group, key), rows, [value per agg])] in result order"""
    sel = set(int(x) for x in sids)
    comps = {}
    for s in sorted((s for s in series if s.sid in sel), key=lambda s: (s.sid, int(s.ts[0]))):
        keys = key_cells(s, key)
        per = {}
        for r in np.nonzero(row_mask(s, preds, tmin, tmax))[0].tolist():
            per.setdefault(keys[r], []).append(r)
        for k, rows in per.items():
            c = comps.setdefault((gid[s.sid], k), Comp())
            c.rows += len(rows)
            c.parts.append((s, np.array(rows, dtype=np.int64)))
    out = []
    for ck, c in comps.items():
        vals = []
        for f, fn in aggs:
            x = np.concatenate([s.fields[f][1][r][~s.fields[f][2][r]] for s, r in c.parts])
            vals.append((fold(series[0].fields[f][0], fn, x), x))
        out.append((ck, c.rows, vals))
    if top:
        n, a, desc = top
        out = sorted(out, key=lambda e: e[2][a][0], reverse=desc)[:n]   # stable: ties keep insertion order
    return out


def lane_model(series, sids, aggs, preds, tmin, tmax, key, values):
    """(blocks_slow_lane, slow_lane_reasons) summed over the V passes"""
    fields = list(dict.fromkeys(f for f, _ in aggs))
    need = dict.fromkeys(fields, 0)
    for f, fn in aggs:
        need[f] |= 1 if fn in (SUM, MEAN) else 2 if fn in (MIN, MAX) else 0
    slow = reasons = 0
    for s, lo, hi in selected_blocks(series, sids, tmin, tmax):
        if not ((s.ts[lo:hi] >= tmin) & (s.ts[lo:hi] <= tmax)).any():
            continue
        if any(p.tag in s.tags and s.kind(("t", p.tag), lo, hi)[0] in DEFER_TAG for p in preds):
            slow += len(values)
            reasons |= 2
            continue
        why = next((4 << c for c, f in enumerate(fields) for k, nl in [s.kind(("f", f), lo, hi)]
                    if (k == "raw" and (need[f] or nl)) or (k == "wide" and need[f])), 0)
        if why:
            keys = key_cells(s, key)
            m = row_mask(s, preds, tmin, tmax)
            live = {keys[r] for r in range(lo, hi) if m[r]}
            slow += len(live & set(values))
            reasons |= why if live else 0
    return slow, reasons


class KScan:
    """Parts registered once for many keyed queries; each is checked against the oracle, key_model and the counters."""

    def __init__(self, bydb, gpu_ctx, parts_series, groups=None):
        self.bydb, self.ctx = bydb, gpu_ctx
        self.parts = [p for p, _ in parts_series]
        self.series = [s for _, ss in parts_series for s in ss]
        self.usid = np.array(sorted({s.sid for s in self.series}), dtype=np.uint64)
        self.gid = groups or {int(sid): g for g, sid in enumerate(self.usid.tolist())}
        self.handles = []

    def __enter__(self):
        pid = _next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, p in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def oquery(self, aggs, preds, tmin, tmax, top, sids, handles_order=None):
        sids = self.usid if sids is None else np.array(sorted(sids), dtype=np.uint64)
        groups = np.array([self.gid[int(s)] for s in sids.tolist()], dtype=np.int32)
        n_groups = max(self.gid.values()) + 1
        tn, ta, td = top or (0, 0, True)
        parts = self.parts if handles_order is None else [self.parts[i] for i in handles_order]
        oq = O.Query(parts, sids, list(aggs), groups=groups, n_groups=n_groups, tmin=tmin, tmax=tmax, preds=list(preds),
                     top_n=tn, top_agg=ta, top_desc=td)
        handles = self.handles if handles_order is None else [self.handles[i] for i in handles_order]
        return oq, to_gpu_query(self.bydb, handles, oq)

    def query(self, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, sids=None, key=KT, max_values=256, order=None, ctx=""):
        preds = list(preds)
        oq, q = self.oquery(aggs, preds, tmin, tmax, top, sids, order)
        ctx = f"{ctx}/key={key}/{[(f, fn) for f, fn in aggs]}/{[(p.tag, p.op, p.value) for p in preds]}" \
              f"/{(tmin - T0) // STEP if tmin > I64_MIN else '-'}..{(tmax - T0) // STEP if tmax < I64_MAX else '-'}/top{top}"
        got = self.ctx.scan_agg_keyed(q, FAM, key, max_values)
        want = O.run_query(dataclasses.replace(oq, group_key=(FAM, key)))
        assert_parity(got, want, aggs, ctx)
        assert got.key == want.key, f"{ctx}: keys {got.key[:12]} vs oracle {want.key[:12]}"
        # the model
        exp = key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, key, top)
        got_comp = list(zip(got.group_id.tolist(), got.key))
        assert got_comp == [e[0] for e in exp], f"{ctx}: composite groups {got_comp[:12]}, model {[e[0] for e in exp][:12]}"
        assert got.rows.tolist() == [e[1] for e in exp], f"{ctx}: rows vs model"
        for i, (ck, _, vals) in enumerate(exp):
            for a, ((f, fn), (m, x)) in enumerate(zip(aggs, vals)):
                where = f"{ctx}: group {ck} agg {a} ({f},{fn})"
                if not got.is_float[a]:
                    assert int(got.val_i64[i, a]) == m, f"{where}: {got.val_i64[i, a]}, model {m}"
                elif fn in (MIN, MAX):
                    assert got.val_f64[i:i + 1, a].view(np.uint64)[0] == np.array([m]).view(np.uint64)[0], \
                        f"{where}: {got.val_f64[i, a]!r}, model {m!r} (bit-exact)"
                else:
                    tol = 1e-9 * float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1)
                    assert abs(float(got.val_f64[i, a]) - m) <= tol, f"{where}: {got.val_f64[i, a]!r}, model {m!r}"
        # key discovery and the counters
        blocks = selected_blocks(self.series, oq.sids, tmin, tmax)
        values = {c for s, lo, hi in blocks for c in key_cells(s, key)[lo:hi]}
        V = len(values)
        st = got.stats
        assert got.n_keys == V and set(want.key) <= values, f"{ctx}: n_keys {got.n_keys}, {V} values in the selected blocks"
        rows = sum(e[1] for e in key_model(self.series, self.gid, oq.sids, aggs, preds, tmin, tmax, key, None)) if top else \
            sum(e[1] for e in exp)
        assert st.rows_matched == rows, f"{ctx}: rows_matched {st.rows_matched}, model {rows}"
        assert st.rows_scanned == V * sum(hi - lo for _, lo, hi in blocks), f"{ctx}: rows_scanned {st.rows_scanned}"
        assert st.blocks_scanned == V * len(blocks), f"{ctx}: blocks_scanned {st.blocks_scanned}, {V} x {len(blocks)}"
        assert st.blocks_express_lane == 0, f"{ctx}: express-lane blocks {st.blocks_express_lane}"
        lanes = lane_model(self.series, oq.sids, aggs, preds, tmin, tmax, key, values)
        assert (st.blocks_slow_lane, st.slow_lane_reasons) == lanes, \
            f"{ctx}: (slow blocks, reasons) {(st.blocks_slow_lane, st.slow_lane_reasons)}, model {lanes}"
        return got

    def fails(self, code, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, sids=None, key=KT, max_values=256, order=None):
        """the keyed call fails with `code`; afterwards the context still answers a plain query"""
        _, q = self.oquery(aggs, preds, tmin, tmax, None, sids, order)
        with pytest.raises(self.bydb.BydbError) as e:
            self.ctx.scan_agg_keyed(q, FAM, key, max_values)
        assert e.value.code == code, (code, e.value)
        oq, q = self.oquery(AGGS, [], I64_MIN, I64_MAX, None, self.usid[:1], None if order is None else order[:1])
        got = self.ctx.scan_agg(q)
        assert_parity(got, O.run_query(oq), AGGS, "plain query after a keyed error")


# ------------------------------------------------------------------ the INT64_MAX first-row timestamp (a suspected defect)
def sentinel_series():
    """one-row series at INT64_MAX / INT64_MIN: a value whose first block in a series has ts_min == INT64_MAX is present"""
    out = []
    for sid, ts, key in [(30, I64_MAX, b"m"), (31, T0, b"n"), (32, I64_MIN, b"m"), (33, I64_MAX, b"o"), (34, I64_MAX - 1, b"o"),
                         (35, I64_MAX, None)]:
        s = mk(sid, [key])
        s.ts = np.array([ts], dtype=np.int64)
        out.append(s)
    return out


@gpu
def test_first_row_at_int64_max(bydb, gpu_ctx):
    """A block at the last representable timestamp (which the default tmax includes) places its values where the oracle does,
    in one series group and in one group per series; a range that ends just before it drops them."""
    ss = sentinel_series()
    part = build_keyed(ss)
    with KScan(bydb, gpu_ctx, [(part, ss)], groups={s.sid: 0 for s in ss}) as k:
        got = k.query(ctx="sentinel")
        assert got.key == [b"m", b"n", b"o", b""]
        k.query(tmax=I64_MAX - 1, ctx="sentinel")
        k.query(tmin=I64_MAX, ctx="sentinel")
        k.query(top=(2, 1, False), ctx="sentinel")
    with KScan(bydb, gpu_ctx, [(part, ss)]) as k:
        k.query(ctx="sentinel, a group per series")


# ------------------------------------------------------------------ dictionary shapes
SHAPE_COUNTS = [1, 2, 31, 32, 33, 63, 64, 65, 126, 127, 128, 255, 256]
ONE = [bytes([x]) for x in list(range(0, 62)) + [0x61] + list(range(0x80, 0xbf))]   # 126 one-byte values: \x00, "a", >= 0x80
PREFIX = [b"a\x00", b"ab", b"abc", b"ab\x00"]
LONG = [b"z" * 63, b"z" * 64, b"z" * 63 + b"\x00", b"\xff" * 64, b"\x80" * 63]


@functools.lru_cache(None)
def shape_pool():
    """256 distinct keys: "", 126 one-byte values, prefix pairs of "a", 63- and 64-byte values, short names"""
    pool = [b""] + ONE + PREFIX + LONG
    pool += [b"m%03d" % i for i in range(256 - len(pool))]
    assert len(set(pool)) == 256
    return pool


def _runs(vals, reps=2):
    """each value in runs of 1..3 rows, the value list cycled `reps` times"""
    out = []
    for rep in range(reps):
        for j, v in enumerate(vals):
            out += [v] * (1 + (j + rep) % 3)
    return out


@functools.lru_cache(None)
def shape_blocks():
    """name -> key cells of one block"""
    pool = shape_pool()
    c = {}
    for k in SHAPE_COUNTS:
        st = (k * 37) % 256
        c[f"values{k}"] = _runs([pool[(st + j) % 256] for j in range(k)])
    c["lens_zstd_data_short"] = _runs([None, b""] + ONE[:125], 1)        # 127 entries, 125 value bytes
    c["lens_short_data_zstd"] = _runs(LONG + [b"a", b"a\x00"])
    c["nil_empty"] = [None, b"", b"", None, b"a", None, b""] * 5
    c["prefixes"] = _runs([b"a", b"a\x00", b"ab", b"ab\x00", b"abc", b"\x00", b""])
    c["high_bytes"] = _runs([b"\x80", b"\xff" * 64, b"\xa0", b"\x00", b"\x80" * 63])
    return c


SHAPE_EXPECT = {  # name -> (dictionary entries, packed width, lens zstd, data zstd)
    "values1": (1, 2, False, False), "values2": (2, 2, False, False), "values31": (31, 5, False, True), "values32": (32, 5, False, True),
    "values33": (33, 6, False, True), "values63": (63, 6, False, False), "values64": (64, 6, False, False),
    "values65": (65, 7, False, True), "values126": (126, 7, False, True), "values127": (127, 7, True, True),
    "values128": (128, 7, True, True), "values255": (255, 8, True, True), "values256": (256, 8, True, True),
    "lens_zstd_data_short": (127, 7, True, False), "lens_short_data_zstd": (7, 3, False, True), "nil_empty": (3, 2, False, False),
    "prefixes": (7, 3, False, False), "high_bytes": (5, 3, False, True),
}


def shape_parts():
    """part 1: one series per shape; part 2 (later in time): the same series with the value lists reversed"""
    blocks = shape_blocks()
    s1 = [mk(100 + i, cells) for i, cells in enumerate(blocks.values())]
    s2 = [mk(100 + i, cells[::-1], row0=5000) for i, cells in enumerate(blocks.values())]
    return s1, s2


@gpu
def test_dictionary_shapes(bydb, gpu_ctx):
    """key_values_kernel over dictionaries of 1..256 values (32-value windows carrying the byte offset), short and
    zstd-inflated lens / data blocks in every combination, 0-, 1-, 63- and 64-byte values, nil next to "", bytes >= 0x80 and
    \\x00, prefix pairs, equal bytes at many addresses in two parts: 256 distinct keys, 256 passes per query."""
    s1, s2 = shape_parts()
    groups = {s.sid: i % 5 for i, s in enumerate(s1)}
    with KScan(bydb, gpu_ctx, [(build_keyed(s1), s1), (build_keyed(s2, 2), s2)], groups=groups) as k:
        got = k.query(ctx="shapes")
        assert got.n_keys == 256
        k.query(aggs=[("i", SUM), ("f", MAX)], tmin=T0 + 40 * STEP, tmax=T0 + 5100 * STEP, ctx="shapes")
        k.query(aggs=[("i", COUNT)], sids=[s.sid for s in s1[:3]] + [s1[13].sid, s1[15].sid], ctx="shapes: few blocks")


# ------------------------------------------------------------------ hash-table collisions
@gpu
def test_hash_collisions(bydb, gpu_ctx):
    """40 values homed at slot 1023 (probes wrap to slot 0), values of 2..64 bytes homed at the slot of "" (stored with address
    0, length 0) next to nil and "", and same-slot values of different lengths, spread over blocks of several series."""
    wrap, with_empty, same = hash_sets()
    vals = wrap + with_empty + same
    ss = [mk(200, _runs(wrap[:20] + [None] + with_empty[:2])), mk(201, _runs(wrap[20:] + same[:3] + [b""])),
          mk(202, _runs(with_empty + same + wrap[::7])), mk(203, _runs(same[::-1] + wrap[::-3] + [None, b""]))]
    with KScan(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups={200: 0, 201: 1, 202: 0, 203: 1}) as k:
        got = k.query(ctx="hash")
        assert got.n_keys == len(vals) + 1
        k.query(aggs=[("i", SUM)], sids=[202], ctx="hash")


# ------------------------------------------------------------------ the cap and the other limits
def limit_series():
    c1 = lambda n: (np.ones(n, np.int64), np.zeros(n, bool))   # noqa: E731
    ss = [mk(40, _runs([b"a%02d" % i for i in range(64)], 1)), mk(41, [b"extra"] * 10), mk(42, [b"solo"] * 7),
          mk(43, _runs([b"c%03d" % i for i in range(128)], 1)), mk(44, _runs([b"c%03d" % i for i in range(128, 256)], 1)),
          mk(45, _runs([b"r%02d" % i for i in range(12)], 2)), mk(46, [b"p%03d" % i for i in range(257)]),
          mk(47, [b"ok", b"y" * 65, b"ok"])]
    for s in ss:
        s.tags["c"] = c1(s.n)
    v, nl = ss[5].tags["c"]
    v[:] = [1 if x in (b"r00", b"r01", b"r02") else 0 for x in ss[5].tags[KT]]
    return ss


@gpu
def test_cap_and_limits(bydb, gpu_ctx):
    """max_values 0 (64), 1 and 256 at and one past the cap -> ENOMEM; 257 -> EINVAL; the cap counts the values of the selected
    blocks, not the surviving keys; a 257-value (plain) page and a 65-byte value -> ENOTSUP; 7 user predicates answer, 8 give
    ENOTSUP, 9 EINVAL; overlapping parts -> ENOTSUP unless the range is empty.  The context answers a plain query after each."""
    ss = limit_series()
    P, E = O.Pred, bydb.capi
    with KScan(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        assert k.query(sids=[40], max_values=0, ctx="cap64").n_keys == 64
        k.fails(E.ENOMEM, sids=[40, 41], max_values=0)
        assert k.query(sids=[42], max_values=1, ctx="cap1").n_keys == 1
        k.fails(E.ENOMEM, sids=[41, 42], max_values=1)
        assert k.query(aggs=[("i", SUM), ("f", MIN)], sids=[43, 44], max_values=256, ctx="cap256").n_keys == 256
        k.fails(E.ENOMEM, sids=[41, 43, 44], max_values=256)
        k.fails(E.EINVAL, sids=[40], max_values=257)
        k.fails(E.ENOMEM, sids=[45], preds=[P(FAM, "c", O.OP_EQ, 1)], max_values=8)
        got = k.query(sids=[45], preds=[P(FAM, "c", O.OP_EQ, 1)], max_values=12, ctx="cap counts selected blocks")
        assert got.n_keys == 12 and sorted(set(got.key)) == [b"r00", b"r01", b"r02"]
        k.fails(E.ENOTSUP, sids=[46])
        k.fails(E.ENOTSUP, sids=[47])
        seven = [P(FAM, "c", O.OP_GE, -5), P(FAM, "c", O.OP_LE, 5), P(FAM, "c", O.OP_NE, 9), P(FAM, "c", O.OP_GT, -9),
                 P(FAM, "c", O.OP_LT, 9), P(FAM, "c", O.OP_EQ, 1), P(FAM, "nope", O.OP_NE, b"x")]
        k.query(sids=[40, 45], preds=seven, ctx="seven predicates")
        k.fails(E.ENOTSUP, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)])
        k.fails(E.EINVAL, sids=[40], preds=seven + [P(FAM, "c", O.OP_GE, 0)] * 2)
    over = [mk(40, [b"a00", b"late"] * 20, row0=30)]
    over[0].tags["c"] = (np.ones(40, np.int64), np.zeros(40, bool))
    with KScan(bydb, gpu_ctx, [(build_keyed(ss), ss), (build_keyed(over, 2), over)]) as k:
        k.fails(E.ENOTSUP, sids=[40])
        oq, q = k.oquery(AGGS, [], T0 + 40 * STEP, T0 + 39 * STEP, None, [40])
        got = gpu_ctx.scan_agg_keyed(q, FAM, KT, 0)
        assert got.rows.size == 0 and got.key == [] and got.n_keys == 0
        assert O.run_query(dataclasses.replace(oq, group_key=(FAM, KT))).rows.size == 0


# ------------------------------------------------------------------ insertion order
EDGE_ROWS = [0, 31, 32, 33, 8191, 8192]


def order_series():
    """sid 10: 8193 rows, value e<r> first at row r of EDGE_ROWS, "bg" elsewhere; sid 11: two blocks, values first in the
    second one; sid 12: "A" at rows 5 and 20, "B" at row 10 (a cut or a predicate on row 5 reverses them); sid 13 shows only
    "bg"; sid 14 repeats values of sid 10 in another order.  Tags c (int64, -1 at row 5 of sid 12), s (dictionary, "n" there)
    and dod (a DoD page)."""
    rng = np.random.default_rng(0x0D)
    k10 = [b"bg"] * 8193
    for r in EDGE_ROWS:
        k10[r] = b"e%d" % r
    k11 = [b"bg"] * (BLOCK + 40)
    k11[BLOCK - 1] = b"t1"
    k11[BLOCK] = b"t2"
    k11[BLOCK + 33] = b"t3"
    k11[BLOCK + 7] = b"t4"
    k11[BLOCK + 8] = b"t1"
    k12 = [b"bg"] * 64
    k12[5] = k12[20] = b"A"
    k12[10] = b"B"
    k12[40] = None
    k14 = [b"e8192", b"bg", b"e31", b"B", b"e0"] * 8
    ss = [mk(10, k10), mk(11, k11), mk(12, k12), mk(13, [b"bg"] * 50), mk(14, k14, row0=3)]
    for s in ss:
        c = np.ones(s.n, np.int64)
        if s.sid == 12:
            c[5] = -1
        s.tags["c"] = (c, np.zeros(s.n, bool))
        s.tags["s"] = [b"n" if (s.sid == 12 and r == 5) else b"y" for r in range(s.n)]
        s.tags["dod"] = ((100 + np.concatenate([[0], np.cumsum(rng.integers(1, 9, s.n - 1))])).astype(np.int64), np.zeros(s.n, bool))
    return ss


def ab_parts():
    """two parts that follow each other in time: values n0 / n1 first show in the second (sid 21 shows n0 earlier than sid 20)"""
    a = [mk(20, [b"a", b"b"] * 50), mk(21, [b"a"] * 100)]
    kb20 = [b"b"] * 100
    kb20[50], kb20[60] = b"n1", b"n0"
    kb21 = [b"a"] * 100
    kb21[20] = b"n0"
    b = [mk(20, kb20, row0=100), mk(21, kb21, row0=100)]
    return a, b


@gpu
def test_insertion_order(bydb, gpu_ctx):
    """First surviving rows at rows 0, 31, 32, 33, 8191, 8192 of an 8193-row block (31 / 32 adjacent across a mask word), in
    the second block of a series, behind a tmin cut, an int64 and a dictionary predicate on other tags and a DoD predicate next
    to the key; series-group ids out of first-appearance order, a group that never shows most values; parts in both orders."""
    ss = order_series()
    P = O.Pred
    groups = {10: 2, 11: 0, 12: 3, 13: 1, 14: 2}
    with KScan(bydb, gpu_ctx, [(build_keyed(ss), ss)], groups=groups) as k:
        got = k.query(ctx="order")
        assert got.key[:7] == [b"e0", b"bg", b"e31", b"e32", b"e33", b"e8191", b"e8192"]
        k.query(tmin=T0 + 6 * STEP, ctx="order")
        k.query(tmin=T0 + 33 * STEP, tmax=T0 + (BLOCK + 20) * STEP, ctx="order")
        k.query(preds=[P(FAM, "c", O.OP_GE, 0)], ctx="order")
        k.query(preds=[P(FAM, "s", O.OP_NE, b"n")], ctx="order")
        k.query(preds=[P(FAM, "dod", O.OP_GE, 150)], ctx="order: DoD predicate")
        k.query(aggs=[("i", COUNT)], preds=[P(FAM, "dod", O.OP_LT, 20000), P(FAM, "s", O.OP_EQ, b"y")], ctx="order")
        k.query(sids=[12, 13], ctx="order")
    a, b = ab_parts()
    with KScan(bydb, gpu_ctx, [(build_keyed(a), a), (build_keyed(b), b)], groups={20: 0, 21: 0}) as k:
        for order in ([0, 1], [1, 0]):
            got = k.query(order=order, ctx=f"parts {order}")
            assert got.key == [b"a", b"b", b"n1", b"n0"]
            k.query(order=order, tmin=T0 + 120 * STEP, ctx=f"parts {order}")


# ------------------------------------------------------------------ composite table size and Top-N
def big_series():
    """33 series x 256 values (2 rows each, 3 for every 5th value in every 3rd series), values rotated per series;
    32 series x 32 values (1024 (series, rank) slots) and 41 series x 25 values (1025)"""
    pool = [b"g%03d" % i for i in range(256)]
    ss = []
    for j in range(33):
        vals = pool[j * 7 % 256:] + pool[:j * 7 % 256]
        ss.append(mk(500 + j, [v for i, v in enumerate(vals) for _ in range(3 if (j % 3 == 0 and i % 5 == 0) else 2)]))
    for j in range(32):
        ss.append(mk(600 + j, _runs([b"q%02d" % ((i + j) % 32) for i in range(32)], 1)))
    for j in range(41):
        ss.append(mk(700 + j, _runs([b"u%02d" % ((i * 3 + j) % 25) for i in range(25)], 1)))
    return ss


@gpu
def test_composite_table_size_and_top_n(bydb, gpu_ctx):
    """V x G = 256 x 31 / 32 / 33 composite groups (7936, 8192, 8448: finalisation leaves the single-CTA path above 8192);
    NS x V = 1024 and 1025 (series, rank) slots; Top-N 1 / 2048 / all over COUNT (mass ties), an int64 MAX and a float MAX."""
    ss = big_series()
    with KScan(bydb, gpu_ctx, [(build_keyed(ss), ss)]) as k:
        for G in (31, 32, 33):
            got = k.query(aggs=[("i", SUM), ("i", COUNT), ("f", MAX)], sids=range(500, 500 + G), ctx=f"V x G 256 x {G}")
            assert len(got.key) == 256 * G
        k.query(sids=range(600, 632), ctx="1024 slots")
        k.query(sids=range(700, 741), ctx="1025 slots")
        aggs = [("i", COUNT), ("i", MAX), ("f", MAX)]
        for n in (1, 2048):
            for a in range(3):
                for desc in (True, False):
                    k.query(aggs=aggs, sids=range(500, 533), top=(n, a, desc), ctx="top")
        for a, desc in ((0, True), (1, False), (2, True)):   # every composite group: 1024 and 1025 of them
            k.query(aggs=aggs, sids=range(600, 632), top=(2048, a, desc), ctx="top over all groups")
            k.query(aggs=aggs, sids=range(700, 741), top=(2048, a, not desc), ctx="top over all groups")


# ------------------------------------------------------------------ other lanes under the passes
def lane_series():
    """fields: i (narrow delta), f (decimal), rn (raw cells with nulls in some series), dd (DoD), w (a wide delta in some
    series), fx (non-decimal floats: a raw page without nulls); keys k0..k2, nil and "" unevenly spread; a binary tag bk;
    an int64 tag dod (a DoD page)"""
    rng = np.random.default_rng(0x1A5E)
    ss = []
    for j, n in enumerate([40, 100, 33, BLOCK + 100, 257, 64]):
        sid = 800 + j
        r = np.arange(n)
        keys = [[b"k0", b"k1", None, b"k2", b""][(x // (3 + j)) % (2 + j % 4)] for x in range(n)]
        fl = std_fields(sid, n)
        rn = 5 + np.cumsum(rng.integers(-3, 4, n))
        rn_null = (r % 7 == 3) if j % 2 == 0 else np.zeros(n, bool)
        dd = (100 + np.cumsum(rng.integers(1, 9, n))).astype(np.int64)
        w = 7 + np.cumsum(rng.integers(-60, 60, n))
        if j in (1, 3):
            w[n // 2:] += WIDE
        fx = rng.uniform(-100, 100, n) if j != 2 else np.round(rng.uniform(-100, 100, n), 2)
        fl.update(rn=(I, rn, rn_null), dd=(I, dd, None), w=(I, w, None), fx=(F, fx, None))
        bk = [[b"\x00\xff", b"\x00", None, b"\xff" * 64][(x + j) % 4] for x in range(n)]
        dod = (np.cumsum(rng.integers(1, 90, n)) - 20 * n).astype(np.int64)
        ss.append(mk(sid, keys, fields=fl, tags={"bk": bk, "dod": (dod, np.zeros(n, bool))}))
    return ss


@gpu
def test_lanes_under_the_passes(bydb, gpu_ctx):
    """Raw-cell field pages with nulls, non-decimal floats, DoD and wide delta pages: a pass defers a block only when its value
    has a surviving row there; a DoD int64 predicate defers every pass with a row in range; a VT_BINARY key tag."""
    ss = lane_series()
    P = O.Pred
    aggs = [("i", SUM), ("rn", SUM), ("rn", COUNT), ("dd", MAX), ("w", SUM), ("w", MIN), ("fx", MAX), ("fx", SUM), ("f", MEAN)]
    with KScan(bydb, gpu_ctx, [(build_keyed(ss, binary=("bk",)), ss)], groups={s.sid: s.sid % 2 for s in ss}) as k:
        k.query(aggs=aggs, ctx="lanes")
        k.query(aggs=[("rn", COUNT), ("dd", SUM), ("fx", MIN)], ctx="lanes")
        k.query(aggs=[("w", SUM), ("rn", MEAN)], tmin=T0 + 35 * STEP, tmax=T0 + 8300 * STEP, ctx="lanes")
        k.query(aggs=aggs, preds=[P(FAM, "dod", O.OP_GE, -3000)], ctx="lanes: DoD predicate")
        k.query(aggs=aggs, key="bk", ctx="lanes: binary key")
        k.query(aggs=[("i", SUM), ("fx", MAX)], key="nosuchtag", ctx="lanes: absent tag")


# ------------------------------------------------------------------ the layout claims above, on the CPU
def test_keyed_case_layouts():
    """Each shape the GPU cases claim, through the oracle's codecs and a Python FNV-1a, so a drifting helper fails here."""
    blocks = shape_blocks()
    combos = set()
    for name, want in SHAPE_EXPECT.items():
        cells = blocks[name]
        assert str_tag_class(cells) == "dict" and dict_layout(cells) == want, f"shape_blocks()[{name!r}]: {dict_layout(cells)}"
        combos.add(want[2:])
    assert combos == {(False, False), (False, True), (True, False), (True, True)}
    for k in SHAPE_COUNTS:
        assert len(set(blocks[f"values{k}"])) == k
    pool = shape_pool()
    assert {0, 1, 63, 64} <= {len(v) for v in pool} and b"\x00" in pool and any(v and v[0] >= 0x80 for v in pool)
    assert {b"a", b"a\x00", b"ab", b"ab\x00"} <= set(pool)
    ne = blocks["nil_empty"]
    assert None in ne and b"" in ne
    # the hash sets
    wrap, with_empty, same = hash_sets()
    assert len(set(wrap)) == 40 and {fnv_slot(v) for v in wrap} == {1023}
    assert {fnv_slot(v) for v in with_empty} == {fnv_slot(b"")} and len({len(v) for v in with_empty}) == len(with_empty)
    assert len({fnv_slot(v) for v in same}) == 1 and len({len(v) for v in same}) == len(same) and max(map(len, same)) == 64
    # the limits: 257 values give a plain page, a 65-byte value, the cap sets
    ls = limit_series()
    assert str_tag_class(ls[6].tags[KT]) == "plain" and len(set(ls[6].tags[KT])) == 257
    assert max(map(len, ls[7].tags[KT])) == 65
    assert [len(set(s.tags[KT])) for s in ls[:6]] == [64, 1, 1, 128, 128, 12]
    assert not set(ls[3].tags[KT]) & set(ls[4].tags[KT]) and not set(ls[1].tags[KT]) & set(ls[3].tags[KT] + ls[4].tags[KT])
    # first appearances
    os_ = order_series()
    k10 = os_[0].tags[KT]
    assert os_[0].n == BLOCK and [k10.index(b"e%d" % r) for r in EDGE_ROWS] == EDGE_ROWS and k10.index(b"bg") == 1
    k11 = os_[1].tags[KT]
    assert os_[1].chunks() == [(0, BLOCK), (BLOCK, BLOCK + 40)] and k11.index(b"t1") == BLOCK - 1
    assert min(k11.index(v) for v in (b"t2", b"t3", b"t4")) >= BLOCK
    k12 = os_[2].tags[KT]
    assert k12.index(b"A") == 5 < k12.index(b"B") == 10 < k12.index(b"A", 6) == 20
    assert os_[2].tags["c"][0][5] == -1 and os_[2].tags["s"][5] == b"n" and (os_[2].tags["c"][0] == 1).sum() == 63
    assert {s.kind(("t", "dod"), lo, hi)[0] for s in os_ for lo, hi in s.chunks()} == {"dod"}
    assert [len(set(s.tags[KT])) for s in big_series()] == [256] * 33 + [32] * 32 + [25] * 41
    a, b = ab_parts()
    assert a[0].ts[-1] < b[0].ts[0] and b[0].tags[KT].index(b"n1") < b[0].tags[KT].index(b"n0")
    # page kinds of the lane series
    kinds = {f: {s.kind(("f", f), lo, hi) for s in lane_series() for lo, hi in s.chunks()} for f in ("rn", "dd", "w", "fx")}
    assert ("raw", True) in kinds["rn"] and ("delta", False) in kinds["rn"]
    assert kinds["dd"] == {("dod", False)} and ("wide", False) in kinds["w"] and ("delta", False) in kinds["w"]
    assert ("raw", False) in kinds["fx"] and len(kinds["fx"]) > 1
    assert {s.kind(("t", "dod"), lo, hi)[0] for s in lane_series() for lo, hi in s.chunks()} == {"dod"}
    assert all(str_tag_class(s.tags["bk"][lo:hi]) == "dict" for s in lane_series() for lo, hi in s.chunks())


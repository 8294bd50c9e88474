"""The numeric fallback pages, from admission to the aggregate, against the oracle and an independent model.

The writer turns every int64 / float64 block with a null cell, or with floats that are not short decimals, into
[EncodeTypePlain][encodeDefault page] (column.go:147-153,203-208).  The inner page is a dictionary when the block has <= 256
distinct cells (a value table, then bit-packed (value, run) pairs) and a plain bytes block otherwise; its lens and data blocks
are zstd frames from 128 B on.  At admission classify_pages_kernel / unpack_pages_kernel rewrite each such page into a
raw-cell page [0x40][has_nulls][6 pad][n x u64][n x u8 valid] (unpack_kernels.cu): lane 0 inflates, the warp expands, runs of
more than 64 rows are spread over the warp, and the row offset carries from one 32-run window to the next.  The fast lane hands
every block whose query reads such a page to the slow lane (reason bit 4 << field), where agg_raw_page folds the cells in
double from the function.go MIN/MAX sentinels +-DBL_MAX.  COUNT alone on a raw-cell page without nulls is the row count, so
the express and fast lanes answer it without reading the page.

Every query is checked three ways:
  - against the oracle: group ids and their order, rows, int64 results, float MIN/MAX bit for bit, float SUM/MEAN within
    1e-9 * sum|x| (NaN and +-Inf exactly, which assert_parity cannot compare);
  - against `model`, a plain Python fold over the generated rows (in range, not masked, not shadowed; nulls skipped): int64 SUM
    mod 2^64, MEAN the wrapped sum over the count truncated toward zero, MIN/MAX from the sentinels with strict < / > (so NaN
    never enters), float SUM by math.fsum, and the MEAN quirks of DESIGN 4.5;
  - the lane of every block against `lane_model`, which derives it from the page kind of each block (`page_kind`, through
    the oracle's codecs).  After each registration part_info must report every fallback page unpacked and none left.
Each series is one group unless a case says otherwise, so one query checks every block of a part.

The zero of a MIN/MAX over a group that holds both +0.0 and -0.0 is compared without its sign (DESIGN 6); a group of -0.0
alone must return -0.0.  A plain inner page holds more than 256 distinct cells, hence at least 256 non-null ones, so its lens
and data blocks are always zstd frames: the short-block forms only occur in dictionaries, where the layout test pins them.
"""
import math
import struct
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, build_part, to_gpu_query
from tests.test_gpu_lanes import _varint_lengths
from tests.test_gpu_masks import I64_MAX, I64_MIN, _cblock, _varuint, dict_layout, host_images, str_tag_class, wrap64
from tests.test_oracle_model_sweep import OPS

gpu = pytest.mark.gpu

FAM = "default"
BLOCK = 8193                      # the writer cuts a series into blocks of this many rows
DBL_MAX = float(np.finfo(np.float64).max)
INF, NAN = math.inf, math.nan
PNAN = struct.unpack("<d", struct.pack("<Q", 0x7FF8_0000_0000_0ABC))[0]    # a quiet NaN with a payload
NNAN = struct.unpack("<d", struct.pack("<Q", 0xFFF8_0000_0000_0001))[0]    # ... and with the sign bit set
DENORM = 5e-324
I, F = O.VT_INT64, O.VT_FLOAT64
SUM, COUNT, MIN, MAX, MEAN = O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN
ALL10 = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("i", MEAN), ("f", SUM), ("f", COUNT), ("f", MIN), ("f", MAX), ("f", MEAN)]
EXPRESS_SHAPED = [[("i", COUNT), ("f", COUNT)], [("f", COUNT)], [("f", SUM), ("f", COUNT)], [("i", SUM), ("f", COUNT)]]
_pid = [90_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# ------------------------------------------------------------------ pages, through the oracle's codecs
def cell_bytes(vt, vals, nulls):
    """-> the 8-byte cells column.go stores (int64 order-preserving, float64 IEEE big endian), None for a null"""
    if vt == I:
        raw = (np.asarray(vals, np.int64).view(np.uint64) ^ np.uint64(1 << 63)).astype(">u8").tobytes()
    else:
        raw = np.asarray(vals, np.float64).astype(">f8").tobytes()
    return [None if nl else raw[8 * k:8 * k + 8] for k, nl in enumerate(nulls.tolist())]


def page_kind(vt, vals, nulls):
    """-> (kind, has_nulls) of one block's numeric page: 'raw' (a fallback page: raw cells after admission), 'delta' (every
    varint <= 3 bytes), 'wide' (a delta or DoD page with a varint of 4+ bytes), 'const', 'delta_const' or 'dod'."""
    if nulls.any():
        return "raw", True
    m = vals
    if vt == F:
        try:
            m, _ = O.float64_to_decimal_list(vals)
        except ValueError:
            return "raw", False
    body, enc, _ = O.int64_list_encode(m)
    if enc in (O.ENC_DELTA, O.ENC_DELTA_OF_DELTA) and max(_varint_lengths(body)) > 3:
        return "wide", False   # the fast lane's decoders hand the page to the general one
    return {O.ENC_CONST: "const", O.ENC_DELTA_CONST: "delta_const", O.ENC_DELTA: "delta", O.ENC_DELTA_OF_DELTA: "dod"}[enc], False


def fallback_layout(vt, vals, nulls):
    """Layout of one block's fallback page, or None when the writer makes a regular page: inner kind (9 plain / 10 dictionary),
    lens / data block zstd?, non-null cells in the data block; for a dictionary also the value count, its nil entry ('first',
    'last', 'inner' or None), the packed width, the runs, the longest run and the index of the first run longer than 64."""
    page = O.column_encode(vt, cell_bytes(vt, vals, nulls))
    if page[0] != O.ENC_PLAIN:
        return None
    L = dict(inner=page[1])
    i = 2
    if page[1] == O.ENC_DICTIONARY:
        nv, i = _varuint(page, i)
    lens, lz, i = _cblock(page, i)
    data, dz, i = _cblock(page, i)
    L.update(lens_zstd=lz, data_zstd=dz, data_cells=len(data) // 8)
    if page[1] == O.ENC_DICTIONARY:
        w = 1 << lens[0]
        ls = [int.from_bytes(lens[1 + k * w:1 + (k + 1) * w], "big") for k in range(nv)]
        nil = [k for k, x in enumerate(ls) if x == 0]
        nrle, width = int.from_bytes(page[i:i + 4], "big"), page[i + 4]
        bits = page[i + 5:]
        x, tot = int.from_bytes(bits, "big"), 8 * len(bits)
        f = [(x >> (tot - (k + 1) * width)) & ((1 << width) - 1) for k in range(nrle)]
        runs = f[1::2]
        L.update(n_values=nv, width=width, n_runs=len(runs), longest=max(runs),
                 nil=None if not nil else "first" if nil[0] == 0 else "last" if nil[0] == nv - 1 else "inner",
                 first_long=next((r for r, c in enumerate(runs) if c > 64), None))
    return L


# ------------------------------------------------------------------ series, the model and the lane model
class Series:
    """One series: rows row0.. of the timestamp grid, numeric fields {name: (vt, values, nulls)} and tags {name: (values,
    nulls)} (int64) or {name: [bytes]} (string).  The writer cuts it into blocks of BLOCK rows (`chunks`)."""

    def __init__(self, sid, fields, tags=None, row0=0, name=""):
        self.sid, self.name = sid, name
        self.fields = {}
        for k, (vt, v, nl) in fields.items():
            v = np.asarray(v, np.int64 if vt == I else np.float64)
            self.fields[k] = (vt, v, np.zeros(v.size, bool) if nl is None else np.asarray(nl, bool))
        self.n = next(iter(self.fields.values()))[1].size
        self.tags = tags or {}
        self.ts = T0 + (row0 + np.arange(self.n, dtype=np.int64)) * STEP
        self.alive = np.ones(self.n, bool)    # rows no newer version shadows
        self._cache = {}

    def chunks(self):
        return [(lo, min(lo + BLOCK, self.n)) for lo in range(0, self.n, BLOCK)]

    def kind(self, key, lo, hi):
        """('f', field) -> page_kind of the block rows lo..hi; ('t', tag) -> page_kind of an int64 tag, or ('dict' / 'plain',
        a zstd block?) of a string tag"""
        if (key, lo) not in self._cache:
            src, name = key
            if src == "f":
                vt, v, nl = self.fields[name]
                k = page_kind(vt, v[lo:hi], nl[lo:hi])
            elif isinstance(self.tags[name], tuple):
                v, nl = self.tags[name]
                k = page_kind(I, v[lo:hi], nl[lo:hi])
            else:
                cells = self.tags[name][lo:hi]
                cls = str_tag_class(cells)
                k = (cls, cls == "plain" or any(dict_layout(cells)[2:]))
            self._cache[(key, lo)] = k
        return self._cache[(key, lo)]

    def fallback_pages(self):
        """pages classify_pages_kernel rewrites: numeric Plain pages and string pages with a zstd block"""
        n = 0
        for lo, hi in self.chunks():
            n += sum(self.kind(("f", f), lo, hi)[0] == "raw" for f in self.fields)
            for t, cells in self.tags.items():
                k = self.kind(("t", t), lo, hi)
                n += k[0] == "raw" if isinstance(cells, tuple) else k[1]
        return n

    def passes(self, p):
        """rows of the series the predicate keeps (nil passes only NE; int64 signed, bytes unsigned lexicographic)"""
        key = (p.tag, p.op, p.value)
        if key not in self._cache:
            tag = self.tags[p.tag]
            if isinstance(tag, tuple):
                v, nl = tag
                have, cmp = ~nl, (v > p.value).astype(np.int8) - (v < p.value).astype(np.int8)
            else:
                have = np.array([x is not None for x in tag])
                cmp = np.array([0 if x is None else (x > p.value) - (x < p.value) for x in tag], dtype=np.int8)
            ok = np.zeros(self.n, bool)
            for h in (False, True):
                for c in (-1, 0, 1):
                    ok[(have == h) & (cmp == c)] = OPS[p.op](h, c)
            self._cache[key] = ok
        return self._cache[key]


def build(series, version=1):
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
            cols.append((name, O.VT_STR, [x for s in series for x in s.tags[name]], None))
    return build_part(sids, np.concatenate([s.ts for s in series]), np.full(sids.size, version, np.int64), fields,
                      [(FAM, cols)] if cols else [])


def fsum_model(x):
    if x.size == 0:
        return 0.0
    if np.isnan(x).any() or ((x == INF).any() and (x == -INF).any()):
        return NAN
    if np.isinf(x).any():
        return float(x[np.isinf(x)][0])
    try:
        return math.fsum(x.tolist())
    except OverflowError:   # the cases build overflows whose sign and infinity do not depend on the order of the terms
        return INF if sum(Fraction(v) for v in x.tolist()) > 0 else -INF


def fold(vt, fn, x):
    """one aggregate over the non-null values of a group (aggregation.go:290-312, function.go)"""
    n = x.size
    if fn == COUNT:
        return n
    if vt == I:
        if fn in (SUM, MEAN):
            s = wrap64(sum(x.tolist()))
            if fn == SUM:
                return s
            if n == 0:
                return 0
            q = abs(s) // n * (1 if s >= 0 else -1)
            return 1 if q < 1 else q
        if n == 0:
            return I64_MAX if fn == MIN else I64_MIN
        return int(x.min()) if fn == MIN else int(x.max())
    if fn in (SUM, MEAN):
        s = fsum_model(x)
        if fn == SUM:
            return s
        if n == 0:
            return 0.0
        v = s / n
        return 1.0 if v < 1 else v
    y = x[~np.isnan(x)]
    y = y[y < DBL_MAX] if fn == MIN else y[y > -DBL_MAX]
    if y.size == 0:
        return DBL_MAX if fn == MIN else -DBL_MAX
    return float(y.min()) if fn == MIN else float(y.max())


def lane_model(series, aggs, preds, tmin, tmax, overlap):
    """(express-lane blocks, slow-lane blocks, slow_lane_reasons) of one query.
    express lane (no predicates, no overlapping parts, no MIN/MAX): a block wholly in range whose every field is read as a
    narrow delta page or, COUNT alone, is anything but a raw-cell page with nulls.  Everything else goes to the fast lane,
    which defers a block to the slow lane for a raw-cell, DoD or wide tag page under a predicate (reason 2), or else, when rows
    are left, for the first field (in query order) whose page is raw-cell and read (SUM / MEAN / MIN / MAX, or COUNT with
    nulls), or wide and decoded (reason 4 << field): it stops at the first deferral, so a block carries one reason bit."""
    fields = list(dict.fromkeys(f for f, _ in aggs))
    need = dict.fromkeys(fields, 0)
    for f, fn in aggs:
        need[f] |= 1 if fn in (SUM, MEAN) else 2 if fn in (MIN, MAX) else 0
    express_on = not preds and not overlap and not any(v & 2 for v in need.values())
    ex = slow = reasons = 0
    for s in series:
        act = s.alive & (s.ts >= tmin) & (s.ts <= tmax)
        for p in preds:
            act &= s.passes(p)
        for lo, hi in s.chunks():
            inr = (s.ts[lo:hi] >= tmin) & (s.ts[lo:hi] <= tmax)
            if not inr.any():
                continue
            kinds = [s.kind(("f", f), lo, hi) for f in fields]
            if express_on and inr.all() and all(k != ("raw", True) if need[f] == 0 else k[0] == "delta" for f, k in zip(fields, kinds)):
                ex += 1
                continue
            why = next((2 for p in preds if s.kind(("t", p.tag), lo, hi)[0] in ("raw", "dod", "wide", "plain")), 0)
            if not why and act[lo:hi].any():
                why = next((4 << c for c, (f, (k, nl)) in enumerate(zip(fields, kinds))
                            if (k == "raw" and (need[f] or nl)) or (k == "wide" and need[f])), 0)
            slow += why != 0
            reasons |= why
    return ex, slow, reasons


class Expect:
    def __init__(self, aggs):
        self.rows = 0
        self.vals = [[] for _ in aggs]


def model(series, gid, aggs, preds, tmin, tmax):
    out = {}
    for s in series:
        m = s.alive & (s.ts >= tmin) & (s.ts <= tmax)
        for p in preds:
            m &= s.passes(p)
        e = out.setdefault(gid[s.sid], Expect(aggs))
        e.rows += int(m.sum())
        for a, (f, _) in enumerate(aggs):
            _, v, nl = s.fields[f]
            e.vals[a].append(v[m & ~nl])
    for e in out.values():
        e.x = [np.concatenate(v) for v in e.vals]
        e.val = [fold(series[0].fields[f][0], fn, x) for (f, fn), x in zip(aggs, e.x)]
    return out


def _abs_sum(x):
    try:
        return math.fsum(np.abs(x).tolist())
    except OverflowError:
        return INF


def check(got, want, exp, aggs, ctx, top_n=0):
    """top_n: the result holds the first top_n groups of the oracle's order (which the group-id comparison pins)"""
    assert got.group_id.tolist() == want.group_id.tolist(), f"{ctx}: group ids {got.group_id} vs oracle {want.group_id}"
    assert got.rows.tolist() == want.rows.tolist(), f"{ctx}: rows vs oracle"
    assert got.is_float.tolist() == want.is_float.tolist(), f"{ctx}: output typing"
    got_rows = dict(zip(got.group_id.tolist(), got.rows.tolist()))
    for g, e in exp.items():
        if not top_n or g in got_rows:
            assert got_rows.get(g, 0) == e.rows, f"{ctx}: group {g}: {got_rows.get(g, 0)} rows, model {e.rows}"
    if top_n:
        assert len(got_rows) == min(top_n, sum(e.rows > 0 for e in exp.values())), f"{ctx}: {len(got_rows)} rows of Top-{top_n}"
    for i, g in enumerate(got.group_id.tolist()):
        e = exp[g]
        for a, (f, fn) in enumerate(aggs):
            m, where = e.val[a], f"{ctx}: group {g} agg {a} ({f},{fn})"
            if not want.is_float[a]:
                assert int(got.val_i64[i, a]) == m == int(want.val_i64[i, a]), f"{where}: {got.val_i64[i, a]}, model {m}, oracle {want.val_i64[i, a]}"
                continue
            gv, wv = float(got.val_f64[i, a]), float(want.val_f64[i, a])
            if fn in (MIN, MAX):
                x = e.x[a]
                if m == 0 and (np.signbit(x[x == 0])).any() and (~np.signbit(x[x == 0])).any():
                    assert gv == 0 and wv == 0, f"{where}: {gv!r}, oracle {wv!r}, model a zero"
                else:
                    assert _bits(gv) == _bits(m) == _bits(wv), f"{where}: {gv!r}, model {m!r}, oracle {wv!r} (bit-exact)"
                continue
            tol = 1e-9 * _abs_sum(e.x[a]) / (max(e.x[a].size, 1) if fn == MEAN else 1)
            for other, who in ((m, "model"), (wv, "oracle")):
                if math.isnan(other) or math.isnan(gv):
                    assert math.isnan(other) and math.isnan(gv), f"{where}: {gv!r} vs {who} {other!r}"
                elif math.isinf(other) or math.isinf(gv):
                    assert gv == other, f"{where}: {gv!r} vs {who} {other!r}"
                else:
                    assert abs(gv - other) <= tol, f"{where}: {gv!r} vs {who} {other!r} (tolerance {tol:.3g})"
    assert got.stats.rows_matched == sum(e.rows for e in exp.values()), f"{ctx}: rows_matched {got.stats.rows_matched}"


def _lanes(st):
    return st.blocks_express_lane, st.blocks_slow_lane, st.slow_lane_reasons


class Scan:
    """Parts registered once for many queries; each query is checked against the oracle, the model and the lane model."""

    def __init__(self, bydb, gpu_ctx, parts_series, groups=None):
        self.bydb, self.ctx = bydb, gpu_ctx
        self.parts = [p for p, _ in parts_series]
        self.by_part = [ss for _, ss in parts_series]
        self.series = [s for ss in self.by_part for s in ss]
        self.usid = np.array(sorted({s.sid for s in self.series}), dtype=np.uint64)
        self.gid = groups or {int(sid): g for g, sid in enumerate(self.usid.tolist())}
        self.n_groups = max(self.gid.values()) + 1
        self.handles = []

    def __enter__(self):
        pid = _next_pid()
        for i, (p, ss) in enumerate(zip(self.parts, self.by_part)):
            h = self.ctx.register_part(pid + i, p.files())
            self.handles.append(h)
            info = self.ctx.part_info(h)
            want = sum(s.fallback_pages() for s in ss)
            assert info["fallback_unpacked"] == want and info["fallback_left"] == 0, f"part {i}: {info}, {want} fallback pages"
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def query(self, aggs, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, host=None, graph=False, ctx=""):
        """top: (n, agg, desc); host: None (resident parts), 'pageable' or 'pinned' (bydb_scan_agg_host over the images);
        graph: also replay the query as a prepared graph, which must return the same bits and counters"""
        preds = list(preds)
        groups = np.array([self.gid[int(s)] for s in self.usid.tolist()], dtype=np.int32)
        tn, ta, td = top or (0, 0, True)
        oq = O.Query(self.parts, self.usid, aggs, groups=groups, n_groups=self.n_groups, tmin=tmin, tmax=tmax, preds=preds,
                     top_n=tn, top_agg=ta, top_desc=td)
        ctx = f"{ctx}/{[(f, fn) for f, fn in aggs]}/{[(p.tag, p.op, p.value) for p in preds]}" \
              f"/{(tmin - T0) // STEP if tmin > I64_MIN else '-'}..{(tmax - T0) // STEP if tmax < I64_MAX else '-'}/top{top}"
        if host is None:
            q = to_gpu_query(self.bydb, self.handles, oq)
            got = self.ctx.scan_agg(q)
            if graph:
                g = self.ctx.prepare_graph(q)
                try:
                    for run in range(4):   # run 1 ordinary, run 2 capture, runs 3.. replays
                        r = g.run()
                        assert r.group_id.tolist() == got.group_id.tolist() and r.rows.tolist() == got.rows.tolist(), f"{ctx}: replay {run}"
                        assert r.val_i64.tolist() == got.val_i64.tolist(), f"{ctx}: replay {run}"
                        assert r.val_f64.view(np.uint64).tolist() == got.val_f64.view(np.uint64).tolist(), f"{ctx}: replay {run}"
                        assert _lanes(r.stats) == _lanes(got.stats) and r.stats.rows_matched == got.stats.rows_matched, f"{ctx}: replay {run}"
                finally:
                    g.close()
        else:
            q = to_gpu_query(self.bydb, [], oq)
            q.flags = self.bydb.capi.Q_HOST_ZERO_COPY if host == "pinned" else 0
            got = self.ctx.scan_agg_host(host_images(self.parts, host == "pinned"), q)
        want = O.run_query(oq)
        check(got, want, model(self.series, self.gid, aggs, preds, tmin, tmax), aggs, ctx, tn)
        lanes = lane_model(self.series, aggs, preds, tmin, tmax, len(self.parts) > 1)
        assert _lanes(got.stats) == lanes, f"{ctx}: (express, slow, reasons) {_lanes(got.stats)}, expected {lanes}"
        return got


# ------------------------------------------------------------------ generators
SIZES = [1, 2, 15, 16, 17, 31, 32, 33, 127, 128, 256, 257, 8192, 8193]
PLACES = ["row0", "row31", "row32", "last", "odd", "all_but_one", "all", "none"]
REGION = [b"r0", b"r1", b"r2"]
CODE_VALUES = [None, 7, -3, 12]
CODE_RUNS = [70, 1, 130, 65, 2, 200]


def null_rows(place, n):
    return {"row0": [0], "row31": [31] if n > 31 else None, "row32": [32] if n > 32 else None, "last": [n - 1],
            "odd": list(range(1, n, 2)), "all_but_one": [r for r in range(n) if r != n // 2], "all": list(range(n)),
            "none": []}[place]


def code_tag(n, shift=0):
    """int64 tag cells in long runs over [nil, 7, -3, 12]: a dictionary-inner fallback page (row 0 opens a nil run)"""
    v, r = [], shift
    while len(v) < n:
        v += [CODE_VALUES[r % 4]] * CODE_RUNS[r % len(CODE_RUNS)]
        r += 1
    v = v[:n]
    return np.array([0 if x is None else x for x in v], np.int64), np.array([x is None for x in v])


def row_tags(sid, n):
    return {"region": [REGION[(r * 7 + sid) % 3] for r in range(n)], "code": code_tag(n, sid)}


def noisy_floats(rng, n):
    """16-17 significant digits at mixed exponents and signs: never one decimal exponent for a whole block of 2+ values"""
    return (rng.random(n) * 1e3 + rng.random(n) * 1e-7) * np.where(rng.random(n) < 0.5, -1.0, 1.0) * 10.0 ** rng.integers(-3, 4, n)


def placement_series(seed=0xFA11):
    """{int64, float64} x block sizes x null placements; each series one block with both fields, nulls at the same rows.
    Values are distinct (full-range int64, so sums wrap), so blocks of <= 256 rows get dictionaries and longer ones plain
    pages; 'none' leaves the int64 field a regular page and the float64 field a fallback page without nulls."""
    rng = np.random.default_rng(seed)
    out, sid = [], 1
    for n in SIZES:
        seen = set()
        for place in PLACES:
            rows = null_rows(place, n)
            if rows is None or frozenset(rows) in seen:
                continue
            seen.add(frozenset(rows))
            nl = np.zeros(n, bool)
            nl[rows] = True
            iv = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
            out.append(Series(sid, {"i": (I, iv, nl), "f": (F, noisy_floats(rng, n), nl)}, row_tags(sid, n), name=f"{n}/{place}"))
            sid += 1
    return out


def _tables(rng, k):
    ints = [I64_MIN, I64_MAX, -1, 0, 1] + rng.integers(-(1 << 40), 1 << 40, 300).tolist()
    floats = [5e300, -1e-300, math.pi, -0.1, 2.0 / 3.0] + noisy_floats(rng, 300).tolist()
    return ints[:k], floats[:k]


def dict_cases():
    """name -> ([(table index, run length)], table size, nil entry index or None).  Table entries are numbered in order of
    first appearance, so a nil entry at 0 is the dictionary's first value and at k-1 its last."""
    c = {}
    for k in (1, 2, 16, 17, 126, 127, 255, 256):
        for nil, at in (("first", 0), ("last", k - 1), ("absent", None)):
            c[f"values{k}/nil-{nil}"] = ([(r % k, 1 + r % 3) for r in range(max(2 * k, 8))], k, at)
    for L in (1, 63, 64, 65, 66, 200):
        c[f"runs-of-{L}"] = ([(r % 3, L) for r in range(min(40, max(3, BLOCK // L)))], 3, 1)
    c["run8193/nil"] = ([(0, 8193)], 1, 0)
    c["run8193/value"] = ([(0, 8193)], 1, None)
    c["run8192+1"] = ([(0, 8192), (1, 1)], 2, 1)
    for R in (31, 32, 33, 64, 65):
        c[f"{R}-runs"] = ([(r % 4, 1 + r % 5) for r in range(R)], 4, 2)
    for w in (0, 1):
        for p in range(32):   # one run of 100 rows at lane p of window w (run 32w + p), short runs around it
            c[f"long@{32 * w + p}"] = ([(r % 4, 100 if r == 32 * w + p else 1 + r % 3) for r in range(70)], 4, 3)
    c["long-runs"] = ([(r % 4, 65 + r) for r in range(40)], 4, 0)   # every run longer than 64 over two windows
    return c


def dict_series(seed=0xD1C7):
    rng = np.random.default_rng(seed)
    out = []
    for sid, (name, (runs, k, at)) in enumerate(dict_cases().items(), start=1):
        ti, tf = _tables(rng, k)
        idx = np.array([v for v, c in runs for _ in range(c)])
        nl = idx == (-1 if at is None else at)
        n = idx.size
        out.append(Series(sid, {"i": (I, np.array(ti, np.int64)[idx], nl), "f": (F, np.array(tf)[idx], nl)}, row_tags(sid, n), name=name))
    return out


FLOAT_SPECIALS = {   # name -> the only non-null values of the group
    "qnan": [NAN] * 5, "payload-nan": [PNAN, NNAN, PNAN], "+inf": [INF] * 4, "-inf": [-INF] * 4, "-0": [-0.0] * 4,
    "both-zeros": [-0.0, 0.0, -0.0, 0.0], "+-dblmax": [DBL_MAX, -DBL_MAX], "+-denorm": [DENORM, -DENORM, DENORM],
    "nan+finite": [1.5, NAN, -2.25, 3e10], "+inf+finite": [1.0, INF, -7.5], "-inf+finite": [-INF, 2.0, 1e300],
    "+inf-inf": [INF, -INF, 3.0], "overflow": [0.9e308, 1.0e308, 1.7e308], "-overflow": [-1.7e308, -0.95e308, -0.9e308],
    "dblmax+finite": [DBL_MAX, -DBL_MAX, 1.5, -2.5], "dblmax+3": [3.0, DBL_MAX], "-dblmax-1": [-1.0, -DBL_MAX],
    "-0+1": [-0.0, 1.0], "0-1": [0.0, -1.0], "denorm+1": [DENORM, 1.0], "nan-first": [NAN, -4.0, 4.0],
}
INT_SPECIALS = {
    "min": [I64_MIN] * 3, "max": [I64_MAX] * 3, "-1": [-1] * 5, "0": [0] * 4, "min,max,-1,0": [I64_MIN, I64_MAX, -1, 0],
    "max+1": [I64_MAX, 1], "min-1": [I64_MIN, -1], "max*5": [I64_MAX - 7] * 5, "mean<1": [-9, 3, 4],
}
# groups of two series whose blocks each hold only one special: the reduce must keep the sentinels too
SPECIAL_PAIRS = [("qnan", "-inf"), ("+inf", "-0"), ("-0", "both-zeros"), ("qnan", "+inf")]


def special_series():
    """One series (one block) per special; nulls at row 1 and at the end make every page a fallback page.  The int64 field of
    the same series carries the int64 specials in turn."""
    out, groups = [], {}
    fs, ins = list(FLOAT_SPECIALS.items()), list(INT_SPECIALS.items())

    def cells(vals):
        c = vals[:1] + [None] + vals[1:] + [None]
        return c

    def add(fname, ivals, g):
        fc, ic = cells(FLOAT_SPECIALS[fname]), cells(ivals)
        n = max(len(fc), len(ic))
        fc, ic = fc + [None] * (n - len(fc)), ic + [None] * (n - len(ic))
        sid = len(out) + 1
        out.append(Series(sid, {"i": (I, [0 if x is None else x for x in ic], [x is None for x in ic]),
                                "f": (F, [0.0 if x is None else x for x in fc], [x is None for x in fc])}, row_tags(sid, n), name=fname))
        groups[sid] = g
    for j, (name, _) in enumerate(fs):
        add(name, ins[j % len(ins)][1], j)
    for j, (a, b) in enumerate(SPECIAL_PAIRS):
        add(a, [I64_MAX, 5], len(fs) + j)
        add(b, [I64_MAX, 9], len(fs) + j)
    return out, groups


def mixed_series(seed=0x3113):
    """65 series in two groups (32 and 33 series).  Series 1-8 are three blocks each whose pages alternate between a narrow
    delta page, a Const page and a raw-cell page (with and without nulls); the others are one block of one of those kinds."""
    rng = np.random.default_rng(seed)

    def block(kind, n, is_float):
        if kind == "delta":
            m = 1000 + np.concatenate([[0], np.cumsum(rng.integers(-60, 61, n - 1))])
            return (m / 100.0 if is_float else m), None
        if kind == "const":
            return np.full(n, 12.5 if is_float else -42), None
        nl = np.zeros(n, bool)
        if kind == "raw-nulls":
            nl[::7] = True
        return (noisy_floats(rng, n) if is_float else rng.integers(-(1 << 50), 1 << 50, n)), nl

    kinds = ["delta", "const", "raw-nulls", "raw"]
    out, groups = [], {}
    for sid in range(1, 66):
        if sid <= 8:
            order = ["delta", "const", "raw-nulls" if sid % 2 else "raw"]
            order = order[sid % 3:] + order[:sid % 3]
            plan = [(k, BLOCK if b < 2 else 40 + 37 * sid) for b, k in enumerate(order)]
        else:
            plan = [(kinds[sid % 4], 20 + (sid * 53) % 280)]
        fields = {}
        for name, is_float in (("i", False), ("f", True)):
            vs, ns = [], []
            for kind, n in plan:
                k = "raw-nulls" if kind == "raw" and not is_float else kind   # an int64 page without nulls is a regular page
                v, nl = block(k, n, is_float)
                vs.append(np.asarray(v, np.float64 if is_float else np.int64))
                ns.append(np.zeros(n, bool) if nl is None else nl)
            fields[name] = (F if is_float else I, np.concatenate(vs), np.concatenate(ns))
        n = fields["i"][1].size
        out.append(Series(sid, fields, row_tags(sid, n), name="+".join(k for k, _ in plan)))
        groups[sid] = 0 if sid <= 32 else 1
    return out, groups


def host_series():
    """300 one-block series of regular pages, and a last series of two blocks whose second block alone has a null"""
    rng = np.random.default_rng(0x4057)
    out = []
    for sid in range(1, 301):
        n = 50 + sid % 40
        m = 500 + np.concatenate([[0], np.cumsum(rng.integers(-40, 41, n - 1))])
        out.append(Series(sid, {"i": (I, m, None), "f": (F, m / 100.0, None)}))
    n = BLOCK + 100
    m = 500 + np.concatenate([[0], np.cumsum(rng.integers(-40, 41, n - 1))])
    nl = np.zeros(n, bool)
    nl[BLOCK + 31] = True
    out.append(Series(301, {"i": (I, m, nl), "f": (F, m / 100.0, None)}))
    return out


# ------------------------------------------------------------------ row modes over one part
TIME_CUTS = [(0, 8192), (1, 8192), (31, 8192), (32, 8192), (33, 8192), (0, 0), (0, 31), (0, 32), (0, 33), (31, 31), (32, 255), (33, 8191)]


def run_row_modes(s, ctx, cuts=TIME_CUTS):
    P = O.Pred
    s.query(ALL10, ctx=ctx)
    for aggs in EXPRESS_SHAPED:
        s.query(aggs, ctx=ctx)
    for lo, hi in cuts:
        s.query(ALL10, tmin=T0 + lo * STEP, tmax=T0 + hi * STEP, ctx=ctx)
    s.query([("i", COUNT), ("f", COUNT)], tmin=T0 + 32 * STEP, tmax=T0 + 8192 * STEP, ctx=ctx)
    for preds in ([P(FAM, "region", O.OP_EQ, b"r1")], [P(FAM, "region", O.OP_NE, b"r0")], [P(FAM, "code", O.OP_EQ, 7)],
                  [P(FAM, "code", O.OP_NE, 7)], [P(FAM, "code", O.OP_LT, 0)], [P(FAM, "region", O.OP_NE, b"r2"), P(FAM, "code", O.OP_NE, -3)]):
        s.query(ALL10, preds, ctx=ctx)
        s.query([("f", COUNT), ("i", COUNT)], preds, ctx=ctx)
    s.query(ALL10, [P(FAM, "code", O.OP_NE, 12)], T0 + 31 * STEP, T0 + 8191 * STEP, ctx=ctx)


@gpu
def test_null_placement_matrix(bydb, gpu_ctx):
    """{int64, float64} x block sizes 1 .. 8193 around every short / zstd and dictionary / plain threshold x nulls at rows 0,
    31, 32, count-1, every other row, all but one and every row, plus non-decimal floats without nulls; SUM, COUNT, MIN, MAX,
    MEAN and the express-shaped COUNT queries under every row mode but dedup (test_dedup_shadow_newer_part_fallback)."""
    ss = placement_series()
    with Scan(bydb, gpu_ctx, [(build(ss), ss)]) as s:
        run_row_modes(s, "placement")


@gpu
def test_dictionary_shapes(bydb, gpu_ctx):
    """Numeric dictionaries of 1 .. 256 values with the nil entry first, last or absent; runs of 1, 63 .. 66, 200 and 8193
    rows; 31 .. 65 runs per block; a long run at every lane of the first and second 32-run window; a block of one nil run."""
    ss = dict_series()
    with Scan(bydb, gpu_ctx, [(build(ss), ss)]) as s:
        run_row_modes(s, "dict", cuts=[(0, 8192), (1, 8192), (31, 8192), (32, 63), (33, 8191), (0, 31)])


@gpu
def test_ieee_and_int64_specials(bydb, gpu_ctx):
    """Groups whose only values are NaN (quiet, payload, negative), +-Inf, -0.0, both zeros, +-DBL_MAX, +-5e-324, overflowing
    sums, mixtures with finite values; INT64_MIN / MAX, -1, 0 and wrapping sums; groups of two such series; then Top-N over the
    raw MIN / MAX in both directions, where +-Inf and the +-DBL_MAX sentinels are among the keys (no key is NaN)."""
    ss, groups = special_series()
    with Scan(bydb, gpu_ctx, [(build(ss), ss)], groups) as s:
        s.query(ALL10, ctx="specials")
        for aggs in EXPRESS_SHAPED:
            s.query(aggs, ctx="specials")
        s.query(ALL10, tmin=T0 + 1 * STEP, ctx="specials")
        s.query(ALL10, [O.Pred(FAM, "region", O.OP_NE, b"r1")], ctx="specials")
        aggs = [("f", MIN), ("f", MAX), ("i", MIN), ("i", MAX), ("f", COUNT)]
        for a in range(4):
            for desc in (True, False):
                for n in (1, 5, 13, s.n_groups):
                    s.query(aggs, top=(n, a, desc), ctx="specials-top")


@gpu
def test_mixed_series_and_groups_of_32_33(bydb, gpu_ctx):
    """Series whose blocks alternate narrow delta, Const and raw-cell pages, in groups of 32 and 33 series; the same answers
    from a prepared-graph replay."""
    ss, groups = mixed_series()
    with Scan(bydb, gpu_ctx, [(build(ss), ss)], groups) as s:
        s.query(ALL10, ctx="mixed", graph=True)
        for aggs in EXPRESS_SHAPED + [[("i", SUM), ("i", COUNT)], [("i", SUM), ("f", SUM), ("f", MEAN)]]:
            s.query(aggs, ctx="mixed", graph=True)
        s.query(ALL10, tmin=T0 + 33 * STEP, tmax=T0 + 9000 * STEP, ctx="mixed")
        s.query(ALL10, [O.Pred(FAM, "code", O.OP_NE, 7)], ctx="mixed", graph=True)


@gpu
def test_dedup_shadow_newer_part_fallback(bydb, gpu_ctx):
    """A newer part rewrites rows 20 .. 69 of every series with fallback pages (nulls, non-decimal floats); the older part's
    pages are regular.  The shadow seeds the mask of the older blocks, the newer blocks go to the slow lane."""
    rng = np.random.default_rng(0xDEDE)
    old, new = [], []
    for sid, n in enumerate([33, 70, 128, 257, 8193], start=1):
        m = 700 + np.concatenate([[0], np.cumsum(rng.integers(-50, 51, n - 1))])
        old.append(Series(sid, {"i": (I, m, None), "f": (F, m / 100.0, None)}, row_tags(sid, n)))
        a, e = 20, min(70, n)
        nl = np.zeros(e - a, bool)
        nl[[0, 11, e - a - 1]] = True
        new.append(Series(sid, {"i": (I, rng.integers(I64_MIN, I64_MAX, e - a, dtype=np.int64), nl), "f": (F, noisy_floats(rng, e - a), nl[::-1])},
                          {"region": [REGION[r % 3] for r in range(e - a)], "code": code_tag(e - a, 1)}, row0=a))
        old[-1].alive[a:e] = False
    with Scan(bydb, gpu_ctx, [(build(old, 1), old), (build(new, 2), new)]) as s:
        s.query(ALL10, ctx="dedup")
        for aggs in EXPRESS_SHAPED:
            s.query(aggs, ctx="dedup")
        for lo, hi in [(0, 31), (20, 20), (31, 69), (32, 33), (69, 8192)]:
            s.query(ALL10, tmin=T0 + lo * STEP, tmax=T0 + hi * STEP, ctx="dedup")
        s.query(ALL10, [O.Pred(FAM, "code", O.OP_NE, 7)], ctx="dedup")
        s.query(ALL10, [O.Pred(FAM, "region", O.OP_EQ, b"r2")], ctx="dedup")


@gpu
@pytest.mark.parametrize("host", ["pageable", "pinned"])
def test_cold_host_path_unpacks_for_a_late_fallback_page(bydb, gpu_ctx, host):
    """bydb_scan_agg_host scans the pages as they are and rescans the whole part unpacked when a block reports a fallback
    page.  Here only the last block of the last series has one, so every earlier slice has finished when it is met: the
    answer, rows_matched and the lane counters must count none of them twice."""
    ss = host_series()
    with Scan(bydb, gpu_ctx, [(build(ss), ss)]) as s:
        for aggs in (ALL10, [("i", COUNT), ("f", SUM)], [("i", SUM), ("i", MAX)]):
            s.query(aggs, host=host, ctx=f"host-{host}")
        s.query(ALL10, tmin=T0 + 32 * STEP, host=host, ctx=f"host-{host}")
        s.query([("i", MIN), ("i", MAX)], host=host, ctx=f"host-{host}")


# ------------------------------------------------------------------ the layouts the GPU cases rest on, on the CPU
def _layouts(series):
    out = []
    for s in series:
        for lo, hi in s.chunks():
            for f, (vt, v, nl) in s.fields.items():
                out.append((s.name, f, hi - lo, nl[lo:hi], fallback_layout(vt, v[lo:hi], nl[lo:hi])))
    return out


def test_fallback_case_layouts():
    """Each boundary the GPU cases claim, read back from the pages the oracle's codecs write, so a generator that drifts fails
    here by name instead of quietly losing coverage."""
    # placement: every block with a null is a fallback page, a dictionary up to 256 rows (or <= 256 distinct cells) and plain
    # beyond; the data block flips to zstd at 16 non-null cells; plain pages always have zstd lens and data blocks
    lay = _layouts(placement_series())
    for name, f, n, nl, L in lay:
        if nl.any() or (f == "f" and n >= 15):   # one or two noisy floats may still share a decimal exponent
            assert L is not None, (name, f)
            assert L["inner"] == (O.ENC_DICTIONARY if n - max(int(nl.sum()) - 1, 0) <= 256 else O.ENC_PLAIN), (name, f, L)
            if L["inner"] == O.ENC_PLAIN:
                assert L["lens_zstd"] and L["data_zstd"] and L["data_cells"] >= 256, (name, f, L)
            assert L["data_zstd"] == (8 * L["data_cells"] >= 128), (name, f, L)
        if f == "i" and not nl.any():
            assert L is None, name
    dicts = [L for *_, L in lay if L and L["inner"] == O.ENC_DICTIONARY]
    assert {(L["data_cells"], L["data_zstd"]) for L in dicts} >= {(15, False), (16, True)}
    assert any(L and L["inner"] == O.ENC_PLAIN for *_, L in lay)
    # dictionary shapes
    dl = {(name, f): L for name, f, _, _, L in _layouts(dict_series())}
    D = lambda name, f="f": dl[(name, f)]
    for k in (126, 127, 256):
        assert D(f"values{k}/nil-first")["n_values"] == k and D(f"values{k}/nil-first")["lens_zstd"] == (k >= 127)
    for k in (1, 2, 16, 17, 126, 127, 255, 256):
        assert D(f"values{k}/nil-first", "i")["nil"] == "first" and D(f"values{k}/nil-first", "i")["n_values"] == k
        if k > 1:
            assert D(f"values{k}/nil-last", "i")["nil"] == "last" and D(f"values{k}/nil-absent")["nil"] is None
            assert dl[(f"values{k}/nil-absent", "i")] is None   # an int64 block without nulls is a regular page
    assert (D("values16/nil-last")["data_cells"], D("values16/nil-last")["data_zstd"]) == (15, False)
    assert (D("values17/nil-last")["data_cells"], D("values17/nil-last")["data_zstd"]) == (16, True)
    assert (D("values16/nil-absent")["data_cells"], D("values16/nil-absent")["data_zstd"]) == (16, True)
    one_nil = D("run8193/nil", "i")
    assert one_nil["n_values"] == 1 and one_nil["nil"] == "first" and one_nil["n_runs"] == 1 and one_nil["data_cells"] == 0
    assert D("values1/nil-first")["n_runs"] == 1 and D("values1/nil-first")["data_cells"] == 0
    for L in (1, 63, 64, 65, 66, 200):
        lay = D(f"runs-of-{L}")
        assert lay["longest"] == L and lay["first_long"] == (0 if L > 64 else None), L
    for R in (31, 32, 33, 64, 65):
        assert D(f"{R}-runs")["n_runs"] == R
    for pos in range(64):
        lay = D(f"long@{pos}")
        assert lay["first_long"] == pos and lay["n_runs"] == 70 and lay["longest"] == 100 and lay["width"] == 7, pos
    assert D("long-runs")["first_long"] == 0 and D("long-runs")["n_runs"] == 40
    assert D("runs-of-200")["width"] == 8 and D("values256/nil-absent")["width"] == 8
    assert D("run8192+1")["width"] == 14 and D("run8192+1")["first_long"] == 0 and D("run8192+1")["nil"] == "last"
    assert dl[("run8193/value", "f")] is None   # a single value is a short decimal: a Const page, not a fallback page
    # specials: every page a fallback page with nulls
    ss, groups = special_series()
    for name, f, n, nl, L in _layouts(ss):
        assert L is not None and nl.any(), (name, f)
    assert len(set(groups.values())) == len(FLOAT_SPECIALS) + len(SPECIAL_PAIRS)
    # mixed: the blocks of series 1-8 alternate page kinds; the writer cuts them where `chunks` says
    ss, groups = mixed_series()
    assert build(ss).meta()["blocks_count"] == sum(len(s.chunks()) for s in ss)
    for s in ss[:8]:
        kinds = [s.kind(("f", "i"), lo, hi)[0] for lo, hi in s.chunks()] + [s.kind(("f", "f"), lo, hi)[0] for lo, hi in s.chunks()]
        assert {"delta", "const", "raw"} <= set(kinds), (s.name, kinds)
        assert len(set(kinds[:3])) == 3 or len(set(kinds[3:])) == 3, (s.name, kinds)
    assert sorted(Counter(groups.values()).values()) == [32, 33]
    # the cold path's part: exactly one fallback page, in the last block of the last series
    hs = host_series()
    assert [s.fallback_pages() for s in hs] == [0] * 300 + [1]
    assert [hs[-1].kind(("f", "i"), lo, hi)[0] for lo, hi in hs[-1].chunks()] == ["delta", "raw"]
    # the int64 tag the predicates read: a dictionary-inner fallback page with runs longer than 64 rows
    v, nl = code_tag(8193, 0)
    L = fallback_layout(I, v, nl)
    assert L["inner"] == O.ENC_DICTIONARY and L["longest"] > 64 and L["first_long"] == 0 and L["nil"] == "first"


def test_model_rules():
    """The model's own rules, on known answers: MIN / MAX from the sentinels never take NaN, +Inf is no MIN and -Inf no MAX,
    int64 sums wrap and MEAN truncates the wrapped sum, float MEAN below 1 is 1 (-Inf too), overflow keeps its sign."""
    a = lambda *x: np.array(x, np.float64)
    assert fold(F, MAX, a(NAN, NAN)) == -DBL_MAX and fold(F, MIN, a(NAN)) == DBL_MAX
    assert fold(F, MIN, a(INF, INF)) == DBL_MAX and fold(F, MAX, a(-INF)) == -DBL_MAX
    assert fold(F, MAX, a(INF, 1.0)) == INF and fold(F, MIN, a(-INF, NAN)) == -INF
    assert math.isnan(fold(F, SUM, a(INF, -INF))) and fold(F, SUM, a(0.9e308, 1e308, 1.7e308)) == INF
    assert fold(F, MEAN, a(-INF)) == 1.0 and math.isnan(fold(F, MEAN, a(NAN, 1.0))) and fold(F, MEAN, a()) == 0.0
    assert _bits(fold(F, MIN, a(-0.0, -0.0))) == _bits(-0.0)
    i = lambda *x: np.array(x, np.int64)
    assert fold(I, SUM, i(I64_MAX, 1)) == I64_MIN and fold(I, MEAN, i(I64_MAX, 1)) == 1
    assert fold(I, MEAN, i(-9, 3, 4)) == 1 and fold(I, MEAN, i(7, 8)) == 7 and fold(I, MEAN, i()) == 0
    assert fold(I, MIN, i()) == I64_MAX and fold(I, MAX, i()) == I64_MIN

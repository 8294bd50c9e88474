"""The scan's row-mask stage against the oracle and an independent row count, at the boundaries where it carries state.

Each block in the fast lane gets a row range from its timestamps page, then a row bitmask from the tag predicates, then the
field decoders run under that mask (DESIGN.md 4.2).  The mask comes from one of several paths, chosen by the tag page:

  int64 tag, Const / DeltaConst page                -> first + d*row per lane, in both lanes
  int64 tag, narrow Delta page (varints <= 3 bytes)  -> delta_pred_fast (fast lane)
  int64 tag, DoD / wide Delta / raw-cell page        -> deferred (slow_lane_reasons bit 2): decode_varint_page + CmpCons
  string tag, dictionary page (<= 256 values)        -> apply_dict_pred: match set over the values, bit-packed RLE runs
  string tag, plain page (> 256 values)              -> deferred (bit 2): apply_plain_pred
  tag absent from the block                          -> every cell nil

Every case runs one query through the device and the oracle and checks three things beyond parity:
  - the rows of every group, SUM and COUNT of an int64 `rowid` field (a constant-delta page, so no field decoder can hide a
    wrong mask bit) and rows_matched, against a plain Python model of the predicates over the rows the test generated
    (nil passes only NE; int64 compares signed, bytes unsigned and lexicographically: the OPS table of the oracle sweep);
  - ALL5 on a narrow delta field `v`, so the masked field decoders see the same masks (parity only);
  - the lane of every block: no block in the express lane, and exactly the blocks with a deferred tag page and a row in the
    time range in the slow lane, with reason 2 alone (`tag_lane_model`).
Each series is one block and one group, so one query checks every block of a part.
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_lanes import LIMIT_DELTAS, NARROW3, WIDE, _signed, _varint_lengths
from tests.test_oracle_model_sweep import OPS

gpu = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ALL_OPS = [O.OP_EQ, O.OP_NE, O.OP_LT, O.OP_LE, O.OP_GT, O.OP_GE]
BLOCK_SIZES = [1, 2, 31, 32, 33, 8192, 8193]   # 8193: the longest block the writer cuts
FAM = "default"
AGGS = [("rowid", O.AGG_SUM), ("rowid", O.AGG_COUNT),
        ("v", O.AGG_SUM), ("v", O.AGG_COUNT), ("v", O.AGG_MIN), ("v", O.AGG_MAX), ("v", O.AGG_MEAN)]
DEFERRED = {"dod", "wide", "raw", "plain"}      # tag pages the fast lane hands to the slow lane (reason bit 2)
FAST_CHUNK = 1024                               # bytes of a delta page one fast-lane chunk decodes (32 lanes x 32 B)
_pid = [70_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def wrap64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= (1 << 63) else x


# ------------------------------------------------------------------ page classes, through the oracle's codecs
def int_tag_class(vals):
    """What the writer makes of one block's int64 tag cells: 'raw' (a nil cell: fallback page, raw cells after admission),
    'const', 'delta_const', 'dod', 'delta' (every varint <= 3 bytes) or 'wide' (a delta page with a varint of 4+ bytes)."""
    if any(x is None for x in vals):
        return "raw"
    body, enc, _ = O.int64_list_encode(np.array(vals, dtype=np.int64))
    if enc != O.ENC_DELTA:
        return {O.ENC_CONST: "const", O.ENC_DELTA_CONST: "delta_const", O.ENC_DELTA_OF_DELTA: "dod"}[enc]
    return "wide" if max(_varint_lengths(body)) > 3 else "delta"


def str_tag_class(vals):
    return "dict" if O.dictionary_encode(vals) is not None else "plain"


def _varuint(b, i):
    v = s = 0
    while True:
        x = b[i]
        i += 1
        v |= (x & 0x7f) << s
        s += 7
        if x < 0x80:
            return v, i


def _cblock(b, i):
    """compressBlock at b[i:] -> (payload, zstd?, next offset)"""
    if b[i] == 0:
        n = b[i + 1]
        return b[i + 2:i + 2 + n], False, i + 2 + n
    n, j = _varuint(b, i + 1)
    return O.zstd_decompress(bytes(b[j:j + n])), True, j + n


def dict_layout(vals):
    """-> (value count, packed bit width, lens block is a zstd frame, data block is a zstd frame) of a dictionary page."""
    d = O.dictionary_encode(vals)
    assert d is not None
    nv, i = _varuint(d, 0)
    _, lz, i = _cblock(d, i)
    _, dz, i = _cblock(d, i)
    return nv, d[i + 4], lz, dz


def plain_layout(vals):
    """-> (lens width in bytes, lens block is a zstd frame) of a plain string page."""
    page = O.column_encode(O.VT_STR, vals)
    assert page[0] == O.ENC_PLAIN
    lens, lz, _ = _cblock(page, 1)
    return 1 << lens[0], lz


# ------------------------------------------------------------------ blocks, the row model and the lane model
class Blk:
    """One series = one block: timestamps row0.. of the grid, int64 fields `rowid` (rowid0 + row, a constant-delta page) and
    `v` (a narrow delta page), tag cells {(family, name): list of int / bytes / None}."""

    def __init__(self, sid, tags, row0=0, rowid0=0):
        self.sid, self.tags = sid, tags
        n = self.n = len(next(iter(tags.values())))
        self.ts = T0 + (row0 + np.arange(n, dtype=np.int64)) * STEP
        self.rowid = rowid0 + np.arange(n, dtype=np.int64)
        d = ((np.arange(n - 1, dtype=np.int64) * 37 + sid) % 63 + 1) * np.where(np.arange(n - 1) % 2 == 0, 1, -1)
        self.v = np.concatenate([[1000 + sid], 1000 + sid + np.cumsum(d)]).astype(np.int64)
        self.alive = np.ones(n, dtype=bool)   # rows no newer version shadows
        self.vt = {k: O.VT_INT64 if any(isinstance(x, int) for x in v) else O.VT_STR for k, v in tags.items()}  # build_blocks: the column's
        self._cls, self._cmp = {}, {}

    def tag_class(self, key):
        """page class of a tag in this block, None when the block has no such column"""
        if key not in self.tags:
            return None
        if key not in self._cls:
            vals = self.tags[key]
            self._cls[key] = int_tag_class(vals) if self.vt[key] == O.VT_INT64 else str_tag_class(vals)
        return self._cls[key]

    def _have_cmp(self, key, lit):
        if (key, lit) not in self._cmp:
            vals = self.tags.get(key)
            if vals is None:
                have, cmp = np.zeros(self.n, bool), np.zeros(self.n, np.int8)
            elif isinstance(lit, int):
                have = np.array([x is not None for x in vals])
                a = np.array([0 if x is None else x for x in vals], dtype=np.int64)
                cmp = np.where(have, (a > lit).astype(np.int8) - (a < lit).astype(np.int8), 0)
            else:
                have = np.array([x is not None for x in vals])
                cmp = np.array([0 if x is None else (x > lit) - (x < lit) for x in vals], dtype=np.int8)
            self._cmp[(key, lit)] = (have, cmp)
        return self._cmp[(key, lit)]

    def passes(self, p):
        have, cmp = self._have_cmp((p.family, p.tag), p.value)
        ok = np.zeros(self.n, dtype=bool)
        for h in (False, True):
            for c in (-1, 0, 1):
                ok[(have == h) & (cmp == c)] = OPS[p.op](h, c)
        return ok


def tag_lane_model(blocks, preds, tmin, tmax):
    """Blocks the fast lane hands to the slow lane: a predicate's tag page is DoD, wide delta, raw-cell or plain string, and the
    block has a row in the time range (a block wholly outside it is never scanned, a block without rows in it skips the mask)."""
    return sum(1 for b in blocks if ((b.ts >= tmin) & (b.ts <= tmax)).any()
               and any(b.tag_class((p.family, p.tag)) in DEFERRED for p in preds))


def build_blocks(blocks, version=1):
    keys = list(blocks[0].tags)
    fams = {}
    for fam, name in keys:
        cells = [x for b in blocks for x in b.tags[(fam, name)]]
        vt = O.VT_INT64 if any(isinstance(x, int) for x in cells) else O.VT_STR
        for b in blocks:   # a block of nil cells only takes its column's type
            b.vt[(fam, name)] = vt
        if vt == O.VT_INT64:
            nulls = np.array([x is None for x in cells], dtype=np.uint8)
            col = (name, O.VT_INT64, np.array([0 if x is None else x for x in cells], dtype=np.int64), nulls if nulls.any() else None)
        else:
            col = (name, O.VT_STR, cells, None)
        fams.setdefault(fam, []).append(col)
    sids = np.concatenate([np.full(b.n, b.sid, np.uint64) for b in blocks])
    return build_part(sids, np.concatenate([b.ts for b in blocks]), np.full(sids.size, version, np.int64),
                      [("rowid", O.VT_INT64, np.concatenate([b.rowid for b in blocks]), None),
                       ("v", O.VT_INT64, np.concatenate([b.v for b in blocks]), None)], list(fams.items()))


class Scan:
    """Parts registered once for many queries; each query is checked against the oracle, the row model and the lane model."""

    def __init__(self, bydb, gpu_ctx, parts_blocks):
        self.bydb, self.ctx = bydb, gpu_ctx
        self.parts = [p for p, _ in parts_blocks]
        self.blocks = [b for _, bl in parts_blocks for b in bl]
        self.usid = np.array(sorted({b.sid for b in self.blocks}), dtype=np.uint64)
        self.gid = {int(s): g for g, s in enumerate(self.usid.tolist())}
        self.handles = []

    def __enter__(self):
        pid = _next_pid()
        self.handles = [self.ctx.register_part(pid + i, p.files()) for i, p in enumerate(self.parts)]
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            self.ctx.release_part(h)

    def query(self, preds, tmin=I64_MIN, tmax=I64_MAX, ctx="", host=None):
        """host: None (resident parts), 'pageable' or 'pinned' (bydb_scan_agg_host over the part images)"""
        G = self.usid.size
        oq = O.Query(self.parts, self.usid, AGGS, groups=np.arange(G, dtype=np.int32), n_groups=G, tmin=tmin, tmax=tmax, preds=list(preds))
        if host is None:
            got = self.ctx.scan_agg(to_gpu_query(self.bydb, self.handles, oq))
        else:
            q = to_gpu_query(self.bydb, [], oq)
            q.flags = self.bydb.capi.Q_HOST_ZERO_COPY if host == "pinned" else 0
            got = self.ctx.scan_agg_host(host_images(self.parts, host == "pinned"), q)
        want = O.run_query(oq)
        ctx = f"{ctx}/{[(p.tag, p.op, p.value if not isinstance(p.value, bytes) or len(p.value) < 8 else p.value[:6] + b'..') for p in preds]}" \
              f"/{(tmin - T0) // STEP if tmin > I64_MIN else '-'}..{(tmax - T0) // STEP if tmax < I64_MAX else '-'}"
        assert_parity(got, want, AGGS, ctx)
        rows, rsum = np.zeros(G, np.int64), [0] * G
        for b in self.blocks:
            m = b.alive & (b.ts >= tmin) & (b.ts <= tmax)
            for p in preds:
                m &= b.passes(p)
            g = self.gid[b.sid]
            rows[g] += int(m.sum())
            rsum[g] += int(b.rowid[m].sum())
        got_rows = dict(zip(got.group_id.tolist(), got.rows.tolist()))
        for g in range(G):
            assert got_rows.get(g, 0) == rows[g], f"{ctx}: series {int(self.usid[g])}: {got_rows.get(g, 0)} rows, model {rows[g]}"
        for i, g in enumerate(got.group_id.tolist()):
            assert int(got.val_i64[i, 1]) == rows[g] and int(got.val_i64[i, 0]) == rsum[g], \
                f"{ctx}: series {int(self.usid[g])}: COUNT/SUM(rowid) {got.val_i64[i, 1]}/{got.val_i64[i, 0]}, model {rows[g]}/{rsum[g]}"
        assert got.stats.rows_matched == int(rows.sum()), f"{ctx}: rows_matched {got.stats.rows_matched}, model {int(rows.sum())}"
        slow = tag_lane_model(self.blocks, preds, tmin, tmax)
        st = got.stats
        assert st.blocks_express_lane == 0, f"{ctx}: express-lane blocks {st.blocks_express_lane} under predicates"
        assert st.blocks_slow_lane == slow, f"{ctx}: slow-lane blocks {st.blocks_slow_lane}, expected {slow}"
        assert st.slow_lane_reasons == (2 if slow else 0), f"{ctx}: slow-lane reasons {st.slow_lane_reasons:#x}"
        return got


_pinned_keep = []


def host_images(parts, pinned):
    out = []
    for p in parts:
        files = {k: np.frombuffer(v, dtype=np.uint8) for k, v in p.files().items()}
        if pinned:
            import torch
            pf = {}
            for k, v in files.items():
                t = torch.empty(v.size + 256, dtype=torch.uint8, pin_memory=True)
                t[:v.size].copy_(torch.from_numpy(v.copy()))
                _pinned_keep.append(t)
                pf[k] = t[:v.size].numpy()
            files = pf
        out.append(files)
    return out


# ------------------------------------------------------------------ int64 tag page matrix
INT_KINDS = ["const", "dc_neg", "dc_wrap", "d1", "d2", "d3", "limits", "wrap", "wide", "dod", "raw"]
INT_CLASS = {"const": "const", "dc_neg": "delta_const", "dc_wrap": "delta_const", "d1": "delta", "d2": "delta", "d3": "delta",
             "limits": "delta", "wrap": "delta", "wide": "wide", "dod": "dod", "raw": "raw"}   # of blocks of 3+ rows


def int_tag_values(kind, n, rng):
    """-> list of n int64 tag cells (None = nil) of one block of `kind`."""
    if kind == "const":
        return [-(1 << 40)] * n
    if kind == "dc_neg":
        return [1000 - 7 * r for r in range(n)]
    if kind == "dc_wrap":   # first + d*row passes 2^63 at row 3
        return [wrap64(I64_MAX - 100 + 37 * r) for r in range(n)]
    if kind == "wrap":      # [MAX - a, MIN + b, ...]: 1-byte deltas that wrap the running value at every row
        k = rng.integers(0, 20, n).tolist()
        return [I64_MAX - k[r] if r % 2 == 0 else I64_MIN + k[r] for r in range(n)]
    if kind == "dod":
        return (5000 + np.concatenate([[0], np.cumsum(rng.integers(1, 100, n - 1))])).astype(np.int64).tolist()
    if kind == "wide":
        # narrow deltas, the last one a 4-byte varint; eight 2-byte deltas up front put it in the last 1 KB chunk of long pages
        d = _signed(rng, 0, 63, n - 1)
        d[:min(8, n - 1)] = np.where(np.arange(min(8, n - 1)) % 2 == 0, 100, -100)
        if n >= 2:
            d[-1] = WIDE
    elif kind == "d1" or kind == "raw":
        d = _signed(rng, 0, 63, n - 1)
    elif kind == "d2":
        d = _signed(rng, 64, 8191, n - 1)
    elif kind == "d3":
        d = _signed(rng, 8192, NARROW3, n - 1)
    else:  # "limits"
        d = np.resize(np.array(LIMIT_DELTAS, dtype=np.int64), n - 1)
    v = (500 + np.concatenate([[0], np.cumsum(np.asarray(d, dtype=np.int64))])).astype(np.int64).tolist()
    if kind == "raw":
        v[n // 2] = None
        v[-1] = None
    return v


def int_literals(vals):
    """INT64_MIN, INT64_MAX, min-1, min, rows 0 and 1, the last row, max, max+1 of a block (those inside int64)."""
    have = [x for x in vals if x is not None]
    lits = {I64_MIN, I64_MAX}
    if have:
        mn, mx = min(have), max(have)
        lits |= {mn - 1, mn, mx, mx + 1}
    lits |= {x for x in (vals[0], vals[min(1, len(vals) - 1)], vals[-1]) if x is not None}
    return {x for x in lits if I64_MIN <= x <= I64_MAX}


def int_matrix_blocks(kind, seed=0x3A5C):
    rng = np.random.default_rng(seed + INT_KINDS.index(kind))
    return [Blk(sid, {(FAM, "t"): int_tag_values(kind, n, rng)}) for sid, n in enumerate(BLOCK_SIZES, start=1)]


@gpu
@pytest.mark.parametrize("kind", INT_KINDS)
def test_int64_tag_page_matrix(bydb, gpu_ctx, kind):
    """Every int64 tag page kind x block sizes 1..8193 x six operators x the literals at the block's edges.  Targets the
    arithmetic pages (negative and wrapping steps), delta_pred_fast (1-3 byte deltas, zig-zag limits, a running value that wraps
    at every row), its bail-out after earlier chunks were cleared (wide), and CmpCons in the slow lane (DoD, raw cells)."""
    blocks = int_matrix_blocks(kind)
    lits = sorted(set().union(*(int_literals(b.tags[(FAM, "t")]) for b in blocks)))
    with Scan(bydb, gpu_ctx, [(build_blocks(blocks), blocks)]) as s:
        for lit in lits:
            for op in ALL_OPS:
                s.query([O.Pred(FAM, "t", op, lit)], ctx=f"int/{kind}")


# ------------------------------------------------------------------ a 3- or 4-byte tag varint at every fast-lane boundary
SWEEP_ROWS = 2200
SWEEP_LIT = 10_000_000


def sweep_positions():
    """body bytes 32k +- 40 around lane windows (k 1..3), 1 KB chunk edges (k 31..33) and the 2 KB stage edge (k 63..65); +-40
    covers every 16-byte phase of the TMA window"""
    pos = set()
    for k in (1, 2, 3, 31, 32, 33, 63, 64, 65):
        pos.update(range(max(0, 32 * k - 40), 32 * k + 41))
    return sorted(pos)


def sweep_values(p, width, n=SWEEP_ROWS):
    """Distinct int64 values whose delta page holds 1-byte deltas (+3, -1, ...) but one `width`-byte varint at body byte p;
    the value that varint completes (row p+1) is SWEEP_LIT in every block."""
    d = np.where(np.arange(n - 1) % 2 == 0, 3, -1).astype(np.int64)
    d[p] = WIDE if width == 4 else NARROW3
    first = SWEEP_LIT - int(d[:p + 1].sum())
    return (first + np.concatenate([[0], np.cumsum(d)])).tolist()


@gpu
@pytest.mark.parametrize("width", [3, 4])
def test_tag_varint_at_every_boundary(bydb, gpu_ctx, width):
    """One block per position: EQ / NE / LE / GT against the value the swept varint completes, so a wrong head correction,
    chunk carry or two-word mask clear flips exactly the counted row.  4-byte: every block defers (reason 2) and still matches."""
    blocks = [Blk(i + 1, {(FAM, "t"): sweep_values(p, width)}) for i, p in enumerate(sweep_positions())]
    with Scan(bydb, gpu_ctx, [(build_blocks(blocks), blocks)]) as s:
        for op in (O.OP_EQ, O.OP_NE, O.OP_LE, O.OP_GT):
            got = s.query([O.Pred(FAM, "t", op, SWEEP_LIT)], ctx=f"sweep{width}")
            if op == O.OP_EQ:
                assert got.rows.tolist() == [1] * len(blocks)


# ------------------------------------------------------------------ dictionary and plain string pages
SPECIAL = [None, b"", b"ab", b"abc", b"abd", b"a", b"\x80", b"\xff\x00", b"\xc3\xa9", b"z" * 64, b"z" * 63 + b"y"]
POOL = SPECIAL + [b"v%03d" % i for i in range(300)]
STR_LITS = [b"", b"a", b"ab", b"abb", b"abc", b"abd", b"abcd", b"\x7f", b"\x80", b"\xff", b"z" * 63, b"z" * 64, b"v130", b"p0150"]


def runs(pairs):
    """[(POOL index, run length)] -> cells"""
    return [POOL[v] for v, c in pairs for _ in range(c)]


def _cycle(k, nruns, lens):
    return [(i % k, lens[i % len(lens)]) for i in range(nruns)]


# name -> (cells, expected (value count, bit width) or None)
def str_cases():
    c = {}
    for k in (1, 2, 31, 32, 33, 255, 256):
        c[f"values{k}"] = runs(_cycle(k, max(2 * k, 8), [1, 2, 3]))
    c["runs1"] = runs(_cycle(5, 100, [1]))
    c["runs127-129"] = runs(_cycle(4, 12, [127, 128, 129]))
    c["runs@31-33"] = runs(_cycle(3, 12, [31, 1, 1, 30, 2, 31, 1, 33, 32]))
    c["run8193"] = runs([(3, 8193)])
    c["runs8192+1"] = runs([(2, 8192), (9, 1)])
    c["many_runs"] = runs([(i % 7, 1 + (i * 5) % 17) for i in range(200)])
    c["width3"] = runs(_cycle(8, 30, [1, 2, 3, 4, 5, 6, 7]))
    c["width5"] = runs(_cycle(20, 40, list(range(1, 32))))
    c["width7"] = runs(_cycle(3, 9, [100, 65, 3]))
    c["width9"] = runs([(0, 300), (1, 5), (0, 7)])
    c["width13"] = runs([(0, 5000), (1, 10), (2, 100)])
    c["nil_empty"] = runs([(0, 1), (1, 2), (0, 3), (1, 1), (2, 2), (0, 40), (1, 33)])
    c["high_bytes"] = runs([(6 + i % 3, 1 + i % 5) for i in range(60)] + [(11, 3)])
    c["prefixes"] = runs([(2 + i % 4, 1 + i % 6) for i in range(80)])
    c["long64"] = runs([(9 + i % 2, 1 + i % 40) for i in range(40)] + [(5, 2)])
    c["data>=128"] = runs([(11 + i, 2) for i in range(40)])
    c["values257"] = runs(_cycle(257, 514, [1, 2]))
    plain = [b"p%04d" % i for i in range(320)]
    for r in range(0, 320, 37):
        plain[r] = None
    c["plain"] = plain
    plain_long = [b"p%04d" % i for i in range(400)]
    for r in range(0, 400, 50):
        plain_long[r] = b"z" * 64 + bytes([0x41 + r % 26]) * 236    # 300 bytes: a 2-byte lens width
        plain_long[r + 1] = None
        plain_long[r + 2] = b"ab" + b"\x90" * 298
    c["plain_long"] = plain_long
    return c


STR_EXPECT = {  # name -> (value count, packed width, lens zstd, data zstd) of the dictionary page
    "values1": (1, 4, False, False), "values2": (2, 2, False, False), "values31": (31, 5, False, True),
    "values32": (32, 5, False, True), "values33": (33, 6, False, True), "values255": (255, 8, True, True),
    "values256": (256, 8, True, True), "runs1": (5, 3, False, False), "runs127-129": (4, 8, False, False),
    "runs@31-33": (3, 6, False, False), "run8193": (1, 14, False, False), "runs8192+1": (2, 14, False, False),
    "many_runs": (7, 5, False, False), "width3": (8, 3, False, False), "width5": (20, 5, False, True),
    "width7": (3, 7, False, False), "width9": (2, 9, False, False), "width13": (3, 13, False, False),
    "nil_empty": (3, 6, False, False), "high_bytes": (4, 3, False, False), "prefixes": (4, 3, False, False),
    "long64": (3, 6, False, True), "data>=128": (40, 6, False, True),
}
PLAIN_EXPECT = {"values257": 1, "plain": 1, "plain_long": 2}   # name -> lens width in bytes


@gpu
def test_string_tag_pages(bydb, gpu_ctx):
    """apply_dict_pred over value counts 1..256, runs of 1 / 127..129 / 8193 rows, runs on mask-word edges, odd packed widths,
    nil next to "", bytes >= 0x80, prefix relations, 64-byte values and zstd-inflated blocks; plain pages (257 values, nil cells,
    300-byte cells) in the slow lane.  Literals: empty, prefixes and extensions of values, absent ones, 63 and 64 bytes."""
    cases = str_cases()
    blocks = [Blk(i + 1, {(FAM, "s"): cells}) for i, cells in enumerate(cases.values())]
    with Scan(bydb, gpu_ctx, [(build_blocks(blocks), blocks)]) as s:
        for lit in STR_LITS:
            for op in ALL_OPS:
                s.query([O.Pred(FAM, "s", op, lit)], ctx="str")


# ------------------------------------------------------------------ conjunctions
def conj_blocks():
    """Blocks with every tag page kind side by side: dictionary, plain, narrow delta, DoD, raw cells, constant delta."""
    rng = np.random.default_rng(0xC0)
    blocks = []
    for sid, n in enumerate([33, 300, 700, 2049, 8193], start=1):
        r = np.arange(n)
        cd = [b"r%d" % x for x in rng.integers(0, 4, n)]
        pl = [b"p%05d" % x for x in rng.permutation(n)] if n >= 300 else [b"p%05d" % (x % 5) for x in r]
        idl = (10 + np.concatenate([[0], np.cumsum(_signed(rng, 0, 5, n - 1))])).tolist()
        dod = (100 + np.concatenate([[0], np.cumsum(rng.integers(1, 9, n - 1))])).tolist()
        raw = (20 + np.concatenate([[0], np.cumsum(_signed(rng, 0, 3, n - 1))])).tolist()
        if sid % 2 == 0:
            raw[n // 3] = None
        blocks.append(Blk(sid, {(FAM, "cd"): cd, (FAM, "pl"): pl, (FAM, "id"): idl, (FAM, "dod"): dod, (FAM, "raw"): raw,
                                (FAM, "dc"): (3 * r - 50).tolist()}))
    return blocks


@gpu
def test_conjunctions(bydb, gpu_ctx):
    """Eight predicates (kMaxPreds) over every page kind plus an absent tag and an absent family (all nil); a DoD tag after a
    dictionary predicate that already cleared bits; contradictions; 9 predicates -> EINVAL, a 65-byte literal -> ENOTSUP."""
    blocks = conj_blocks()
    P = O.Pred
    eight = [P(FAM, "cd", O.OP_NE, b"r0"), P(FAM, "pl", O.OP_GE, b"p00100"), P(FAM, "id", O.OP_LE, 14), P(FAM, "dod", O.OP_GT, 500),
             P(FAM, "raw", O.OP_NE, 21), P(FAM, "dc", O.OP_LT, 6000), P(FAM, "nope", O.OP_NE, b"x"), P("ghost", "t", O.OP_NE, 7)]
    cases = [
        eight,
        eight[:1] + eight[2:3] + eight[5:],                                  # the fast-lane kinds only + the absent ones
        [P(FAM, "cd", O.OP_EQ, b"r1"), P(FAM, "dod", O.OP_GE, 300)],         # DoD after a dictionary mask
        [P(FAM, "cd", O.OP_EQ, b"r9"), P(FAM, "dod", O.OP_GE, 0)],           # ... that cleared every bit
        [P(FAM, "id", O.OP_LT, 10), P(FAM, "id", O.OP_GT, 10)],             # contradictions
        [P(FAM, "cd", O.OP_EQ, b"r1"), P(FAM, "cd", O.OP_EQ, b"r2")],
        [P(FAM, "dc", O.OP_GE, 0), P(FAM, "raw", O.OP_LT, 0), P(FAM, "raw", O.OP_GE, 0)],
        [P(FAM, "nope", O.OP_EQ, b"")], [P("ghost", "t", O.OP_NE, 0)], [P(FAM, "nope", O.OP_GE, b""), P(FAM, "cd", O.OP_NE, b"r1")],
        [P(FAM, "pl", O.OP_LT, b"p00500"), P(FAM, "id", O.OP_NE, 10), P(FAM, "cd", O.OP_LE, b"r2")],
    ]
    part = build_blocks(blocks)
    with Scan(bydb, gpu_ctx, [(part, blocks)]) as s:
        for preds in cases:
            s.query(preds, ctx="conj")
        for tmin, tmax in [(T0 + 31 * STEP, T0 + 2048 * STEP), (T0 + 33 * STEP, T0 + 299 * STEP)]:
            s.query(eight, tmin, tmax, ctx="conj")
        G = s.usid.size
        for preds, code in [(eight + [P(FAM, "cd", O.OP_NE, b"r3")], bydb.capi.EINVAL), ([P(FAM, "cd", O.OP_NE, b"r" * 65)], bydb.capi.ENOTSUP)]:
            oq = O.Query([part], s.usid, AGGS, groups=np.arange(G, dtype=np.int32), n_groups=G, preds=preds)
            with pytest.raises(bydb.BydbError) as e:
                gpu_ctx.scan_agg(to_gpu_query(bydb, s.handles, oq))
            assert e.value.code == code, (len(preds), e.value)
        s.query([P(FAM, "cd", O.OP_NE, b"r" * 64)], ctx="conj")   # the context is still healthy; 64 bytes is accepted


# ------------------------------------------------------------------ mask x time range x dedup
def dedup_parts():
    """Part 1 (version 1) and part 2 (version 2), which rewrites rows 20..69 of every series with other tag values: the dedup
    shadow seeds the mask of part 1's blocks."""
    rng = np.random.default_rng(0xDD)
    sizes = [8193, 700, 65, 33]
    b1, b2 = [], []
    for sid, n in enumerate(sizes, start=1):
        cd = [b"r%d" % x for x in rng.integers(0, 3, n)]
        idl = (50 + np.concatenate([[0], np.cumsum(_signed(rng, 0, 4, n - 1))])).tolist()
        b1.append(Blk(sid, {(FAM, "cd"): cd, (FAM, "id"): idl}))
        a, e = 20, min(70, n)
        cd2 = [b"r%d" % x for x in rng.integers(0, 3, e - a)]
        id2 = (50 + np.concatenate([[0], np.cumsum(_signed(rng, 0, 4, e - a - 1))])).tolist()
        b2.append(Blk(sid, {(FAM, "cd"): cd2, (FAM, "id"): id2}, row0=a, rowid0=100_000))
        b1[-1].alive[a:e] = False
    return b1, b2


@gpu
def test_mask_time_range_and_dedup(bydb, gpu_ctx):
    """Predicates with time ranges that cut at rows 0 / 31 / 32 / 33 / count-1, over two overlapping parts.  The cuts include
    empty ranges (tmin > tmax, e.g. rows 33..31): they select no block, like the oracle, instead of failing the overlap check."""
    b1, b2 = dedup_parts()
    P = O.Pred
    pred_sets = [[P(FAM, "cd", O.OP_NE, b"r1")], [P(FAM, "id", O.OP_GE, 50)], [P(FAM, "cd", O.OP_LE, b"r1"), P(FAM, "id", O.OP_NE, 51)]]
    cuts_lo = [0, 31, 32, 33]
    cuts_hi = [31, 32, 33, 64, 699, 8191, 8192]
    with Scan(bydb, gpu_ctx, [(build_blocks(b1, 1), b1), (build_blocks(b2, 2), b2)]) as s:
        for preds in pred_sets:
            s.query(preds, ctx="dedup")
            for lo in cuts_lo:
                for hi in cuts_hi:
                    s.query(preds, T0 + lo * STEP, T0 + hi * STEP, ctx="dedup")


# ------------------------------------------------------------------ the cold path
@gpu
@pytest.mark.parametrize("host", ["pageable", "pinned"])
def test_masks_on_the_cold_host_path(bydb, gpu_ctx, host):
    """bydb_scan_agg_host over pageable images (gathered: every page 16-byte aligned) and pinned ones (read in place, pages at
    their file offsets): the fast lane meets the tag pages at other alignment phases."""
    blocks = []
    for kind in ("d3", "limits", "wrap", "dc_wrap", "dod", "wide"):
        for b in int_matrix_blocks(kind):
            blocks.append(Blk(len(blocks) + 1, b.tags))
    for p in sweep_positions()[::7]:
        blocks.append(Blk(len(blocks) + 1, {(FAM, "t"): sweep_values(p, 3)}))
    with Scan(bydb, gpu_ctx, [(build_blocks(blocks), blocks)]) as s:
        for lit in (SWEEP_LIT, 500, I64_MAX, I64_MIN + 3):
            for op in ALL_OPS:
                s.query([O.Pred(FAM, "t", op, lit)], ctx=f"host-{host}", host=host)
        s.query([O.Pred(FAM, "t", O.OP_GE, 0)], T0 + 32 * STEP, T0 + 2000 * STEP, ctx=f"host-{host}", host=host)


# ------------------------------------------------------------------ the layout claims above, on the CPU
def test_mask_case_layouts():
    """Each layout the GPU cases rest on, checked through the oracle's codecs, so a drifting helper fails here by name."""
    for kind in INT_KINDS:
        blocks = int_matrix_blocks(kind)
        for b in blocks:
            if b.n >= 3:
                assert b.tag_class((FAM, "t")) == INT_CLASS[kind], f"int_tag_values({kind!r}, {b.n})"
        if kind == "wide":
            for b in blocks[-2:]:   # 8192 and 8193 rows: the 4-byte varint starts in the last 1 KB chunk
                body = O.int64_list_encode(np.array(b.tags[(FAM, "t")], dtype=np.int64))[0]
                lens = _varint_lengths(body)
                start = sum(lens[:-1])
                assert lens[-1] == 4 and max(lens[:-1]) <= 2 and start // FAST_CHUNK == (len(body) - 1) // FAST_CHUNK, "int_tag_values('wide')"
        if kind == "dc_wrap":
            v = blocks[-1].tags[(FAM, "t")]
            assert v[2] > 0 > v[3], "int_tag_values('dc_wrap') must wrap past 2^63"
    for width in (3, 4):
        for p in sweep_positions():
            v = sweep_values(p, width)
            body, enc, _ = O.int64_list_encode(np.array(v, dtype=np.int64))
            lens = _varint_lengths(body)
            assert enc == O.ENC_DELTA and lens[p] == width and sum(lens[:p]) == p, f"sweep_values({p}, {width})"
            assert set(lens[:p] + lens[p + 1:]) == {1} and v.count(SWEEP_LIT) == 1 and v[p + 1] == SWEEP_LIT, f"sweep_values({p}, {width})"
    cases = str_cases()
    for name, want in STR_EXPECT.items():
        assert str_tag_class(cases[name]) == "dict" and dict_layout(cases[name]) == want, f"str_cases()[{name!r}]: {dict_layout(cases[name])}"
    for name, width in PLAIN_EXPECT.items():
        assert str_tag_class(cases[name]) == "plain" and plain_layout(cases[name]) == (width, True), f"str_cases()[{name!r}]"
    assert len(cases["run8193"]) == 8193 and None in cases["nil_empty"] and b"" in cases["nil_empty"]
    assert {b"ab", b"abc", b"abd", b"a"} <= set(cases["prefixes"]) and b"z" * 64 in cases["long64"]
    assert any(x is not None and max(x, default=0) >= 0x80 for x in cases["high_bytes"])
    # conjunction and dedup blocks: the page kinds their predicates are meant to reach
    cb = conj_blocks()
    assert [b.tag_class((FAM, "pl")) for b in cb] == ["dict"] + ["plain"] * 4
    assert {b.tag_class((FAM, k)) for b in cb for k in ("cd", "id", "dod", "dc")} == {"dict", "delta", "dod", "delta_const"}
    assert [b.tag_class((FAM, "raw")) for b in cb] == ["delta", "raw", "delta", "raw", "delta"]
    b1, b2 = dedup_parts()
    assert {b.tag_class((FAM, "id")) for b in b1 + b2} == {"delta"}

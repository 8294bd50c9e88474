"""The scan's page decoders against the oracle at the boundaries where they carry state.

An EncodeTypeDelta page reaches one of several decoders (DESIGN.md 4.2), chosen from what its field needs:

  SUM / COUNT / MEAN only, no predicates, no overlapping parts, block wholly in range -> scan_sum_express_kernel (express lane)
  SUM / COUNT / MEAN only, every row                                                -> delta_page_sum_all (SWAR)
  SUM / COUNT / MEAN only, time-range cut or row mask                                -> delta_page_sum_masked<kRowsRange / kRowsMask>
  MIN / MAX, alone or with SUM                                                       -> delta_page_fast<kNeedMinMax / kNeedSum|kNeedMinMax>
  any of the above with a varint of 4+ bytes                                         -> bail-out: rest list / slow lane, general decoder

Every case compares with the oracle (int64 and float64 min/max bit-exact, float64 sums within 1e-9) and checks the lane through
the counters: blocks_express_lane, blocks_slow_lane and slow_lane_reasons.  `lane_model` predicts both from the pages the part
writer produces, so a block that silently took another lane fails the test as surely as a wrong sum.

Values are built as int64 mantissas: an int64 field stores them as they are, a float64 field stores mantissa / 100 (the writer
turns it back into the same mantissas with exponent -2, which `page_class` checks through the oracle's own codec).
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, run_both

gpu = pytest.mark.gpu

SUMS = [O.AGG_SUM, O.AGG_COUNT, O.AGG_MEAN]
MINMAX = [O.AGG_MIN, O.AGG_MAX]
ALL5 = [O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN]
BLOCK_SIZES = [1, 2, 31, 32, 33, 8192, 8193]   # 8193: the longest block the writer cuts (measure.go first-block quirk)
# zig-zag length limits: 63/64 and -64/-65 (1 -> 2 bytes), 8191/8192 and -8192/-8193 (2 -> 3 bytes), the largest 3-byte values
LIMIT_DELTAS = [63, 64, -64, -65, 8191, 8192, -8192, -8193, (1 << 20) - 1, -((1 << 20) - 1), -(1 << 20)]
WIDE = 1 << 20          # zig-zag 2^21: the narrowest 4-byte varint
NARROW3 = (1 << 20) - 1  # zig-zag 2^21 - 2: the widest 3-byte varint
SHAPES = ["d1", "d2", "d3", "limits", "mix", "wide", "const", "delta_const", "dod", "null"]
_pid = [50_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def _signed(rng, lo, hi, n):
    """n deltas with |d| in [lo, hi] and random sign; the first two have opposite signs, so the page is neither a monotone
    (delta-of-delta) nor a constant-delta page."""
    d = rng.integers(lo, hi + 1, n) * np.where(rng.random(n) < 0.5, -1, 1)
    if n >= 2:
        d[0], d[1] = abs(d[0]), -abs(d[1])
    return d


def shape_values(kind, n, rng):
    """-> (int64 mantissas [n], null mask or None) of one block of `kind`."""
    first = 1_000_000 + int(rng.integers(0, 1000)) * 10 + 3   # >= 0 (a negative first value makes the writer pick delta-of-delta)
    nulls = None
    k = n - 1
    if kind == "d1":
        d = _signed(rng, 0, 63, k)
    elif kind == "d2":
        d = _signed(rng, 64, 8191, k)
    elif kind == "d3":
        d = _signed(rng, 8192, NARROW3, k)
    elif kind == "limits":
        d = np.resize(np.array(LIMIT_DELTAS, dtype=np.int64), k)
    elif kind == "mix":
        ln = rng.integers(0, 3, k)
        d = np.where(ln == 0, _signed(rng, 0, 63, k), np.where(ln == 1, _signed(rng, 64, 8191, k), _signed(rng, 8192, NARROW3, k)))
    elif kind == "wide":
        d = _signed(rng, 0, 63, k)
        if k >= 3:
            d[k // 2] = WIDE
    elif kind == "const":
        return np.full(n, first, dtype=np.int64), None
    elif kind == "delta_const":
        return first - 7 * np.arange(n, dtype=np.int64), None
    elif kind == "dod":
        d = rng.integers(1, 100, k)
    else:  # "null": a raw-cell fallback page
        d = _signed(rng, 0, 63, k)
        nulls = np.zeros(n, dtype=np.uint8)
        nulls[n // 2] = 1
    v = np.concatenate([[first], first + np.cumsum(np.asarray(d, dtype=np.int64))]).astype(np.int64)
    return v, nulls


def _varint_lengths(body):
    lens, run = [], 0
    for b in body:
        run += 1
        if b < 0x80:
            lens.append(run)
            run = 0
    assert run == 0, "truncated varint"
    return lens


def page_class(mantissas, nulls, is_float):
    """What the writer makes of one block's values: 'raw' (a null cell: fallback page), 'const', 'delta_const', 'dod',
    'delta' (every varint <= 3 bytes) or 'wide' (a delta page with a varint of 4+ bytes)."""
    if nulls is not None and nulls.any():
        return "raw"
    m = np.asarray(mantissas, dtype=np.int64)
    if is_float:
        back, exp = O.float64_to_decimal_list(m / 100.0)
        assert exp == -2 and back.tolist() == m.tolist(), "float64 values must store the intended mantissas"
    body, enc, first = O.int64_list_encode(m)
    assert first == m[0]
    if enc != 3:
        return {1: "const", 2: "delta_const", 4: "dod"}[enc]
    return "wide" if max(_varint_lengths(body)) > 3 else "delta"


def field_values(m, is_float):
    return m / 100.0 if is_float else m


class Block:
    def __init__(self, sid, ts, m, nulls, is_float):
        self.sid, self.ts, self.m, self.nulls = sid, ts, m, nulls
        self.cls = page_class(m, nulls, is_float)


def lane_model(blocks, active, sums_only, express_allowed):
    """(expected express-lane blocks, expected slow-lane blocks) of one query over one field.
    active[i]: rows of block i the query keeps (time range, predicates, dedup); whole[i]: block wholly inside the time range."""
    express = slow = 0
    for b, (n_active, whole) in zip(blocks, active):
        if sums_only and express_allowed and whole and b.cls == "delta":
            express += 1
        elif n_active > 0 and b.cls in ("wide", "raw"):
            slow += 1
    return express, slow


def assert_lanes(got, express, slow, ctx):
    st = got.stats
    assert st.blocks_express_lane == express, f"{ctx}: express-lane blocks {st.blocks_express_lane}, expected {express}"
    assert st.blocks_slow_lane == slow, f"{ctx}: slow-lane blocks {st.blocks_slow_lane}, expected {slow}"
    assert st.slow_lane_reasons == (4 if slow else 0), f"{ctx}: slow-lane reasons {st.slow_lane_reasons:#x}"


# ------------------------------------------------------------------ the matrix
def _matrix_part(is_float, seed):
    rng = np.random.default_rng(seed)
    blocks = []
    sid = 1
    for kind in SHAPES:
        for n in BLOCK_SIZES:
            m, nulls = shape_values(kind, n, rng)
            blocks.append(Block(sid, T0 + np.arange(n, dtype=np.int64) * STEP, m, nulls, is_float))
            sid += 1
    return blocks


def _build(blocks, is_float, version=1):
    sids = np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks])
    ts = np.concatenate([b.ts for b in blocks])
    vals = np.concatenate([field_values(b.m, is_float) for b in blocks])
    nulls = np.concatenate([b.nulls if b.nulls is not None else np.zeros(b.m.size, np.uint8) for b in blocks])
    rows = np.concatenate([np.arange(b.m.size) for b in blocks])
    region = [b"r%d" % ((r * 7 + s) % 3) for r, s in zip(rows.tolist(), sids.tolist())]
    # int64 tag: 3, 1, then 1..3 -- a narrow delta page (or const / constant-delta for 1-2 rows), which the fast lane compares
    code = np.where(rows == 0, 3, np.where(rows == 1, 1, 1 + (rows * 5 + sids.astype(np.int64)) % 3)).astype(np.int64)
    vt = O.VT_FLOAT64 if is_float else O.VT_INT64
    return build_part(sids, ts, np.full(sids.size, version, np.int64), [("v", vt, vals, nulls if nulls.any() else None)],
                      [("default", [("region", O.VT_STR, region, None), ("code", O.VT_INT64, code, None)])]), rows, region, code


MODES = ["all", "range", "dict_mask", "int_mask", "dedup"]


@gpu
@pytest.mark.parametrize("is_float", [False, True], ids=["int64", "float64"])
@pytest.mark.parametrize("mode", MODES)
def test_decoder_matrix(bydb, gpu_ctx, mode, is_float):
    """Every page shape x block size x aggregate set under one row mode.  Targets: the express lane (mode all, sums), SWAR
    delta_page_sum_all (mode all, sums, only what the express lane hands on), delta_page_sum_masked<range / mask> (sums under the
    other modes), delta_page_fast<minmax / both> (MIN+MAX and all five), dod_page_fast, the arithmetic pages and the slow lane
    (wide and raw-cell pages)."""
    blocks = _matrix_part(is_float, 0x1A7E + int(is_float))
    part, rows, region, code = _build(blocks, is_float)
    parts = [part]
    usid = np.array([b.sid for b in blocks], dtype=np.uint64)
    tmin, tmax, preds = -(1 << 63), (1 << 63) - 1, []
    keep = [np.ones(b.m.size, bool) for b in blocks]
    if mode == "range":
        tmin, tmax = T0 + STEP, T0 + 8000 * STEP        # cuts row 0 of every block and the tail of the long ones
    elif mode == "dict_mask":
        preds = [O.Pred("default", "region", O.OP_EQ, b"r1")]
        keep = [np.array([(r * 7 + b.sid) % 3 == 1 for r in range(b.m.size)]) for b in blocks]
    elif mode == "int_mask":
        preds = [O.Pred("default", "code", O.OP_NE, 2)]
        keep = [np.array([(3 if r == 0 else 1 if r == 1 else 1 + (r * 5 + b.sid) % 3) != 2 for r in range(b.m.size)]) for b in blocks]
    elif mode == "dedup":
        # a second part rewrites the first 5 rows of every series with a higher version: those rows of the first part are shadowed
        rng = np.random.default_rng(99)
        shadow = []
        for b in blocks:
            k = min(5, b.m.size)
            shadow.append(Block(b.sid, b.ts[:k], shape_values("d1", k, rng)[0], None, is_float))
        parts.append(_build(shadow, is_float, version=2)[0])
        keep = [np.arange(b.m.size) >= 5 for b in blocks]
    ts_in = [(b.ts >= tmin) & (b.ts <= tmax) for b in blocks]
    active = [(int((k & t).sum()), bool(t.all())) for k, t in zip(keep, ts_in)]
    for aggset in (SUMS, MINMAX, ALL5):
        aggs = [("v", f) for f in aggset]
        oq = O.Query(parts, usid, aggs, groups=np.arange(usid.size, dtype=np.int32), n_groups=usid.size, tmin=tmin, tmax=tmax, preds=preds)
        got, want = run_both(bydb, gpu_ctx, parts, oq, _next_pid())
        ctx = f"{mode}/{'f64' if is_float else 'i64'}/{[f for _, f in aggs]}"
        assert_parity(got, want, aggs, ctx)
        sums_only = aggset is SUMS
        # dedup: the shadowing part's blocks are narrow delta / const pages, none of them bails out
        express, slow = lane_model(blocks, active, sums_only, mode == "all")
        assert_lanes(got, express, slow, ctx)


# ------------------------------------------------------------------ the same answer from two lanes
@gpu
@pytest.mark.parametrize("is_float", [False, True], ids=["int64", "float64"])
def test_same_sum_from_express_swar_masked_and_fast(bydb, gpu_ctx, is_float):
    """SUM is an exact 128-bit sum converted once, so the lane that computed it must not show.  [(f,SUM),(f,COUNT)] takes the
    express lane; adding (g,MAX) keeps f's need at SUM but closes the express lane (delta_page_sum_all); under a mask [(f,SUM)]
    takes delta_page_sum_masked<kRowsMask> and [(f,SUM),(f,MAX)] delta_page_fast<kNeedSum|kNeedMinMax>."""
    rng = np.random.default_rng(404 + int(is_float))
    kinds = ["d1", "d2", "d3", "limits", "mix"]
    blocks, sid = [], 1
    for kind in kinds:
        for n in (33, 700, 2049, 4097, 8193):
            m, _ = shape_values(kind, n, rng)
            blocks.append(Block(sid, T0 + np.arange(n, dtype=np.int64) * STEP, m, None, is_float))
            sid += 1
    sids = np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks])
    ts = np.concatenate([b.ts for b in blocks])
    vt = O.VT_FLOAT64 if is_float else O.VT_INT64
    vals = np.concatenate([field_values(b.m, is_float) for b in blocks])
    g = np.round(rng.normal(0, 1, sids.size), 2)
    region = [b"r%d" % v for v in rng.integers(0, 3, sids.size)]
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("f", vt, vals, None), ("g", O.VT_FLOAT64, g, None)],
                      [("default", [("region", O.VT_STR, region, None)])])
    usid = np.unique(sids)
    groups = np.arange(usid.size, dtype=np.int32)
    col = 1 if is_float else 0   # val_f64 / val_i64

    def run(aggs, preds=()):
        oq = O.Query([part], usid, aggs, groups=groups, n_groups=usid.size, preds=list(preds))
        got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
        assert_parity(got, want, aggs, str(aggs))
        return got

    def sums(res):
        return (res.val_f64[:, 0] if col else res.val_i64[:, 0]).view(np.uint64).tolist()

    express = run([("f", O.AGG_SUM), ("f", O.AGG_COUNT)])
    assert express.stats.blocks_express_lane == len(blocks) and express.stats.blocks_slow_lane == 0
    swar = run([("f", O.AGG_SUM), ("f", O.AGG_COUNT), ("g", O.AGG_MAX)])
    assert swar.stats.blocks_express_lane == 0 and swar.stats.blocks_slow_lane == 0
    assert sums(express) == sums(swar), "express lane and delta_page_sum_all must give the same bits"
    pred = [O.Pred("default", "region", O.OP_NE, b"r2")]
    masked = run([("f", O.AGG_SUM)], pred)
    both = run([("f", O.AGG_SUM), ("f", O.AGG_MAX)], pred)
    assert masked.stats.blocks_express_lane == 0 and masked.stats.blocks_slow_lane == 0 and both.stats.blocks_slow_lane == 0
    assert sums(masked) == sums(both), "delta_page_sum_masked and delta_page_fast must give the same bits"


# ------------------------------------------------------------------ a wide varint at every boundary
def wide_at(p, n, width=4):
    """int64 values of one block whose delta page body is all 1-byte varints except one `width`-byte varint starting at body
    byte p (p 1-byte deltas before it)."""
    d = np.where(np.arange(n - 1) % 2 == 0, 1, -1).astype(np.int64)
    d[p] = WIDE if width == 4 else NARROW3
    return np.concatenate([[1000], 1000 + np.cumsum(d)]).astype(np.int64)


def _boundary_positions():
    pos = set()
    for k in (1, 2, 3, 31, 32, 33, 64):          # 64 B lane windows; 64 * 32 = 2048 (chunk / TMA stage), 64 * 64 = 4096
        pos.update(range(64 * k - 40, 64 * k + 41))
    return sorted(pos)


BOUNDARY_ROWS = 4300


@pytest.mark.parametrize("width", [3, 4])
def test_wide_at_helper_places_the_varint(width):
    """The layout claim the boundary sweep rests on, checked against the oracle's encoder: body byte p starts the only
    multi-byte varint, and the float64 form of the values stores the same mantissas."""
    for p in [0, 1, 63, 64, 2047, 2048, 4095, 4096, 4136] + _boundary_positions()[::17]:
        v = wide_at(p, BOUNDARY_ROWS, width)
        body, enc, first = O.int64_list_encode(v)
        assert enc == 3 and first == 1000, p
        lens = _varint_lengths(body)
        assert len(lens) == BOUNDARY_ROWS - 1 and lens[p] == width and set(lens[:p] + lens[p + 1:]) == {1}, p
        assert sum(lens[:p]) == p
        assert page_class(v, None, True) == ("wide" if width == 4 else "delta")


def test_stats_struct_layout(bydb):
    """blocks_express_lane took the place of a reserved word: bydb_stats keeps its size and every other offset."""
    import ctypes
    S = bydb.capi._Stats
    assert ctypes.sizeof(S) == 80 and S.blocks_express_lane.offset == 76 and S.slow_lane_reasons.offset == 72


@gpu
@pytest.mark.parametrize("width", [3, 4])
def test_varint_at_every_boundary(bydb, gpu_ctx, width):
    """One block per series, one group per series: a single query checks every position.  4-byte: every block must bail out
    of the express lane, delta_page_sum_all, delta_page_fast and delta_page_sum_masked alike (slow lane) and still match the oracle;
    3-byte: no block may bail out."""
    pos = _boundary_positions()
    sids = np.repeat(np.arange(1, len(pos) + 1, dtype=np.uint64), BOUNDARY_ROWS)
    ts = np.tile(T0 + np.arange(BOUNDARY_ROWS, dtype=np.int64) * STEP, len(pos))
    m = np.concatenate([wide_at(p, BOUNDARY_ROWS, width) for p in pos])
    region = [b"r%d" % (r % 4) for r in range(sids.size)]
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("i", O.VT_INT64, m, None), ("f", O.VT_FLOAT64, m / 100.0, None)],
                      [("default", [("region", O.VT_STR, region, None)])])
    usid = np.unique(sids)
    nb = usid.size
    wide = width == 4
    cases = [  # (aggs, preds, tmax, express blocks, decoder behind the express lane)
        ("express -> delta_page_sum_all", lambda f: [(f, O.AGG_SUM), (f, O.AGG_COUNT)], [], (1 << 63) - 1, 0 if wide else nb),
        ("delta_page_fast<minmax>", lambda f: [(f, O.AGG_MIN), (f, O.AGG_MAX)], [], (1 << 63) - 1, 0),
        ("delta_page_fast<both>", lambda f: [(f, O.AGG_SUM), (f, O.AGG_MAX)], [], (1 << 63) - 1, 0),
        ("delta_page_sum_masked<mask>", lambda f: [(f, O.AGG_SUM)], [O.Pred("default", "region", O.OP_NE, b"r2")], (1 << 63) - 1, 0),
        ("delta_page_sum_masked<range>", lambda f: [(f, O.AGG_SUM)], [], T0 + (BOUNDARY_ROWS - 2) * STEP, 0),
    ]
    for name, mk, preds, tmax, express in cases:
        for f in ("i", "f"):
            aggs = mk(f)
            oq = O.Query([part], usid, aggs, groups=np.arange(nb, dtype=np.int32), n_groups=nb, tmax=tmax, preds=preds)
            got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
            ctx = f"{width}-byte/{name}/{f}"
            assert_parity(got, want, aggs, ctx)
            assert_lanes(got, express, nb if wide else 0, ctx)


# ------------------------------------------------------------------ express batch hand-over
def handover_blocks():
    """-> (kinds, rows, int64 values) of the blocks of test_express_batch_handover, in series order."""
    rng = np.random.default_rng(8)
    pattern = [("n", 1), ("b", 2049), ("b", 2048), ("w", 2050), ("b", 4097), ("b", 2050), ("d3", 600), ("b", 4096)]
    lens, kinds = [], []
    for i in range(72_000):
        k, n = pattern[i % 8] if i < 4000 else ("b", 24)
        lens.append(n)
        kinds.append(k)
    vals = []
    for k, n in zip(kinds, lens):
        if k == "n":
            v = np.array([int(rng.integers(0, 100))], np.int64)
        elif k == "d3":
            v = shape_values("d3", n, rng)[0]
        else:
            v = wide_at(n // 2, n, 4) if k == "w" else np.concatenate([[50], 50 + np.cumsum(_signed(rng, 0, 63, n - 1))])
        vals.append(np.asarray(v, np.int64))
    return kinds, lens, vals


@gpu
def test_express_batch_handover(bydb, gpu_ctx):
    """A warp of the express lane takes up to 8 blocks at a time and streams their pages through one TMA ring; it does so while
    more than 16 blocks per warp are left, so the part holds ~72k blocks and the mixed pages sit at its front.  The mix: 1-row
    blocks (no page body), bodies of exactly 2048 and 4096 bytes (a stage / two), 2047 and 2049, narrow 3-byte pages, and one
    wide page per group of 8, which leaves the ring while its neighbours stay.  These pages keep their varints (no dense form,
    tests/test_gpu_dense_boundaries.py), so the test pins the SWAR decode."""
    kinds, lens, vals = handover_blocks()
    sids = np.repeat(np.arange(1, len(lens) + 1, dtype=np.uint64), lens)
    ts = np.concatenate([T0 + np.arange(n, dtype=np.int64) * STEP for n in lens])
    expect_express = expect_slow = 0
    for v in vals:
        cls = page_class(v, None, False) if v.size > 1 else "const"
        expect_express += cls == "delta"
        expect_slow += cls == "wide"
    body = {("b", 2049): 2048, ("b", 2048): 2047, ("b", 2050): 2049, ("b", 4097): 4096, ("b", 4096): 4095}
    for (k, n), want_body in body.items():   # the page bodies the case claims
        i = list(zip(kinds, lens)).index((k, n))
        assert len(O.int64_list_encode(vals[i])[0]) == want_body
    v = np.concatenate(vals)
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("c", O.VT_INT64, v, None)])
    usid = np.unique(sids)
    aggs = [("c", O.AGG_SUM), ("c", O.AGG_COUNT)]
    oq = O.Query([part], usid, aggs, groups=(np.arange(usid.size) % 4096).astype(np.int32), n_groups=4096)
    got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
    assert_parity(got, want, aggs, "express batches")
    assert_lanes(got, expect_express, expect_slow, "express batches")


# ------------------------------------------------------------------ int64 wrap-around
@gpu
def test_int64_sum_wraps_mod_2_64(bydb, gpu_ctx):
    """Narrow deltas around a first value near 2^63: the page stays on the SWAR / express path while n * first and the sum wrap
    modulo 2^64 (a first value below zero makes the writer choose delta-of-delta, which dod_page_fast takes)."""
    rng = np.random.default_rng(63)
    firsts = [(1 << 63) - 200_000, (1 << 63) - 100_000, -(1 << 63) + 200_000, (1 << 62) + 12345]
    n = 8193
    blocks = []
    for i, f in enumerate(firsts):
        d = _signed(rng, 0, 63, n - 1)
        v = [f]
        for x in d.tolist():
            v.append(v[-1] + x)
        assert all(-(1 << 63) <= x < (1 << 63) for x in v)
        blocks.append(np.array(v, dtype=np.int64))
    sids = np.repeat(np.arange(1, len(firsts) + 1, dtype=np.uint64), n)
    ts = np.tile(T0 + np.arange(n, dtype=np.int64) * STEP, len(firsts))
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("c", O.VT_INT64, np.concatenate(blocks), None)],
                      [("default", [("region", O.VT_STR, [b"r%d" % (r % 3) for r in range(sids.size)], None)])])
    usid = np.unique(sids)
    groups = np.arange(usid.size, dtype=np.int32)

    def wrap(x):
        x &= (1 << 64) - 1
        return x - (1 << 64) if x >= (1 << 63) else x
    for aggs, preds, mask in [([("c", O.AGG_SUM), ("c", O.AGG_COUNT)], [], None),                    # express
                              ([("c", O.AGG_SUM), ("c", O.AGG_MIN)], [], None),                      # delta_page_fast<both>
                              ([("c", O.AGG_SUM)], [O.Pred("default", "region", O.OP_EQ, b"r1")], 1)]:  # delta_page_sum_masked
        oq = O.Query([part], usid, aggs, groups=groups, n_groups=usid.size, preds=preds)
        got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
        assert_parity(got, want, aggs, f"wrap/{aggs}")
        for gi, b in enumerate(blocks):
            rows = range(n) if mask is None else [r for r in range(n) if ((gi * n + r) % 3) == mask]
            assert int(got.val_i64[gi, 0]) == wrap(sum(int(b[r]) for r in rows)), (aggs, gi)
        assert got.stats.blocks_slow_lane == 0
    express = run_both(bydb, gpu_ctx, [part], O.Query([part], usid, [("c", O.AGG_SUM)], groups=groups, n_groups=usid.size), _next_pid())[0]
    assert express.stats.blocks_express_lane == 3   # the delta-of-delta page (first value below zero) is not an express page


# ------------------------------------------------------------------ mask edges of delta_page_sum_masked
@gpu
@pytest.mark.parametrize("is_float", [False, True], ids=["int64", "float64"])
def test_masked_sum_mask_and_range_edges(bydb, gpu_ctx, is_float):
    """delta_page_sum_masked<kRowsMask> with masks selecting no row, only row 0, only the last row, every row but one, and runs
    crossing 32-row mask words; <kRowsRange> with ranges starting at row 0 and ending at row count-1.  Each series is one block
    of a mixed-length delta page; a per-row int64 tag (row index, a constant-delta page) drives the mask."""
    rng = np.random.default_rng(77 + int(is_float))
    sizes = [31, 32, 33, 64, 65, 700, 2049, 8193]
    blocks = [shape_values("mix", n, rng)[0] for n in sizes]
    sids = np.repeat(np.arange(1, len(sizes) + 1, dtype=np.uint64), sizes)
    ts = np.concatenate([T0 + np.arange(n, dtype=np.int64) * STEP for n in sizes])
    rows = np.concatenate([np.arange(n, dtype=np.int64) for n in sizes])
    runs = [b"in" if (r % 97) in range(30, 70) else b"out" for r in rows.tolist()]   # runs of 40 rows crossing mask words
    m = np.concatenate(blocks)
    vt = O.VT_FLOAT64 if is_float else O.VT_INT64
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("v", vt, field_values(m, is_float), None)],
                      [("default", [("row", O.VT_INT64, rows, None), ("run", O.VT_STR, runs, None)])])
    usid = np.unique(sids)
    groups = np.arange(usid.size, dtype=np.int32)
    aggs = [("v", O.AGG_SUM)]
    cases = [[O.Pred("default", "row", O.OP_LT, 0)], [O.Pred("default", "row", O.OP_EQ, 0)], [O.Pred("default", "row", O.OP_NE, 0)],
             [O.Pred("default", "row", O.OP_GE, 30)], [O.Pred("default", "row", O.OP_NE, 31)], [O.Pred("default", "row", O.OP_NE, 32)],
             [O.Pred("default", "run", O.OP_EQ, b"in")]]
    cases += [[O.Pred("default", "row", O.OP_EQ, n - 1)] for n in sizes] + [[O.Pred("default", "row", O.OP_NE, n - 1)] for n in sizes]
    for preds in cases:
        oq = O.Query([part], usid, aggs, groups=groups, n_groups=usid.size, preds=preds)
        got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
        ctx = f"mask/{[(p.tag, p.op, p.value) for p in preds]}"
        assert_parity(got, want, aggs, ctx)
        assert_lanes(got, 0, 0, ctx)
    for tmin, tmax in [(T0, T0 + 30 * STEP), (T0, T0 + 31 * STEP), (T0 + 1 * STEP, T0 + 8192 * STEP), (T0 + 32 * STEP, T0 + 8192 * STEP),
                       (T0, T0), (T0 + 8192 * STEP, T0 + 9000 * STEP)] + [(T0, T0 + (n - 2) * STEP) for n in sizes]:
        oq = O.Query([part], usid, aggs, groups=groups, n_groups=usid.size, tmin=tmin, tmax=tmax)
        got, want = run_both(bydb, gpu_ctx, [part], oq, _next_pid())
        ctx = f"range/{(tmin - T0) // STEP}-{(tmax - T0) // STEP}"
        assert_parity(got, want, aggs, ctx)
        whole = sum(1 for n in sizes if tmin <= T0 and T0 + (n - 1) * STEP <= tmax)
        assert_lanes(got, whole, 0, ctx)

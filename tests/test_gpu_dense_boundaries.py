"""Dense pages (DESIGN.md 3.3) at their boundaries: which pages admission converts, every plane width on the device, and dense
pages next to varint pages in one express batch.

`dense_model` restates admission from the page bytes the oracle's writer makes, without the CUDA code: an EncodeTypeDelta page
(type 3) in fv.bin of a block of 1 .. 65,536 rows, every varint of at most 3 bytes, a first value at least count << 20 inside
int64, values spanning at most 2^32 - 1 (b = the span's bit length), and a descriptor plus planes smaller than the page.  The
non-GPU tests hold every fixture block to what it is built for (encode type, b, page length, the side of a rule it sits on) and
the fixtures' pages to the part's fv.bin byte for byte.  The GPU tests run two contexts, dense pages on and off, and want
bit-identical answers that match the oracle, an exact reference (int64 sums modulo 2^64, float64 sums against a `fractions`
sum of the decimal integers), the lane counters `lane_model` predicts and the `dense_pages` / `dense_bytes` the model predicts.

What the writer cannot make, and only tests/native/dense_page_test.cc covers: b = 0 (a constant block is EncodeTypeConst), the
32-bit plane and the span rule (b >= 24 never passes the size rule with varints of at most 3 bytes) and blocks of more than
8,193 rows."""
from collections import namedtuple
from fractions import Fraction
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_lanes import NARROW3, WIDE, handover_blocks, lane_model

gpu = pytest.mark.gpu
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
MASK64 = (1 << 64) - 1
STAGE = 4096
WIDTHS = (32, 16, 8, 4, 2, 1)


# ------------------------------------------------------------------ the model of admission
def align_up(x, a):
    return (x + a - 1) // a * a


def plane_bytes(n, w):
    return (n * w + 127) // 128 * 16


def stream_bytes(n, b):
    return sum(plane_bytes(n, w) for w in WIDTHS if b & w)


def read_varints(body):
    """-> (zig-zag decoded values as int64, byte lengths) of a varint stream"""
    a = np.frombuffer(bytes(body), np.uint8)
    ends = np.flatnonzero(a < 0x80)
    assert a.size == 0 or (ends.size and ends[-1] == a.size - 1), "truncated varint"
    starts = np.concatenate([[0], ends[:-1] + 1]).astype(np.int64)
    lens = ends - starts + 1
    idx = np.repeat(np.arange(ends.size), lens)
    shift = (7 * (np.arange(a.size) - starts[idx])).astype(np.uint64)
    x = np.zeros(ends.size, np.uint64)
    np.add.at(x, idx, (a & 0x7F).astype(np.uint64) << shift)
    return (x >> np.uint64(1)).astype(np.int64) ^ -(x & np.uint64(1)).astype(np.int64), lens


def page_first(page, is_float):
    """the page's first value: big-endian with the sign bit flipped (encoding.Int64ToBytes)"""
    hdr = 11 if is_float else 9
    u = int.from_bytes(page[hdr - 8:hdr], "big") ^ (1 << 63)
    return u - (1 << 64) if u >> 63 else u


def page_values(page, count, is_float):
    """-> (values, varint lengths) of a type-3 page; the values as python ints, exact while no prefix leaves int64"""
    hdr = 11 if is_float else 9
    deltas, lens = read_varints(page[hdr:])
    assert deltas.size == count - 1
    with np.errstate(over="ignore"):
        v = np.concatenate([[0], np.cumsum(deltas)]) + np.int64(page_first(page, is_float))
    return v, lens


Dense = namedtuple("Dense", "m b plane_bytes exp n")


def dense_model(page, count, is_float):
    """The dense form admission gives this fv.bin page of a block of `count` rows, or None (the page keeps its varints)."""
    hdr = 11 if is_float else 9
    if not 1 <= count <= 65536 or len(page) < hdr or page[0] != 3:
        return None
    first = page_first(page, is_float)
    reach = count << 20
    if not I64_MIN + reach <= first <= I64_MAX - reach:
        return None
    v, lens = page_values(page, count, is_float)   # exact: a varint of <= 3 bytes moves a value by less than 2^20
    if max(lens, default=0) > 3:
        return None
    m, span = int(v.min()), int(v.max()) - int(v.min())
    if span > 0xFFFFFFFF:
        return None
    b = span.bit_length()
    pb = stream_bytes(count, b)
    if 32 + pb >= len(page):
        return None
    return Dense(m, b, pb, int.from_bytes(page[1:3], "big", signed=True) if is_float else 0, count)


def page_kind(page, count, is_float):
    """What the express lane makes of a page it sums: 'delta' (type 3, varints of at most 3 bytes), 'wide' (a varint of 4+
    bytes: the block goes on to the fast lane, whose decoder bails out to the slow lane) or 'other'."""
    if count < 2 or page[0] != 3:
        return "other"
    return "wide" if max(page_values(page, count, is_float)[1]) > 3 else "delta"


def int_page(v):
    body, enc, first = O.int64_list_encode(v)
    return bytes([enc]) + O.conv_int64_to_bytes(first) + body


def float_page(f):
    ints, exp = O.float64_to_decimal_list(f)
    body, enc, first = O.int64_list_encode(ints)
    return bytes([enc]) + int(exp).to_bytes(2, "big", signed=True) + O.conv_int64_to_bytes(first) + body


def expected_dense(pages):
    """pages: [(page, rows, is_float)] of a part -> (dense pages, sum of their plane bytes)"""
    ds = [d for d in (dense_model(p, n, f) for p, n, f in pages) if d is not None]
    return len(ds), sum(d.plane_bytes for d in ds)


# ------------------------------------------------------------------ fixtures
_CLASS = {1: (1, 63), 2: (65, 8191), 3: (8193, NARROW3)}   # |delta| of a zig-zag varint of that many bytes, either sign


def walk(rng, b, lengths, base, u0=0):
    """base + u_i: u starts at u0 and stays in [0, 2^b - 1], each step a delta whose varint has the given length.  It climbs
    until the next step would leave the range and then turns, so it passes 2^(b-1) and the span has bit length b."""
    span, u, up, out = (1 << b) - 1, u0, True, [u0]
    for L in lengths:
        lo, hi = _CLASS[L]
        if up and span - u < lo:
            up = False
        elif not up and u < lo:
            up = True
        room = span - u if up else u
        assert room >= lo, (b, L)
        mag = int(rng.integers(lo, min(hi, room) + 1))
        u += mag if up else -mag
        out.append(u)
    return np.array([base + x for x in out], dtype=np.int64)


def narrow_len(b):
    """the varint length that makes a b-bit walk's planes smaller than its varints"""
    return 1 if b <= 7 else 2 if b <= 14 else 3


class Blk:
    """One series = one block: int64 field i, float64 field f, int64 field c (counted only), and what the block claims."""

    def __init__(self, name, i, f, c=None, claim_i=None, claim_f=None):
        self.name, self.i, self.f = name, np.asarray(i, np.int64), np.asarray(f, np.float64)
        self.n = self.i.size
        assert self.f.size == self.n
        self.c = np.asarray(c if c is not None else np.arange(self.n) % 3 + 7 * (np.arange(self.n) % 2), np.int64)
        self.pi, self.pf, self.pc = int_page(self.i), float_page(self.f), int_page(self.c)
        self.di, self.df = dense_model(self.pi, self.n, False), dense_model(self.pf, self.n, True)
        self.claim_i, self.claim_f = claim_i or {}, claim_f or {}


def fvals(rng, b, n, exp, base=None, u0=0, lengths=None):
    """float64 values whose decimal integers walk b bits with the given exponent (< 0: the integers are not multiples of 10)"""
    base = (10 ** 6 + 3) if base is None else base
    ints = walk(rng, b, lengths or [narrow_len(b)] * (n - 1), base, u0)
    return ints.astype(np.float64) / 10.0 ** -exp if exp < 0 else ints.astype(np.float64)


def size_pair_lengths(n, b, is_float, converted):
    """varint lengths (1- and 2-byte) of an n-row page whose size is 32 + planes (kept) or one byte more (converted)"""
    hdr = 11 if is_float else 9
    body = 32 + stream_bytes(n, b) - hdr + (1 if converted else 0)
    twos = body - (n - 1)
    assert 0 < twos < n - 1
    lens = [1] * (n - 1)
    for k in range(twos):   # spread the 2-byte varints over the page
        lens[(k * (n - 1)) // twos] = 2
    return lens


def main_blocks(seed):
    """The blocks of the main part: every b from 1 to 23 for both types, the stream geometry, the admission pairs, the values."""
    rng = np.random.default_rng(seed)
    out = []
    # every reachable bit length: int64 and float64 (exponents -1 .. -15 and 0)
    for b in range(1, 24):
        n = 1000 + 61 * b
        exp = -(1 + b % 15) if b != 15 else 0
        i = walk(rng, b, [narrow_len(b)] * (n - 1), 1_000 + int(rng.integers(0, 10 ** 6)))
        f = fvals(rng, b, n, exp, base=(10 ** 6 + 3) if exp < 0 else 10 ** 6 + 7)
        out.append(Blk(f"b{b}", i, f, claim_i=dict(b=b), claim_f=dict(b=b, exp=exp)))
    # stream geometry (int64 and float64 alike): one 16-byte piece, a stream ending on a 4 KB stage, one piece past a stage,
    # 8,193 rows
    for n, b, want in ((41, 1, 16), (64, 1, 16), (128, 1, 16), (129, 1, 32), (4096, 8, STAGE), (8192, 12, 3 * STAGE),
                       (4097, 8, STAGE + 16), (8193, 13, None), (8193, 23, None)):
        i = walk(rng, b, [narrow_len(b)] * (n - 1), 5_000)
        f = fvals(rng, b, n, -3)
        out.append(Blk(f"geom n{n} b{b}", i, f, claim_i=dict(b=b, plane_bytes=want), claim_f=dict(b=b, plane_bytes=want, exp=-3)))
    # the size rule: 32 + planes == page (kept) and one byte more (converted)
    for n, b in ((1024, 8), (700, 10), (3000, 9)):
        for conv in (False, True):
            i = walk(rng, b, size_pair_lengths(n, b, False, conv), 2_000)
            f = fvals(rng, b, n, -2, lengths=size_pair_lengths(n, b, True, conv))
            claim = dict(b=b, dense=conv, page=32 + stream_bytes(n, b) + conv)
            out.append(Blk(f"size n{n} b{b} {'conv' if conv else 'kept'}", i, f, claim_i=claim, claim_f=dict(claim, exp=-2)))
    # the reach rule: first == INT64_MAX - (count << 20) (converted) and one more (kept); float64 pages stay far inside
    for n, b in ((3000, 10), (8193, 14)):
        for extra in (0, 1):
            first = I64_MAX - (n << 20) + extra
            i = walk(rng, b, [narrow_len(b)] * (n - 1), first)
            out.append(Blk(f"reach n{n} +{extra}", i, fvals(rng, b, n, -1), claim_i=dict(first=first, dense=extra == 0)))
    # b = 24: kept, whatever the length
    for n in (1500, 8193):
        i = walk(rng, 24, [3] * (n - 1), 100)
        out.append(Blk(f"b24 n{n}", i, fvals(rng, 24, n, -4, lengths=[3] * (n - 1)), claim_i=dict(b=24, dense=False),
                       claim_f=dict(b=24, dense=False)))
    # a 4-byte varint: kept, and the block leaves the express lane (for both fields: one page bails out)
    i = walk(rng, 6, [1] * 2999, 77)
    i[1500:] += WIDE + 64   # a delta of more than 2^20
    out.append(Blk("wide", i, fvals(rng, 6, 3000, -2), claim_i=dict(dense=False, kind="wide"), claim_f=dict(b=6, dense=True)))
    # m < 0: the first value >= 0, then a reset below zero
    for b in (5, 12, 20):
        n = 2500
        span = (1 << b) - 1
        i = walk(rng, b, [narrow_len(b)] * (n - 1), -(span // 2), u0=span)
        f = fvals(rng, b, n, -2, base=-(span // 2), u0=span)
        out.append(Blk(f"neg b{b}", i, f, claim_i=dict(b=b, neg=True), claim_f=dict(b=b, neg=True, exp=-2)))
    # int64 blocks near the top of the reach window: n * m and the group sums wrap
    for k, b in enumerate((3, 11, 17, 22)):
        n = 8193 - 997 * k
        i = walk(rng, b, [narrow_len(b)] * (n - 1), I64_MAX - (n << 20) - 12345 * k)
        out.append(Blk(f"top b{b}", i, fvals(rng, b, n, -5), claim_i=dict(b=b, dense=True, top=True)))
    # float64 pages of 15, 16 and 17 significant digits
    for digits, exp, b in ((15, -3, 9), (16, -2, 13), (17, -2, 18), (16, -8, 21), (15, -15, 16), (16, 0, 11)):
        n = 3000
        f = fvals(rng, b, n, exp, base=10 ** (digits - 1) + 123456789)
        # 17 digits are more than a float64 holds: the writer's decimal integers are the values' shortest forms, not the walk
        claim = dict(b=b) if digits < 17 else dict(dense=True)
        out.append(Blk(f"digits{digits} e{exp}", walk(rng, 4, [1] * (n - 1), 9), f, claim_f=dict(claim, exp=exp, digits=digits)))
    return out


def second_blocks(seed):
    """A smaller part: a few of the same kinds, for the two-part shape (it follows the main part in time)."""
    rng = np.random.default_rng(seed)
    out = []
    for b in (1, 4, 8, 13, 16, 19, 23):
        n = 1500 + 97 * b
        out.append(Blk(f"p2 b{b}", walk(rng, b, [narrow_len(b)] * (n - 1), 500), fvals(rng, b, n, -3),
                       claim_i=dict(b=b), claim_f=dict(b=b)))
    out.append(Blk("p2 one row", [42], [0.25]))
    return out


def make_part(blocks, t0=T0, sid0=1):
    sizes = [bk.n for bk in blocks]
    sids = np.repeat(np.arange(sid0, sid0 + len(blocks), dtype=np.uint64), sizes)
    ts = np.concatenate([t0 + np.arange(n, dtype=np.int64) * STEP for n in sizes])
    cat = lambda k: np.concatenate([getattr(bk, k) for bk in blocks])   # noqa: E731
    return build_part(sids, ts, np.ones(sids.size, np.int64), [("i", O.VT_INT64, cat("i"), None), ("f", O.VT_FLOAT64, cat("f"), None),
                                                                ("c", O.VT_INT64, cat("c"), None)]), np.unique(sids)


def part_pages(blocks):
    return [pg for bk in blocks for pg in ((bk.pi, bk.n, False), (bk.pf, bk.n, True), (bk.pc, bk.n, False))]


@pytest.fixture(scope="module")
def fixtures():
    main, second = main_blocks(0xDE45E), second_blocks(0x5EC0D)
    p1, s1 = make_part(main)
    p2, s2 = make_part(second, t0=T0 + 10_000 * STEP, sid0=1)
    return dict(main=main, second=second, parts=[(p1, s1), (p2, s2)])


# ------------------------------------------------------------------ CPU: the fixtures are what they claim
def _claims_hold(bk, page, d, claim, is_float):
    ctx = (bk.name, "f" if is_float else "i")
    vals, lens = page_values(page, bk.n, is_float) if page[0] == 3 else (None, None)
    if claim.get("kind") == "wide":
        assert page[0] == 3 and max(lens) == 4 and d is None, ctx
        return
    if "b" in claim:
        assert page[0] == 3, ctx   # EncodeTypeDelta: not monotone, not incremental
        assert (int(vals.max()) - int(vals.min())).bit_length() == claim["b"], ctx
        assert max(lens) <= 3, ctx
    if "dense" in claim or "b" in claim:
        assert (d is not None) == claim.get("dense", claim.get("b", 99) <= 23), (ctx, d, len(page))
    if d is not None and "b" in claim:
        assert d.b == claim["b"] and d.n == bk.n, ctx
    if claim.get("plane_bytes") is not None:
        assert d.plane_bytes == claim["plane_bytes"], (ctx, d)
    if "page" in claim:
        assert len(page) == claim["page"], (ctx, len(page))
    if "first" in claim:
        assert page_first(page, is_float) == claim["first"] and page[0] == 3, ctx
    if "exp" in claim:
        assert int.from_bytes(page[1:3], "big", signed=True) == claim["exp"], ctx
    if claim.get("neg"):
        assert vals[0] >= 0 and d.m < 0, ctx
    if claim.get("top"):
        assert d.m + bk.n * (1 << 20) > I64_MAX - (1 << 40) and (bk.n * d.m) > I64_MAX, ctx
    if "digits" in claim:
        assert len(str(abs(int(vals[0])))) == claim["digits"], (ctx, vals[0])


def test_fixture_blocks_are_what_they_claim(fixtures):
    for bk in fixtures["main"] + fixtures["second"]:
        _claims_hold(bk, bk.pi, bk.di, bk.claim_i, False)
        _claims_hold(bk, bk.pf, bk.df, bk.claim_f, True)
    # the float64 pages hold the decimal integers of the values (17 digits: the writer's shortest forms, which need not
    # convert back to the same float64)
    for bk in fixtures["main"]:
        if bk.pf[0] == 3 and bk.claim_f.get("digits", 0) < 17:
            ints = page_values(bk.pf, bk.n, True)[0]
            exp = int.from_bytes(bk.pf[1:3], "big", signed=True)
            assert O.decimal_list_to_float64(ints, exp).view(np.uint64).tolist() == bk.f.view(np.uint64).tolist(), bk.name


def test_every_plane_width_runs_for_both_types(fixtures):
    """each b from 1 to 23 has a converted page of each value type, so planes 16, 8, 4, 2 and 1 run in every combination"""
    for is_float in (False, True):
        bs = {(bk.df if is_float else bk.di).b for bk in fixtures["main"] if (bk.df if is_float else bk.di) is not None}
        assert set(range(1, 24)) <= bs, sorted(bs)
    # the model's pages are the part's pages, byte for byte
    for blocks, (part, _) in zip((fixtures["main"], fixtures["second"]), fixtures["parts"]):
        assert part.files()["fv.bin"] == b"".join(p for p, _, _ in part_pages(blocks))


def test_boundary_pairs_sit_on_either_side(fixtures):
    by = {bk.name: bk for bk in fixtures["main"]}
    for n, b in ((1024, 8), (700, 10), (3000, 9)):
        kept, conv = by[f"size n{n} b{b} kept"], by[f"size n{n} b{b} conv"]
        for page_k, page_c, dk, dc in ((kept.pi, conv.pi, kept.di, conv.di), (kept.pf, conv.pf, kept.df, conv.df)):
            assert len(page_k) == 32 + stream_bytes(n, b) and len(page_c) == len(page_k) + 1
            assert dk is None and dc is not None and dc.b == b
    for n in (3000, 8193):
        a, k = by[f"reach n{n} +0"], by[f"reach n{n} +1"]
        assert page_first(a.pi, False) == I64_MAX - (n << 20) and page_first(k.pi, False) == I64_MAX - (n << 20) + 1
        assert a.di is not None and k.di is None
        # the kept page fails the reach rule alone: its span and size would pass
        v = page_values(k.pi, n, False)[0]
        b = (int(v.max()) - int(v.min())).bit_length()
        assert b <= 14 and max(page_values(k.pi, n, False)[1]) <= 3 and 32 + stream_bytes(n, b) < len(k.pi)


def test_the_model_reads_the_writers_pages():
    """int_page / float_page are the oracle writer's column pages (column.go), and page_first its int64 order"""
    rng = np.random.default_rng(3)
    for v in (np.array([5, 9, 3, 4]), np.array([7]), walk(rng, 12, [2] * 99, 1 << 40), np.array([I64_MAX - 5, I64_MAX, 0])):
        raw = (v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)).astype(">u8").tobytes()
        assert int_page(v) == O.column_encode(O.VT_INT64, [raw[8 * k:8 * k + 8] for k in range(v.size)])
        if int_page(v)[0] == 3:
            assert page_values(int_page(v), v.size, False)[0].tolist() == v.tolist()
    for f in (np.array([1.25, 2.5, -0.75]), fvals(rng, 9, 50, -4), np.array([0.5])):
        raw = f.astype(">f8").tobytes()
        assert float_page(f) == O.column_encode(O.VT_FLOAT64, [raw[8 * k:8 * k + 8] for k in range(f.size)])
    for x in (0, 1, -1, I64_MAX, I64_MIN, 123456789):
        assert page_first(b"\x03" + O.conv_int64_to_bytes(x), False) == x


def _pin_pages_convert_nothing(blocks):
    for k, (page, n, is_float) in enumerate(blocks):
        assert dense_model(page, n, is_float) is None, (k, n, is_float, len(page))


def test_varint_pins_read_varints():
    """test_express_batch_handover and test_express_units_at_every_edge pin the SWAR varint decode: admission converts none of
    their pages, so an admission change that starts converting them fails here instead of moving their coverage."""
    from tests.test_gpu_express_units import _blocks
    _, _, vals = handover_blocks()
    _pin_pages_convert_nothing([(int_page(v), v.size, False) for v in vals])
    blocks, _ = _blocks(np.random.default_rng(4096))
    _pin_pages_convert_nothing([pg for _, v in blocks for pg in ((int_page(v), v.size, False), (float_page(v / 100.0), v.size, True))])


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def pair(bydb):
    on, off = bydb.Context(device=0), bydb.Context(device=0, dense_pages=False)
    yield on, off
    on.close()
    off.close()


def same_result(a, b, ctx):
    assert a.group_id.tolist() == b.group_id.tolist(), ctx
    assert a.rows.tolist() == b.rows.tolist(), ctx
    assert a.val_i64.tolist() == b.val_i64.tolist(), ctx
    assert a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist(), ctx


def same_rows(a, b, ctx):
    for k, y in b.items():
        if k == "stats":
            continue
        x = a[k]
        if isinstance(y, np.ndarray):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), (ctx, k)
        else:
            assert x == y, (ctx, k)


def block_class(bk, fields):
    """the lane class of a block for a query summing `fields`: every summed page must be a plain delta page"""
    kinds = [page_kind(bk.pi if fd == "i" else bk.pf, bk.n, fd == "f") for fd in fields]
    return SimpleNamespace(cls="wide" if "wide" in kinds else "delta" if all(k == "delta" for k in kinds) else "other")


def check_lanes(res, blocks, active, ctx):
    """express- and slow-lane blocks as lane_model predicts them for a query summing i and f; slow_lane_reasons holds 4 << k
    for each field k (the query's field order: i, f) whose page sent a block to the slow lane"""
    express, slow = lane_model([block_class(bk, ("i", "f")) for bk in blocks], active, True, True)
    reasons = 0
    for bk, (n_active, _) in zip(blocks, active):
        for k, (page, is_float) in enumerate(((bk.pi, False), (bk.pf, True))):
            if n_active and page_kind(page, bk.n, is_float) == "wide":
                reasons |= 4 << k
    st = res.stats
    assert (st.blocks_express_lane, st.blocks_slow_lane, st.slow_lane_reasons) == (express, slow, reasons), (ctx, st, express, slow, reasons)


def check_exact(res, blocks_by_sid, sids, groups, aggs, ctx):
    """int64 SUM = the python-int sum modulo 2^64 per group; float64 SUM within 1e-9 of the exact sum of decimal integers"""
    for a, (fd, fn) in enumerate(aggs):
        if fn != O.AGG_SUM:
            continue
        exact = {}
        for s, g in zip(sids.tolist(), groups.tolist()):
            for bk, lo, hi in blocks_by_sid.get(s, []):
                if fd == "i":
                    exact[g] = exact.get(g, 0) + sum(int(x) for x in bk.i[lo:hi])
                else:
                    ints, e = O.float64_to_decimal_list(bk.f[lo:hi]) if hi > lo else (np.zeros(0, np.int64), 0)
                    exact[g] = exact.get(g, Fraction(0)) + Fraction(int(sum(int(x) for x in ints))) * Fraction(10) ** int(e)
        for r, g in enumerate(res.group_id.tolist()):
            if fd == "i":
                w = exact[g] & MASK64
                assert int(res.val_i64[r, a]) & MASK64 == w, (ctx, g)
            else:
                w = exact[g]
                assert abs(Fraction(float(res.val_f64[r, a])) - w) <= Fraction(1, 10 ** 9) * max(abs(w), Fraction(1, 10 ** 300)), (ctx, g)


SUMS = [(fd, fn) for fd in ("i", "f") for fn in (O.AGG_SUM, O.AGG_COUNT, O.AGG_MEAN)]


def _register(ctx, parts, pid0):
    return [ctx.register_part(pid0 + k, p.files()) for k, (p, _) in enumerate(parts)]


def _release(ctx, hs):
    for h in hs:
        ctx.release_part(h)


def check_part_info(ctx, h, blocks, dense_on):
    info = ctx.part_info(h)
    n, pb = expected_dense(part_pages(blocks))
    _, cols = ctx.part_directory(h)
    if not dense_on or n == 0:
        assert info["dense_pages"] == 0 and info["dense_bytes"] == 0, info
    else:
        assert info["dense_pages"] == n, (info, n)
        assert info["dense_bytes"] == align_up(cols.shape[0] * 32, 256) + align_up(pb, 256), (info, cols.shape, pb)
    return info


@gpu
@pytest.mark.parametrize("shape", ["series", "groups", "top_desc", "top_asc", "two_parts", "cut"])
def test_dense_boundaries_answer_like_the_reference(bydb, pair, fixtures, shape):
    on, off = pair
    ps = fixtures["parts"] if shape == "two_parts" else fixtures["parts"][:1]
    blocks = fixtures["main"] + (fixtures["second"] if shape == "two_parts" else [])
    sids = np.unique(np.concatenate([s for _, s in ps]))
    kw, tmin, tmax = {}, I64_MIN, I64_MAX
    groups = np.arange(sids.size, dtype=np.int32)
    if shape in ("groups", "two_parts"):
        groups = (np.arange(sids.size) % 5).astype(np.int32)
    if shape.startswith("top"):
        kw = dict(top_n=9, top_agg=0, top_desc=shape == "top_desc")
    if shape == "cut":
        tmax = T0 + 3000 * STEP   # blocks of more than 3,001 rows are cut: the fast lane reads their reference pages
    oq = O.Query([p for p, _ in ps], sids, SUMS, groups=groups, n_groups=int(groups.max()) + 1, tmin=tmin, tmax=tmax, **kw)
    h_on, h_off = _register(on, ps, 10), _register(off, ps, 10)
    try:
        for h, bl in zip(h_on, (fixtures["main"], fixtures["second"])):
            check_part_info(on, h, bl, True)
        r_on, r_off = on.scan_agg(to_gpu_query(bydb, h_on, oq)), off.scan_agg(to_gpu_query(bydb, h_off, oq))
    finally:
        _release(on, h_on)
        _release(off, h_off)
    same_result(r_on, r_off, shape)
    assert_parity(r_on, O.run_query(oq), SUMS, shape)
    # rows of every series the query keeps, by part
    by_sid, active = {}, []
    t_parts = [T0, T0 + 10_000 * STEP]
    for (part_blocks, t0) in zip((fixtures["main"], fixtures["second"])[:len(ps)], t_parts):
        for k, bk in enumerate(part_blocks):
            ts = t0 + np.arange(bk.n, dtype=np.int64) * STEP
            keep = (ts >= tmin) & (ts <= tmax)
            lo, hi = (int(np.argmax(keep)), int(keep.size - np.argmax(keep[::-1]))) if keep.any() else (0, 0)
            by_sid.setdefault(k + 1, []).append((bk, lo, hi))
            active.append((int(keep.sum()), bool(keep.all())))
    check_exact(r_on, by_sid, sids, groups, SUMS, shape)
    s_on, s_off = r_on.stats, r_off.stats
    assert s_on.blocks_express_lane == s_off.blocks_express_lane and s_on.page_bytes == s_off.page_bytes, (s_on, s_off)
    check_lanes(r_on, blocks, active, f"{shape} on")
    check_lanes(r_off, blocks, active, f"{shape} off")


@gpu
def test_dense_boundaries_prepared_graph_and_partials(bydb, pair, fixtures):
    """graph replay past its third run, run_partials, and three release / register rounds with the same answers and dense bytes"""
    on, off = pair
    (p, sids), _ = fixtures["parts"]
    groups = (np.arange(sids.size) % 3).astype(np.int32)
    oq = O.Query([p], sids, SUMS, groups=groups, n_groups=3)
    want = O.run_query(oq)
    first, infos = None, []
    for rnd in range(3):
        h_on, h_off = on.register_part(20, p.files()), off.register_part(20, p.files())
        infos.append(check_part_info(on, h_on, fixtures["main"], True)["dense_bytes"])
        check_part_info(off, h_off, fixtures["main"], False)
        g_on, g_off = on.prepare_graph(to_gpu_query(bydb, [h_on], oq)), off.prepare_graph(to_gpu_query(bydb, [h_off], oq))
        try:
            for it in range(5):
                r_on, r_off = g_on.run(), g_off.run()
                same_result(r_on, r_off, f"graph round {rnd} run {it}")
                assert_parity(r_on, want, SUMS, f"graph round {rnd} run {it}")
                if first is None:
                    first = r_on
                same_result(r_on, first, f"round {rnd} run {it} against the first run")
            same_rows(g_on.run_partials(), g_off.run_partials(), f"partials round {rnd}")
        finally:
            g_on.close()
            g_off.close()
            on.release_part(h_on)
            off.release_part(h_off)
    assert len(set(infos)) == 1 and infos[0] > 0, infos


@gpu
def test_dense_boundaries_budget_edges(bydb, pair, fixtures):
    on, off = pair
    (p, _), (q, _) = fixtures["parts"]
    sizes = {}
    for name, part in (("p", p), ("q", q)):
        h_on, h_off = on.register_part(30, part.files()), off.register_part(30, part.files())
        sizes[name] = (on.part_info(h_on)["hbm_bytes"], off.part_info(h_off)["hbm_bytes"])
        on.release_part(h_on)
        off.release_part(h_off)
    p_on, p_off = sizes["p"]
    q_on, _ = sizes["q"]
    assert p_on > p_off
    with bydb.Context(device=0, hbm_budget_bytes=p_on) as exact:   # exactly the dense-on size admits the part
        h = exact.register_part(1, p.files())
        check_part_info(exact, h, fixtures["main"], True)
        exact.release_part(h)
    budget = p_off + 1   # the part's pages fit, their dense form does not
    # the second part fits the budget only if the refused part left nothing reserved
    assert q_on <= budget and q_on > budget - p_off, (sizes, budget)
    with bydb.Context(device=0, hbm_budget_bytes=budget) as tight:
        with pytest.raises(bydb.BydbError) as ei:
            tight.register_part(1, p.files())
        assert ei.value.code == bydb.capi.ENOMEM
        h = tight.register_part(2, q.files())
        check_part_info(tight, h, fixtures["second"], True)
        tight.release_part(h)


# ------------------------------------------------------------------ dense and varint pages in one express batch
def batch_blocks(seed, n_pad=72_000, n_front=64):
    """8-block patterns at the front of a ~72k-block part (a warp grabs 8 blocks while more than 16 per warp are left), each
    rotated by its index so every kind meets every batch position: dense pages of 1 to 4 stages, varint pages of 3-byte
    varints over several stages, a 1-row block, a short dense stream behind a long varint page (its ring slot still holds the
    varint page's bytes), a block with a 4-byte varint, and a block whose int64 page is dense while its float64 page bails out."""
    rng = np.random.default_rng(seed)

    def kind(k):
        if k == "dense1":
            return Blk(k, walk(rng, 8, [2] * 1999, 300), fvals(rng, 6, 2000, -2))
        if k == "varint3":
            return Blk(k, walk(rng, 24, [3] * 2999, 300), fvals(rng, 24, 3000, -1, lengths=[3] * 2999))
        if k == "dense2":
            return Blk(k, walk(rng, 12, [2] * 3999, 300), fvals(rng, 11, 4000, -3))
        if k == "one":
            return Blk(k, [int(rng.integers(0, 100))], [0.5])
        if k == "short":
            return Blk(k, walk(rng, 1, [1] * 99, 300), fvals(rng, 2, 100, -2))
        if k == "wide":
            i = walk(rng, 5, [1] * 1999, 300)
            i[1000:] += WIDE + 64
            return Blk(k, i, fvals(rng, 5, 2000, -2))
        if k == "dense4":
            return Blk(k, walk(rng, 16, [3] * 8191, 300), fvals(rng, 16, 8192, -4))
        if k == "split":   # int64 dense, float64 with a 4-byte varint: the whole block goes to the fast lane
            f = walk(rng, 6, [1] * 2499, 10 ** 6 + 3)
            f[1200:] += WIDE + 64
            return Blk(k, walk(rng, 9, [2] * 2499, 300), f / 100.0)
        raise KeyError(k)
    # the short stream always follows the long varint page
    units = [["dense1"], ["varint3", "short"], ["dense2"], ["one"], ["wide"], ["dense4"], ["split"]]
    out = []
    for r in range(n_front // 8):
        out += [kind(k) for u in units[r % 7:] + units[:r % 7] for k in u]
    pad_i = [walk(rng, 5, [1] * 23, 40) for _ in range(4)]
    pad = [Blk("pad", pad_i[k], pad_i[k] / 100.0) for k in range(4)]
    out += [pad[k % 4] for k in range(n_pad)]
    return out


@pytest.fixture(scope="module")
def batch_fixture():
    blocks = batch_blocks(0xBA7C)
    part, sids = make_part(blocks)
    return blocks, part, sids


def test_batch_fixture_mixes_forms(batch_fixture):
    blocks, part, _ = batch_fixture
    front = blocks[:64]
    stages = {bk.di.plane_bytes // STAGE + (bk.di.plane_bytes % STAGE > 0) for bk in front if bk.di is not None}
    assert {1, 2, 4} <= stages, stages
    assert any(bk.di is None and page_kind(bk.pi, bk.n, False) == "delta" and len(bk.pi) > 2 * STAGE for bk in front)
    for a, b in zip(front, front[1:]):
        if b.name == "short":
            assert a.name == "varint3" and b.di is not None and b.di.plane_bytes == 16
    split = [bk for bk in front if bk.name == "split"]
    assert split and all(bk.di is not None and page_kind(bk.pf, bk.n, True) == "wide" for bk in split)
    assert all(bk.di is None and bk.df is None for bk in blocks[64:70])   # the padding keeps its varints
    assert part.files()["fv.bin"] == b"".join(p for p, _, _ in part_pages(blocks))


@gpu
def test_dense_and_varint_pages_in_one_express_batch(bydb, pair, batch_fixture):
    on, off = pair
    blocks, part, sids = batch_fixture
    aggs = [("i", O.AGG_SUM), ("i", O.AGG_COUNT), ("f", O.AGG_SUM), ("f", O.AGG_MEAN), ("c", O.AGG_COUNT)]
    groups = (np.arange(sids.size) % 4096).astype(np.int32)
    oq = O.Query([part], sids, aggs, groups=groups, n_groups=4096)
    h_on, h_off = on.register_part(40, part.files()), off.register_part(40, part.files())
    try:
        check_part_info(on, h_on, blocks, True)
        r_on, r_off = on.scan_agg(to_gpu_query(bydb, [h_on], oq)), off.scan_agg(to_gpu_query(bydb, [h_off], oq))
    finally:
        on.release_part(h_on)
        off.release_part(h_off)
    same_result(r_on, r_off, "batch")
    assert_parity(r_on, O.run_query(oq), aggs, "batch")
    check_exact(r_on, {k + 1: [(bk, 0, bk.n)] for k, bk in enumerate(blocks)}, sids, groups, aggs, "batch")
    assert r_on.stats.page_bytes == r_off.stats.page_bytes
    check_lanes(r_on, blocks, [(bk.n, True) for bk in blocks], "batch on")
    check_lanes(r_off, blocks, [(bk.n, True) for bk in blocks], "batch off")

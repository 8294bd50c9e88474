"""Delta-of-delta pages (EncodeTypeDeltaOfDelta, enc 4) against the oracle at the boundaries where their decoders carry state.

The writer picks delta-of-delta for every ascending or descending list that is not constant-step (every irregular timestamp
page), for counters with a few resets and for any list whose first value is negative (int_list.go:27-53).  Three decoders read
such a page:

  field page, second differences <= 3 bytes                -> dod_page_fast (32 B lanes, 1 KB chunks, two per 2 KB TMA stage)
  field page with a 4+ byte second difference               -> bail-out of dod_page_fast (stream_drain), block to the slow lane,
                                                               decode_varint_page<true> (16 B lanes, 512 B chunks)
  timestamp page cut by the time range, int64 tag page,     -> decode_varint_page<true> in the slow lane (TsCons, CmpCons,
  timestamps of overlapping parts                              decode_list_to)

dod_page_fast reads the first difference alone, then streams the second differences from the unaligned byte after it, so
where that byte falls in its 16 B-aligned copy (the body start) shifts every lane and chunk edge.  The sweeps here place
one varint at each lane, chunk and stage edge of either decoder for each body start, and every query is checked three ways:
against the oracle (assert_parity), against a plain fold over the generated values (Python ints mod 2^64 for int64,
math.fsum for float64 sums), and through the lane counters (blocks_slow_lane, slow_lane_reasons).

Values are int64 mantissas: an int64 field stores them as they are, a float64 field stores mantissa / 100 (exponent -2).
"""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_lanes import (ALL5, LIMIT_DELTAS, MINMAX, NARROW3, SUMS, WIDE, assert_lanes, lane_model, page_class,
                                  shape_values)

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "skywalking-banyandb_b200", "csrc")
M64 = 1 << 64
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
_pid = [90_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def wrap(x):
    """a Python int reduced to int64 the way Go's int64 arithmetic wraps"""
    x &= M64 - 1
    return x - M64 if x >= (1 << 63) else x


def varint_lengths(body):
    lens, run = [], 0
    for b in body:
        run += 1
        if b < 0x80:
            lens.append(run)
            run = 0
    assert run == 0, "truncated varint"
    return lens


def from_dod(first, d1, sd):
    """values first, first + d1, ... whose second differences are sd, wrapping mod 2^64 like the writer's arithmetic"""
    steps = np.concatenate([[np.int64(d1)], np.asarray(sd, dtype=np.int64)]).astype(np.uint64)
    diffs = np.cumsum(steps, dtype=np.uint64)                       # running first difference (mod 2^64)
    v = np.uint64(first % M64) + np.concatenate([[np.uint64(0)], np.cumsum(diffs, dtype=np.uint64)])
    return v.view(np.int64)


def page_kind(m):
    """-> (enc, class) of one block's values as the writer encodes them; class 'dod_wide' is a delta-of-delta page whose
    second differences include a varint of 4+ bytes (the fast lane bails out; the first difference is read on its own and
    may be any width), 'wide' the same for a delta page."""
    body, enc, first = O.int64_list_encode(np.asarray(m, dtype=np.int64))
    assert first == m[0]
    if enc == 4:
        lens = varint_lengths(body)
        return enc, ("dod_wide" if max(lens[1:], default=0) > 3 else "dod")
    if enc == 3:
        return enc, ("wide" if max(varint_lengths(body)) > 3 else "delta")
    return enc, {1: "const", 2: "delta_const"}[enc]


class Blk:
    """one series = one block: timestamps, int64 mantissas and the page class lane_model reads ('wide' = bails out)"""

    def __init__(self, sid, ts, m, is_float=False):
        self.sid, self.ts, self.m = sid, np.asarray(ts, np.int64), np.asarray(m, np.int64)
        self.enc, kind = page_kind(self.m)
        if is_float and self.m.size > 1:
            page_class(self.m, None, True)   # asserts that mantissa / 100 stores the same mantissas with exponent -2
        self.kind = kind
        self.cls = "wide" if kind in ("wide", "dod_wide") else kind


def regular_ts(n):
    return T0 + np.arange(n, dtype=np.int64) * STEP


class _Builder(O.PartBuilder):
    """PartBuilder whose string columns may also be given as (codes, palette), cells palette[codes]: the cell table is
    filled with numpy instead of one ctypes buffer per cell (the boundary sweeps write millions of rows)"""

    @staticmethod
    def _column(name, vt, values, nulls, keep):
        if not isinstance(values, tuple):
            return O.PartBuilder._column(name, vt, values, nulls, keep)
        codes, palette = values
        bufs = [C.create_string_buffer(v, max(len(v), 1)) for v in palette]
        arr = (O._Bytes * max(codes.size, 1))()
        cells = np.frombuffer(arr, dtype=[("p", np.uint64), ("len", np.int64)], count=codes.size)
        cells["p"] = np.array([C.addressof(b) for b in bufs], dtype=np.uint64)[codes]
        cells["len"] = np.array([len(v) for v in palette], dtype=np.int64)[codes]
        col = O._Column()
        nb = name.encode()
        keep.extend([arr, bufs, nb])
        col.name = nb
        col.value_type = vt
        col.bytes = arr
        return col


def make_part(blocks, is_float, version=1, tags=True):
    """one part, one block per series: the field `v`, a dictionary tag `region` and a narrow delta int64 tag `code` (the
    fast lane compares it itself, so the only reason a block leaves the fast lane is its field page)."""
    sids = np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks])
    ts = np.concatenate([b.ts for b in blocks])
    m = np.concatenate([b.m for b in blocks])
    rows = np.concatenate([np.arange(b.m.size, dtype=np.int64) for b in blocks])
    region = ((rows * 7 + sids.astype(np.int64)) % 3, [b"r0", b"r1", b"r2"])
    code = np.where(rows == 0, 3, np.where(rows == 1, 1, 1 + (rows * 5 + sids.astype(np.int64)) % 3)).astype(np.int64)
    vt = O.VT_FLOAT64 if is_float else O.VT_INT64
    b = _Builder()
    b.append(sids, ts, np.full(sids.size, version, np.int64), [("v", vt, m / 100.0 if is_float else m, None)],
             [("default", [("region", O.VT_STR, region, None), ("code", O.VT_INT64, code, None)])] if tags else [])
    return b.finish()


def mode_keep(b, mode):
    """rows of block b the predicate of `mode` keeps (the time range is applied separately)"""
    r = np.arange(b.m.size, dtype=np.int64)
    if mode == "dict_mask":
        return (r * 7 + b.sid) % 3 == 1
    if mode == "int_mask":
        return np.where(r == 0, 3, np.where(r == 1, 1, 1 + (r * 5 + b.sid) % 3)) != 2
    return np.ones(b.m.size, bool)


MODE_PREDS = {"dict_mask": [O.Pred("default", "region", O.OP_EQ, b"r1")], "int_mask": [O.Pred("default", "code", O.OP_NE, 2)]}


def got_value(got, r, a):
    return float(got.val_f64[r, a]) if got.is_float[a] else int(got.val_i64[r, a])


def check_model(got, mants, keeps, aggs, is_float, ctx, cols=None):
    """the query result against a plain fold over the generated values (one group per block, in block order); cols[i]: the
    result column of aggs[i] (default: i)"""
    cols = list(range(len(aggs))) if cols is None else cols
    want_groups = [i for i, k in enumerate(keeps) if k.any()]
    assert got.group_id.tolist() == want_groups, f"{ctx}: groups"
    for r, gi in enumerate(want_groups):
        x = mants[gi][keeps[gi]]
        cnt = int(x.size)
        assert int(got.rows[r]) == cnt, f"{ctx}: rows of group {gi}"
        xs = x.tolist()                                   # Python ints
        for (_, f), a in zip(aggs, cols):
            g = got_value(got, r, a)
            if f == O.AGG_COUNT:
                assert g == cnt, f"{ctx}: count of group {gi}"
                continue
            if not is_float:
                s = wrap(sum(xs))
                want = {O.AGG_SUM: s, O.AGG_MIN: min(xs), O.AGG_MAX: max(xs)}.get(f)
                if f == O.AGG_MEAN:
                    q = abs(s) // cnt * (1 if s >= 0 else -1)   # Go's division truncates toward zero
                    want = q if q >= 1 else 1
                assert g == want, f"{ctx}: int64 agg {f} of group {gi}: {g} vs {want}"
            elif f in (O.AGG_MIN, O.AGG_MAX):
                want = np.float64(min(xs) if f == O.AGG_MIN else max(xs)) / 100.0
                assert np.float64(g).view(np.uint64) == want.view(np.uint64), f"{ctx}: float64 agg {f} of group {gi}: {g} vs {want}"
            else:
                want = math.fsum((x / 100.0).tolist())
                if f == O.AGG_MEAN:
                    want = want / cnt
                    want = want if want >= 1 else 1.0
                assert abs(g - want) <= 1e-9 * max(abs(want), 1e-300), f"{ctx}: float64 agg {f} of group {gi}: {g} vs {want}"


class Registered:
    """parts registered once on the GPU for many queries (one group per series of blocks)"""

    def __init__(self, bydb, ctx, parts):
        self.bydb, self.ctx, self.parts = bydb, ctx, parts
        pid = _next_pid()
        self.handles = [ctx.register_part(pid + i, p.files()) for i, p in enumerate(parts)]

    def close(self):
        for h in self.handles:
            self.ctx.release_part(h)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def run(self, usid, aggs, tmin=I64_MIN, tmax=I64_MAX, preds=()):
        oq = O.Query(self.parts, usid, aggs, groups=np.arange(usid.size, dtype=np.int32), n_groups=usid.size, tmin=tmin, tmax=tmax,
                     preds=list(preds))
        got = self.ctx.scan_agg(to_gpu_query(self.bydb, self.handles, oq))
        return got, O.run_query(oq)


def run_modes(bydb, gpu_ctx, blocks, is_float, modes, aggsets, tag, extra_parts=(), older_keep=None, model_mants=None):
    """every mode x aggregate set over one part (one group per block): parity, the model and the lane counters.
    extra_parts: newer parts that shadow rows of this one; older_keep(b): the rows of block b they leave to it, and
    model_mants: the values the query then sees."""
    part = make_part(blocks, is_float)
    usid = np.array([b.sid for b in blocks], dtype=np.uint64)
    mants = model_mants if model_mants is not None else [b.m for b in blocks]
    with Registered(bydb, gpu_ctx, [part, *extra_parts]) as reg:
        for mode in modes:
            tmin, tmax = I64_MIN, I64_MAX
            if mode == "range":
                tmin, tmax = T0 + STEP, T0 + 3000 * STEP       # cuts row 0 of every block and the tail of the long ones
            preds = MODE_PREDS.get(mode, [])
            in_range = [(b.ts >= tmin) & (b.ts <= tmax) for b in blocks]
            keeps = [mode_keep(b, mode) & t for b, t in zip(blocks, in_range)]
            older = [k & older_keep(b) for k, b in zip(keeps, blocks)] if older_keep else keeps
            active = [(int(k.sum()), bool(t.all())) for k, t in zip(older, in_range)]
            for aggset in aggsets:
                aggs = [("v", f) for f in aggset]
                got, want = reg.run(usid, aggs, tmin, tmax, preds)
                ctx = f"{tag}/{mode}/{'f64' if is_float else 'i64'}/{[f for _, f in aggs]}"
                assert_parity(got, want, aggs, ctx)
                check_model(got, mants, keeps, aggs, is_float, ctx)
                express, slow = lane_model(blocks, active, aggset is SUMS, mode == "all" and not extra_parts)
                assert_lanes(got, express, slow, ctx)


# ------------------------------------------------------------------ 1. a varint at every boundary of either decoder
# dod_page_fast: 32 B lanes, 1 KB chunks, 2 KB stages (k = 64: the second stage, k = 128: the third, which reuses ring slot 0),
# in the coordinates of the 16 B-aligned copy of the second differences; decode_varint_page: 16 B lanes, 512 B chunks, in the
# coordinates of the aligned copy of the whole body
FAST_EDGES = [32 * k for k in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129)]
SLOW_EDGES = [16 * k for k in (1, 2, 31, 32, 33, 127, 128, 129)]
D1_WIDTHS = (1, 2, 3, 5, 9, 10)
FLOAT_D1_WIDTHS = (1, 2, 3, 5)   # mantissas stay below 2^53: mantissa / 100 keeps exponent -2
WIDTHS = (3, 4, 10)


def d1_of(d1_width):
    """the smallest positive first difference whose zig-zag varint takes d1_width bytes (10 bytes: 2^62 + 2^21, so that a
    10-byte negative second difference leaves the step positive)"""
    if d1_width == 1:
        return 5
    if d1_width == 10:
        return (1 << 62) + (1 << 21)
    return 1 << (7 * (d1_width - 1) - 1)


def dod_at(p, n, width, d1_width):
    """int64 values of one block whose delta-of-delta body holds a d1_width-byte first difference, then 1-byte second
    differences (+1, -1, ... around an ascending step) except one width-byte second difference starting at body byte p."""
    d1 = d1_of(d1_width)
    j = p - d1_width                         # index of the wide one among the second differences
    assert 0 <= j < n - 2
    sd = np.where(np.arange(n - 2) % 2 == 0, 1, -1).astype(np.int64)
    if width == 10:
        step = d1 + (j % 2)                  # the first difference in front of it
        sd[j] = (1 << 62) if step < (1 << 62) else -((1 << 62) + 1)
    else:
        sd[j] = WIDE if width == 4 else NARROW3
    return from_dod(1000, d1, sd)


def sweep(width, is_float):
    """The blocks of one boundary sweep, in part order: for each first-difference width, each edge of either geometry and each
    position within width + 2 bytes of it, the body byte p that puts the width-byte varint there.  A field page is
    [enc][exponent (float64)][first, 8 bytes][body] and fv.bin holds the pages one after the other, 256 B aligned on the
    device, so the body starts at (page offset + header) mod 16 in its aligned copy and the second differences at that plus
    the first difference's width.  Each page is 7 bytes longer than a multiple of 16, so consecutive blocks step through all
    16 starts.  Odd positions get a 600-row tail, so a bail-out in one stage finds the next in flight."""
    hdr = 11 if is_float else 9
    off, out = 0, []
    for d1w in (FLOAT_D1_WIDTHS if is_float else D1_WIDTHS):
        for geo, edges in (("fast", FAST_EDGES), ("slow", SLOW_EDGES)):
            for e in edges:
                for s in range(e - width - 2, e + width + 3):
                    body_start = (off + hdr) & 15
                    stream_start = (body_start + d1w) & 15
                    p = d1w + s - stream_start if geo == "fast" else s - body_start
                    if p < d1w:
                        continue                 # inside the first difference: nothing to place
                    n = p - d1w + 48 + (600 if s % 2 else 0)
                    n += (7 - (hdr + d1w + (n - 3) + width)) % 16   # page length = 7 mod 16: the next body starts 7 bytes on
                    out.append(dict(d1w=d1w, geo=geo, edge=e, s=s, p=p, n=n, off=off, body_start=body_start, stream_start=stream_start))
                    off += hdr + d1w + (n - 3) + width
    return out


def sweep_blocks(width, is_float):
    spec = sweep(width, is_float)
    return spec, [Blk(i + 1, regular_ts(d["n"]), dod_at(d["p"], d["n"], width, d["d1w"])) for i, d in enumerate(spec)]


@pytest.mark.parametrize("width", WIDTHS)
def test_dod_at_places_the_varint(width):
    """The layout the boundary sweep rests on, checked against the oracle's encoder: a delta-of-delta page whose first varint
    takes d1_width bytes, whose second differences are 1-byte varints but the one of `width` bytes starting at body byte p."""
    for d1w in D1_WIDTHS:
        for p in sorted({d1w, d1w + 1, 31, 32, 33, 511, 512, 1023, 1024, 2047, 2048, 4095, 4096, 4127, 4140}):
            if p < d1w:
                continue
            n = p - d1w + 48
            v = dod_at(p, n, width, d1w)
            body, enc, first = O.int64_list_encode(v)
            assert enc == 4 and first == 1000, (d1w, p)
            lens = varint_lengths(body)
            j = 1 + p - d1w
            assert len(lens) == n - 1 and lens[0] == d1w and lens[j] == width, (d1w, p)
            assert set(lens[1:j] + lens[j + 1:]) == {1} and sum(lens[:j]) == p, (d1w, p)
            assert page_kind(v)[1] == ("dod" if width == 3 else "dod_wide")
            assert O.int64_list_decode(body, enc, first, n).tolist() == v.tolist()
            if width != 10 and d1w in FLOAT_D1_WIDTHS:
                assert page_class(v, None, True) == "dod"    # exponent -2, the same mantissas


@pytest.fixture(scope="module")
def dump_exe(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = tmp_path_factory.mktemp("dump") / "part_dir_dump"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", str(exe), os.path.join(ROOT, "tests", "native", "part_dir_dump.cc"),
                           os.path.join(CSRC, "part_dir.cc"), "-ldl", "-lpthread"])
    return str(exe)


def field_pages(exe, tmp_path, part):
    """(offset, size) of every block's field page, from the part's block directory as the library parses it"""
    d = tmp_path / "part"
    d.mkdir()
    for k, v in part.files().items():
        (d / k).write_bytes(v)
    out = subprocess.run([exe, str(d)], input="", capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("RC 0"), out.stdout[:500] + out.stderr
    files = next(line.split()[1:] for line in out.stdout.splitlines() if line.startswith("FILES"))
    pages = []
    for line in out.stdout.splitlines():
        if line.startswith("C "):
            _, name_id, vt, off, size, fid = line.split()
            if files[int(fid)] == "fv.bin":
                pages.append((int(off), int(size)))
    return pages


@pytest.mark.parametrize("width,is_float", [(3, False), (10, False), (4, True)], ids=["3-int64", "10-int64", "4-float64"])
def test_sweep_covers_every_body_start(dump_exe, tmp_path, width, is_float):
    """The sweep's claims against the part itself: file images sit 256 B aligned on the device (capi.cu: the arena places
    each file 256 B aligned), so a page's bytes fall in their 16 B-aligned copy at (page offset + header) mod 16.  The page
    offsets the sweep computes are the directory's; every body start 0..15 and every second-difference start 0..15 occurs;
    and each block's wide varint starts at the intended byte of its aligned copy."""
    spec, blocks = sweep_blocks(width, is_float)
    part = make_part(blocks, is_float, tags=False)
    pages = field_pages(dump_exe, tmp_path, part)
    hdr = 11 if is_float else 9
    assert len(pages) == len(spec)
    for d, b, (off, size) in zip(spec, blocks, pages):
        body, enc, _ = O.int64_list_encode(b.m)
        assert enc == 4 and off == d["off"] and size == hdr + len(body), d
        lens = varint_lengths(body)
        j = 1 + d["p"] - d["d1w"]
        assert lens[j] == width and sum(lens[:j]) == d["p"], d
        base = d["stream_start"] - d["d1w"] if d["geo"] == "fast" else d["body_start"]
        assert base + d["p"] == d["s"], d
    for geo in ("fast", "slow"):
        for d1w in (FLOAT_D1_WIDTHS if is_float else D1_WIDTHS):
            sel = [d for d in spec if d["geo"] == geo and d["d1w"] == d1w]
            key = "stream_start" if geo == "fast" else "body_start"
            assert {d[key] for d in sel} == set(range(16)), (geo, d1w)
            # (the first 16 bytes of a body may all belong to a wide first difference)
            assert {d["edge"] for d in sel} >= set(FAST_EDGES if geo == "fast" else SLOW_EDGES[1:])


@gpu
@pytest.mark.parametrize("width", WIDTHS)
def test_varint_at_every_boundary(bydb, gpu_ctx, width):
    """One block per series, one group per series.  3-byte second differences: no block leaves dod_page_fast; 4- and 10-byte:
    every block bails out of it (reason 4 << 0, the first field) and the slow lane's decode_varint_page answers."""
    for is_float in ((False, True) if width != 10 else (False,)):
        _, blocks = sweep_blocks(width, is_float)
        assert all(b.kind == ("dod" if width == 3 else "dod_wide") for b in blocks)
        run_modes(bydb, gpu_ctx, blocks, is_float, ["all", "range", "dict_mask", "int_mask"], (SUMS, ALL5), f"{width}-byte")


@gpu
def test_narrow_page_after_a_wide_one(bydb, gpu_ctx):
    """Two fields per block: `w` holds a 4-byte second difference in the first stage of a three-stage page, `n` only narrow
    ones.  In the slow lane one warp decodes w (dod_page_fast bails out, drains the stage in flight, decode_varint_page takes
    the page) and then n with dod_page_fast on the same ring; with n first, n is done in the fast lane and w defers the block
    (reason 4 << 1)."""
    rng = np.random.default_rng(41)
    n = 4300
    bw, bn = [], []
    for i in range(64):
        d1w = D1_WIDTHS[i % len(D1_WIDTHS)]
        bw.append(Blk(i + 1, regular_ts(n), dod_at(d1w + 40 + 31 * i, n, 4, d1w)))
        bn.append(Blk(i + 1, regular_ts(n), 500 + np.concatenate([[0], np.cumsum(3000 + rng.integers(0, 2000, n - 1))])))
    assert all(b.kind == "dod_wide" for b in bw) and all(b.kind == "dod" for b in bn)
    sids = np.concatenate([np.full(n, b.sid, np.uint64) for b in bw])
    ts = np.concatenate([b.ts for b in bw])
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("w", O.VT_INT64, np.concatenate([b.m for b in bw]), None),
                                                               ("n", O.VT_INT64, np.concatenate([b.m for b in bn]), None)])
    usid = np.array([b.sid for b in bw], dtype=np.uint64)
    keeps = [np.ones(n, bool)] * len(bw)
    with Registered(bydb, gpu_ctx, [part]) as reg:
        for order in (("w", "n"), ("n", "w")):
            for aggset in (SUMS, ALL5):
                aggs = [(f, a) for f in order for a in aggset]
                got, want = reg.run(usid, aggs)
                ctx = f"wide then narrow/{order}/{aggset}"
                assert_parity(got, want, aggs, ctx)
                for f in order:
                    cols = [a for a, (ff, _) in enumerate(aggs) if ff == f]
                    check_model(got, [b.m for b in (bw if f == "w" else bn)], keeps, [aggs[a] for a in cols], False, f"{ctx}/{f}", cols)
                assert got.stats.blocks_slow_lane == len(bw), ctx
                assert got.stats.slow_lane_reasons == 4 << order.index("w"), ctx


# ------------------------------------------------------------------ 2. the shape matrix
DOD_SHAPES = ["c1", "c2", "c3", "limits", "desc", "reset1", "reset2", "resets_wide", "negwalk1", "negwalk3"]
DOD_SIZES = [2, 3, 31, 32, 33, 1023, 1024, 1025, 2049, 4097, 8193]


def dod_shape(kind, n, rng):
    """int64 mantissas of one block of `kind`: monotone counters with 1-, 2- and 3-byte second differences, second differences
    at the zig-zag limits, a strictly descending list, counters with 1 / 2 narrow resets and with a wide reset every 64 rows
    (fewer than n/8 resets: still delta-of-delta), random walks from a negative first value."""
    first = 1000 + int(rng.integers(0, 1000)) * 10 + 3
    k = n - 1
    if kind in ("c1", "c2", "c3"):
        spread = {"c1": 32, "c2": 4096, "c3": 1 << 19}[kind]
        return first + np.concatenate([[0], np.cumsum((1 << 20) + rng.integers(0, spread, k))]).astype(np.int64)
    if kind == "limits":
        sd = np.resize(np.array(LIMIT_DELTAS, dtype=np.int64), max(k - 1, 0))
        return from_dod(first, 1 << 31, sd)[:n]
    if kind == "desc":
        return first + (1 << 40) - np.concatenate([[0], np.cumsum(1 + rng.integers(0, 4096, k))]).astype(np.int64)
    if kind in ("reset1", "reset2", "resets_wide"):
        start, step = ((1 << 30), 1 << 10) if kind == "resets_wide" else (first, 30)
        resets = {"reset1": {max(n // 2, 2)}, "reset2": {max(n // 3, 2), max((2 * n) // 3, 3)}}.get(kind, set(range(64, n, 64)))
        v, cur = [], start
        for i in range(n):
            if i in resets:
                cur = int(rng.integers(0, min(100, (cur >> 3) + 1)))   # a reset: at most an eighth of the value before
            elif i > 0:
                cur += step + int(rng.integers(0, 8))
            v.append(cur)
        return np.array(v, dtype=np.int64)
    # negative-first random walks: steps in [-K, K], so second differences up to 2K
    K = 63 if kind == "negwalk1" else (1 << 19) - 1
    return -(1 << 40) - first + np.concatenate([[0], np.cumsum(rng.integers(-K, K + 1, k))]).astype(np.int64)


def _shape_blocks(is_float, seed):
    rng = np.random.default_rng(seed)
    blocks, sid = [], 1
    for kind in DOD_SHAPES:
        for n in DOD_SIZES:
            m = dod_shape(kind, n, rng)
            assert m.size == n
            blocks.append(Blk(sid, regular_ts(n), m, is_float))
            blocks[-1].shape = kind
            sid += 1
    return blocks


def test_dod_shapes_are_delta_of_delta_pages():
    """Each shape is what its name claims, as the oracle's encoder sees it: a delta-of-delta page from 3 rows on (a 2-row
    list is always constant-step), narrow (<= 3-byte second differences) except the wide resets, which bail out."""
    for is_float in (False, True):
        for b in _shape_blocks(is_float, 0xD0D + int(is_float)):
            if b.m.size == 2:
                assert b.enc == 2, b.shape
                continue
            if b.shape == "resets_wide" and b.m.size > 64:
                assert (b.enc, b.kind) == (4, "dod_wide"), (b.shape, b.m.size)
                continue
            assert (b.enc, b.kind) == (4, "dod"), (b.shape, b.m.size)
            lens = varint_lengths(O.int64_list_encode(b.m)[0])[1:]
            if b.shape in ("c1", "negwalk1") or b.m.size < 4:
                continue
            want = {"c2": 2, "c3": 3, "limits": 3, "negwalk3": 3}.get(b.shape)
            if want and b.m.size > 1000:
                assert max(lens) == want, (b.shape, b.m.size)


@gpu
@pytest.mark.parametrize("is_float", [False, True], ids=["int64", "float64"])
@pytest.mark.parametrize("mode", ["all", "range", "dict_mask", "int_mask", "dedup"])
def test_dod_shape_matrix(bydb, gpu_ctx, mode, is_float):
    """Every delta-of-delta shape x block size x aggregate set under one row mode: dod_page_fast<all / range / mask> for the
    narrow pages, its bail-out and decode_varint_page<true> for the wide resets."""
    blocks = _shape_blocks(is_float, 0xD0D + int(is_float))
    if mode != "dedup":
        run_modes(bydb, gpu_ctx, blocks, is_float, [mode], (SUMS, MINMAX, ALL5), "shapes")
        return
    # a second part rewrites the first 5 rows of every series with a higher version (narrow delta / constant-step pages)
    rng = np.random.default_rng(98)
    shadow = [Blk(b.sid, b.ts[:min(5, b.m.size)], shape_values("d1", min(5, b.m.size), rng)[0]) for b in blocks]
    seen = [np.concatenate([s.m, b.m[s.m.size:]]) for s, b in zip(shadow, blocks)]
    run_modes(bydb, gpu_ctx, blocks, is_float, ["all"], (SUMS, MINMAX, ALL5), "shapes/dedup", extra_parts=(make_part(shadow, is_float, version=2),),
              older_keep=lambda b: np.arange(b.m.size) >= 5, model_mants=seen)


# ------------------------------------------------------------------ 3. wrap-around mod 2^64
@gpu
def test_int64_dod_wraps_mod_2_64(bydb, gpu_ctx):
    """First values near +-2^63 and first differences near +-2^62: V0 + n_ex * D0 + r_ex and the 128-bit block sum wrap.  MIN,
    MAX and SUM are checked exactly against Python ints reduced mod 2^64."""
    rng = np.random.default_rng(62)
    cases = [(I64_MAX - 1000, (1 << 62) + 7), (I64_MIN + 1000, (1 << 62) - 3), (-5, (1 << 62) + 11), (I64_MAX - 5, -(1 << 62) - 1),
             (I64_MIN + 3, -(1 << 62) + 5), ((1 << 62), (1 << 61) + 1)]
    blocks, sid = [], 1
    for first, d1 in cases:
        for n in (3, 33, 1025, 8193):
            sd = rng.integers(-40, 41, n - 2)
            sd[sd == 0] = 1                                       # never constant-step
            v = [first, wrap(first + d1)]
            step = d1
            for x in sd.tolist():
                step += x
                v.append(wrap(v[-1] + step))
            m = np.array(v, dtype=np.int64)
            assert m.tolist() == from_dod(first, d1, sd).tolist()
            blocks.append(Blk(sid, regular_ts(n), m))
            assert blocks[-1].kind == "dod", (first, d1, n)
            sid += 1
    run_modes(bydb, gpu_ctx, blocks, False, ["all", "range", "int_mask"], (SUMS, MINMAX, ALL5), "wrap")


# ------------------------------------------------------------------ 4. irregular timestamps: the time range at every position
# decode_varint_page geometry of a timestamp body: 16 B lanes, 512 B chunks, 2 KB stages
TS_EDGES = [16, 32, 496, 512, 528, 2032, 2048, 2064, 4096, 6144, 8192, 16384, 30720]
TS_SIZES = (2049, 4097, 8193)


def irregular_ts(kind, n, rng):
    """ascending timestamps whose page is delta-of-delta: narrow jitter (tens of ns), wide jitter (up to 10 ms: 4-byte second
    differences) or a 9-byte first step followed by narrow jitter"""
    if kind == "narrow":
        steps = STEP + rng.integers(-20, 21, n - 1)
    elif kind == "wide":
        steps = STEP + rng.integers(-10_000_000, 10_000_001, n - 1)
    else:
        steps = STEP + rng.integers(-20, 21, n - 1)
        steps[0] = 1 << 58
    return T0 + np.concatenate([[0], np.cumsum(steps)]).astype(np.int64)


def ts_blocks(seed):
    rng = np.random.default_rng(seed)
    blocks, sid = [], 1
    for kind in ("narrow", "wide", "first"):
        for n in TS_SIZES:
            ts = irregular_ts(kind, n, rng)
            m = from_dod(100 + sid, 50, rng.integers(-20, 21, n - 2))      # a narrow counter field
            b = Blk(sid, ts, m)
            body, enc, _ = O.int64_list_encode(ts)
            assert enc == 4
            b.ts_body = body
            b.ts_kind = kind
            blocks.append(b)
            sid += 1
    return blocks


def edge_rows_of(body, start):
    """rows whose varint holds an edge byte (TS_EDGES) of decode_varint_page's aligned copy of a page body starting at byte
    `start` of its 16 B-aligned copy (varint i is row i + 1)"""
    ends = np.cumsum(varint_lengths(body))          # end byte (exclusive) of each varint
    rows = []
    for e in TS_EDGES:
        i = int(np.searchsorted(ends, e - start, side="right"))
        if i < ends.size:
            rows.append(i + 1)
    return rows


def edge_rows(blocks):
    """(block, row) pairs at the edges of the timestamp bodies: timestamps.bin holds each block's timestamp body then its
    version body (empty: one version), and files sit 256 B aligned on the device, so a body starts at its offset mod 16"""
    off, out = 0, []
    for b in blocks:
        out += [(b, r) for r in edge_rows_of(b.ts_body, off & 15)]
        off += len(b.ts_body)
    return out


@gpu
def test_time_range_cut_at_every_edge(bydb, gpu_ctx):
    """tmin and tmax at, just before and just after the timestamp of a row whose varint sits at a lane, chunk or stage edge
    of its block's timestamp body; then a range between two timestamps of a block (selects it, keeps no row), one-row
    ranges and tmin > tmax.  Each cut block goes to the slow lane (reason bit 0: irregular timestamps), where TsCons counts
    lt / le over decode_varint_page<true>; the kept rows are checked against np.searchsorted."""
    blocks = ts_blocks(0x75)
    parts = [build_part(np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks]), np.concatenate([b.ts for b in blocks]),
                        np.ones(sum(b.m.size for b in blocks), np.int64),
                        [("v", O.VT_INT64, np.concatenate([b.m for b in blocks]), None),
                         ("f", O.VT_FLOAT64, np.concatenate([b.m for b in blocks]) / 100.0, None)])]
    usid = np.array([b.sid for b in blocks], dtype=np.uint64)
    ranges = []
    for b, r in edge_rows(blocks):
        t = int(b.ts[r])
        for dt in (-1, 0, 1):
            ranges += [(t + dt, I64_MAX), (I64_MIN, t + dt)]
        ranges.append((t, t))                                   # one row
        ranges.append((int(b.ts[r - 1]) + 1, t - 1))            # between two timestamps: the block is selected, keeps nothing
        ranges.append((t + 1, t - 1))                           # tmin > tmax
    assert len(ranges) > 300
    aggs = [("v", O.AGG_SUM), ("v", O.AGG_COUNT), ("v", O.AGG_MIN), ("v", O.AGG_MAX), ("f", O.AGG_SUM), ("f", O.AGG_MAX)]
    with Registered(bydb, gpu_ctx, parts) as reg:
        for tmin, tmax in ranges:
            got, want = reg.run(usid, aggs, tmin, tmax)
            ctx = f"ts [{tmin - T0}, {tmax - T0}]"
            assert_parity(got, want, aggs, ctx)
            kept = [int(np.searchsorted(b.ts, tmax, side="right")) - int(np.searchsorted(b.ts, tmin, side="left")) for b in blocks]
            kept = [max(k, 0) for k in kept]
            assert got.stats.rows_matched == sum(kept), ctx
            keeps = [(b.ts >= tmin) & (b.ts <= tmax) for b in blocks]
            assert [int(k.sum()) for k in keeps] == kept
            check_model(got, [b.m for b in blocks], keeps, aggs[:4], False, ctx)
            cut = sum(1 for b in blocks if tmin <= tmax and not (b.ts[-1] < tmin or b.ts[0] > tmax)
                      and (tmin > b.ts[0] or tmax < b.ts[-1]))
            assert got.stats.blocks_slow_lane == cut, f"{ctx}: slow-lane blocks {got.stats.blocks_slow_lane}, expected {cut}"
            assert got.stats.slow_lane_reasons == (1 if cut else 0), ctx


# ------------------------------------------------------------------ 5. dedup and int64 tag predicates over long DoD pages
@gpu
def test_dedup_over_long_dod_timestamps(bydb, gpu_ctx):
    """Two overlapping parts with 8193-row irregular-timestamp blocks: the newer part rewrites the rows around every edge of
    the older part's timestamp bodies, so the shadowed rows straddle them, and decode_list_to decodes both parts' timestamp
    pages in the dedup."""
    blocks = [b for b in ts_blocks(0xDD) if b.m.size == 8193]
    older = build_part(np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks]), np.concatenate([b.ts for b in blocks]),
                       np.ones(sum(b.m.size for b in blocks), np.int64), [("v", O.VT_INT64, np.concatenate([b.m for b in blocks]), None)])
    shadow = {b.sid: set() for b in blocks}
    for b, r in edge_rows(blocks):
        shadow[b.sid].update(range(max(r - 2, 0), min(r + 3, b.m.size)))
    rows = {s: np.array(sorted(v), dtype=np.int64) for s, v in shadow.items()}
    newer_vals = {b.sid: -7 * rows[b.sid] - 11 for b in blocks}
    newer = build_part(np.concatenate([np.full(rows[b.sid].size, b.sid, np.uint64) for b in blocks]),
                       np.concatenate([b.ts[rows[b.sid]] for b in blocks]), np.full(sum(r.size for r in rows.values()), 2, np.int64),
                       [("v", O.VT_INT64, np.concatenate([newer_vals[b.sid] for b in blocks]), None)])
    for b in blocks:
        assert page_kind(b.ts[rows[b.sid]])[0] == 4, "the newer part's timestamps are a delta-of-delta page too"
    usid = np.array([b.sid for b in blocks], dtype=np.uint64)
    merged = []
    for b in blocks:
        m = b.m.copy()
        m[rows[b.sid]] = newer_vals[b.sid]
        merged.append(m)
    with Registered(bydb, gpu_ctx, [older, newer]) as reg:
        for tmin, tmax in ((I64_MIN, I64_MAX), (int(blocks[0].ts[600]), int(blocks[1].ts[5000]))):
            for aggset in (SUMS, ALL5):
                aggs = [("v", f) for f in aggset]
                got, want = reg.run(usid, aggs, tmin, tmax)
                ctx = f"dedup/[{tmin}, {tmax}]/{aggset}"
                assert_parity(got, want, aggs, ctx)
                keeps = [(b.ts >= tmin) & (b.ts <= tmax) for b in blocks]
                check_model(got, merged, keeps, aggs, False, ctx)


@gpu
def test_int64_dod_tag_predicates_at_every_edge(bydb, gpu_ctx):
    """An int64 tag whose pages are delta-of-delta (a jittered counter) on 8193-row blocks: the fast lane defers every block
    (reason bit 1) and the slow lane's CmpCons clears mask bits over decode_varint_page<true>.  The literals are the tag values
    of the rows whose varints sit at the edges of the tag body, and one off."""
    rng = np.random.default_rng(0x7A6)
    blocks = []
    for sid, spread in enumerate((8, 1 << 18, 1 << 26), start=1):     # 1-byte, 3-byte and 4-byte second differences
        seq = from_dod(1 << 20, 1 << 27, np.diff(rng.integers(0, spread, 8192)))
        b = Blk(sid, regular_ts(8193), from_dod(40 + sid, 9, rng.integers(-30, 31, 8191)))
        b.seq = seq
        body, enc, _ = O.int64_list_encode(seq)
        assert enc == 4
        b.seq_body = body
        blocks.append(b)
    sids = np.concatenate([np.full(b.m.size, b.sid, np.uint64) for b in blocks])
    part = build_part(sids, np.concatenate([b.ts for b in blocks]), np.ones(sids.size, np.int64),
                      [("v", O.VT_INT64, np.concatenate([b.m for b in blocks]), None)],
                      [("default", [("seq", O.VT_INT64, np.concatenate([b.seq for b in blocks]), None)])])
    usid = np.array([b.sid for b in blocks], dtype=np.uint64)
    # the tag pages in default.tf: [enc][first, 8 bytes][body], one after the other, so a body starts 9 bytes into its page
    lits, off = set(), 0
    for b in blocks:
        for r in edge_rows_of(b.seq_body, (off + 9) & 15):
            lits.update(int(b.seq[r]) + d for d in (-1, 0, 1))
        off += 9 + len(b.seq_body)
    ops = {O.OP_LT: np.less, O.OP_LE: np.less_equal, O.OP_GT: np.greater, O.OP_GE: np.greater_equal, O.OP_EQ: np.equal, O.OP_NE: np.not_equal}
    aggs = [("v", O.AGG_SUM), ("v", O.AGG_COUNT), ("v", O.AGG_MAX)]
    with Registered(bydb, gpu_ctx, [part]) as reg:
        for lit in sorted(lits):
            for op, fn in ops.items():
                got, want = reg.run(usid, aggs, preds=[O.Pred("default", "seq", op, lit)])
                ctx = f"seq op {op} {lit}"
                assert_parity(got, want, aggs, ctx)
                check_model(got, [b.m for b in blocks], [fn(b.seq, lit) for b in blocks], aggs, False, ctx)
                assert got.stats.blocks_slow_lane == len(blocks) and got.stats.slow_lane_reasons == 2, ctx

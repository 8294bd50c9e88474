"""The partial-table reduce against the oracle at its boundaries: per-rank tables, the rank-order combine, the finalisation,
the wire-shape rows and the peer mailboxes.

After the scan, every multi-table route runs the same step: per-table partials are merged word by word in rank order
(`combine_tables_kernel`) and the merged table is finalised.  The routes are bydb_scan_partials -> bydb_partials_combine ->
bydb_reduce_finalize / bydb_partials_rows, the root of bydb_scan_reduce (the ranks' tables in its mailbox slots), and the cold
path of bydb_scan_agg_host (one table per block-index slice).  The combine depends on how the table encodes its values
(bydb_gpu.h): MIN as -min (float) and ~min (int64), "met the column" in the other type's maximum word, type and status in the
coltype words, float sums added in rank order.  So the tests here

  - restate the combine in numpy over the raw tables and require the device's combined table to be bit-identical to it;
  - finalise the combined table and compare with the oracle over all shards (int64 and MIN / MAX exactly, float sums and means
    to 1e-12 relative; a zero MIN / MAX without its sign, DESIGN 6), and with one context scanning every shard where the
    reference's order is ill-defined (NaN);
  - put the edges of that encoding on different ranks: INT64_MIN / INT64_MAX, wrapping sums, groups on one rank, groups that
    met only null cells or never met the column, +-0.0, +-Inf and NaN, means below 1;
  - fail a field that is int64 in one table and float64 in another (BYDB_EINVAL), like one scan over the same parts does.
"""
from __future__ import annotations

import math
import re

import numpy as np
import pytest

from oracle import oracle as O
from tests import schema_mix as M
from tests.helpers import STEP, T0, build_part, grid

gpu = pytest.mark.gpu
SUM, COUNT, MIN, MAX, MEAN = O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN
I, F = O.VT_INT64, O.VT_FLOAT64
EINVAL = -22
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
INF, NAN = math.inf, math.nan
ROW_PATH = 2   # BYDB_Q_ROW_PATH_TYPES
K_ERR_TYPE_MIX = 5

_pid = [1_300_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


# ------------------------------------------------------------------ the combine, restated
def merge_coltype(words):
    """scan_kernels.cu merge_coltype over a rank-ordered list of coltype words: the first non-zero type, kErrTypeMix when two
    non-zero types differ, the worst status (bits 8..)"""
    typ = err = 0
    for w in words:
        w = int(np.int64(np.uint64(w)))
        wt, we = w & 0xFF, w >> 8
        if wt and typ and wt != typ:
            err = max(err, K_ERR_TYPE_MIX)
        if typ == 0:
            typ = wt
        err = max(err, we)
    return np.uint64((typ | (err << 8)) & (2**64 - 1))


def regions(G, Fn):
    """word ranges of bydb_gpu.h's table: float sums | float maxima (max, -min) | int64 sums (sum, cnt, rows) | int64 maxima
    (max, ~min) | coltype"""
    GF = G * Fn
    return dict(fsum=slice(0, GF), fmax=slice(GF, 3 * GF), isum=slice(3 * GF, 5 * GF + G), imax=slice(5 * GF + G, 7 * GF + G),
                coltype=slice(7 * GF + G, 7 * GF + G + Fn))


def fold(tables, G, Fn):
    """tables: uint64 [R, words] in rank order -> the combined table, folded in rank order like combine_tables_kernel"""
    rg = regions(G, Fn)
    a = tables[0].copy()
    with np.errstate(all="ignore"):
        for b in tables[1:]:
            s = rg["fsum"]
            a[s] = (a[s].view(np.float64) + b[s].view(np.float64)).view(np.uint64)
            s = rg["fmax"]
            x, y = a[s].view(np.float64), b[s].view(np.float64)
            a[s] = np.where(y > x, b[s], a[s])
            s = rg["isum"]
            a[s] = a[s] + b[s]                                  # uint64: wraps like Go's int64
            s = rg["imax"]
            a[s] = np.where(b[s].view(np.int64) > a[s].view(np.int64), b[s], a[s])
            s = rg["coltype"]
            a[s] = [merge_coltype([x, y]) for x, y in zip(a[s], b[s])]
    return a


def assert_same_table(got, want, G, Fn, ctx):
    """bit-identical, except that two NaNs in a float word may carry different payloads (the device's arithmetic NaN is
    canonical, numpy's keeps an operand's)"""
    differ = got != want
    f = slice(0, 3 * G * Fn)
    both_nan = np.isnan(got[f].view(np.float64)) & np.isnan(want[f].view(np.float64))
    differ[f] &= ~both_nan
    assert not differ.any(), f"{ctx}: words {np.nonzero(differ)[0][:16].tolist()} differ: {got[differ][:8]} vs {want[differ][:8]}"


# ------------------------------------------------------------------ comparisons
def _float_eq(g, w, fn, rel=1e-12):
    if math.isnan(w):
        return math.isnan(g)
    if w == 0.0:
        return g == 0.0                    # the sign of a zero is not compared (DESIGN 6)
    if math.isinf(w) or fn in (MIN, MAX):
        return g == w
    return abs(g - w) <= rel * abs(w)


def check_oracle(got, want, aggs, ftype, ctx, row_path=False):
    """got: a device Result; want: the oracle's.  ftype: field -> value type of the field (absent: no block has it)."""
    assert got.group_id.tolist() == want.group_id.tolist(), f"{ctx}: group ids {got.group_id.tolist()} vs {want.group_id.tolist()}"
    assert got.rows.tolist() == want.rows.tolist(), f"{ctx}: rows"
    for a, (f, fn) in enumerate(aggs):
        isf = ftype.get(f) == F
        out_float = isf and (fn != COUNT or row_path)
        assert bool(got.is_float[a]) == out_float, f"{ctx}: output type of agg {a} ({f}, {fn})"
        if fn == COUNT:
            g = got.val_f64[:, a] if out_float else got.val_i64[:, a]
            assert g.tolist() == want.val_i64[:, a].astype(g.dtype).tolist(), f"{ctx}: COUNT({f})"
        elif not isf:
            assert got.val_i64[:, a].tolist() == want.val_i64[:, a].tolist(), f"{ctx}: int64 agg {a} ({f}, {fn})"
        else:
            for k, (g, w) in enumerate(zip(got.val_f64[:, a].tolist(), want.val_f64[:, a].tolist())):
                assert _float_eq(g, w, fn), f"{ctx}: group {int(got.group_id[k])} agg {a} ({f}, {fn}): {g!r} vs {w!r}"


def check_same_answer(got, want, ctx):
    """two device answers over the same rows: equal, NaN for NaN and a zero for a zero of either sign"""
    assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), ctx
    assert got.is_float.tolist() == want.is_float.tolist() and got.val_i64.tolist() == want.val_i64.tolist(), ctx
    for g, w in zip(got.val_f64.ravel().tolist(), want.val_f64.ravel().tolist()):
        assert (math.isnan(g) and math.isnan(w)) or g == w, f"{ctx}: {got.val_f64} vs {want.val_f64}"


# ------------------------------------------------------------------ shards
ABSENT = "absent"   # the series' blocks lack fields i and f (another measure of the same part)


def rank_part(series):
    """series: [(sid, i cells, f cells)], cells with None for a null; i cells ABSENT for a series whose blocks lack i and f.
    -> one part; a mixed part when some series lack the fields"""
    def rows(ss):
        n = [len(c[1]) if c[1] is not ABSENT else 2 for c in ss]
        sid = np.concatenate([np.full(k, s[0], np.uint64) for s, k in zip(ss, n)])
        ts = np.concatenate([T0 + np.arange(k, dtype=np.int64) * STEP for k in n])
        return sid, ts, np.ones(sid.size, np.int64)

    def col(cells, dt):
        return np.array([0 if c is None else c for c in cells], dt), np.array([c is None for c in cells], np.uint8)
    have = sorted((s for s in series if s[1] is not ABSENT), key=lambda s: s[0])
    lack = sorted((s for s in series if s[1] is ABSENT), key=lambda s: s[0])
    measures = []
    if have:
        sid, ts, ver = rows(have)
        iv, inl = col([c for s in have for c in s[1]], np.int64)
        fv, fnl = col([c for s in have for c in s[2]], np.float64)
        measures.append((sid, ts, ver, [("i", I, iv, inl), ("f", F, fv, fnl)], []))
    if lack:
        sid, ts, ver = rows(lack)
        measures.append((sid, ts, ver, [("other", I, np.arange(sid.size, dtype=np.int64), None)], []))
    return build_part(*measures[0]) if len(measures) == 1 else O.build_mixed_part(measures)


class Shards:
    """R series-disjoint shards (rank order), each an oracle part registered on `ctx`, with the global series -> group map"""

    def __init__(self, bydb, ctx, parts, sids, groups, G):
        import torch
        self.bydb, self.ctx, self.parts, self.G = bydb, ctx, parts, G
        self.sids = [np.asarray(s, np.uint64) for s in sids]
        self.groups = [np.asarray(g, np.int32) for g in groups]
        order = np.argsort(np.concatenate(self.sids), kind="stable")
        self.all_sids = np.concatenate(self.sids)[order]
        self.all_groups = np.concatenate(self.groups)[order]
        self.handles = [ctx.register_part(_next_pid(), p.files()) for p in parts]
        self.stream = torch.cuda.current_stream().cuda_stream

    def close(self):
        for h in self.handles:
            self.ctx.release_part(h)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def q(self, r, aggs, **kw):
        o = np.argsort(self.sids[r], kind="stable")
        return self.bydb.Query([self.handles[r]], self.sids[r][o], aggs, series_group=self.groups[r][o], n_groups=self.G, **kw)

    def q_final(self, aggs, **kw):
        return self.bydb.Query([], self.all_sids, aggs, series_group=self.all_groups, n_groups=self.G, **kw)

    def q_whole(self, aggs, **kw):
        return self.bydb.Query(self.handles, self.all_sids, aggs, series_group=self.all_groups, n_groups=self.G, **kw)

    def oracle(self, aggs, **kw):
        kw.pop("flags", None)
        return O.run_query(O.Query(self.parts, self.all_sids, aggs, groups=self.all_groups, n_groups=self.G, **kw))

    def tables(self, aggs, order=None, **kw):
        """every rank's table, back to back in `order` (default: rank order) -> (device tensor, host uint64 [R, words], layout)"""
        import torch
        order = list(range(len(self.parts))) if order is None else list(order)
        lay = self.ctx.partials_layout(self.q_final(aggs, **kw))
        nb = lay["total_bytes"]
        t = torch.zeros(len(order) * nb // 8, dtype=torch.int64, device="cuda")
        for slot, r in enumerate(order):
            self.ctx.scan_partials(self.q(r, aggs, **kw), t.data_ptr() + slot * nb, nb, self.stream)
        host = t.cpu().numpy().view(np.uint64).reshape(len(order), nb // 8).copy()
        return t, host, lay

    def combine(self, t, n, lay, aggs, **kw):
        self.ctx.partials_combine(self.q_final(aggs, **kw), t.data_ptr(), n, lay["total_bytes"], self.stream)
        return t[: lay["total_bytes"] // 8].cpu().numpy().view(np.uint64).copy()

    def finalize(self, t, lay, aggs, **kw):
        return self.ctx.reduce_finalize(self.q_final(aggs, **kw), t.data_ptr(), lay["total_bytes"], self.stream)


def n_fields(aggs):
    return len(dict.fromkeys(f for f, _ in aggs))


# ------------------------------------------------------------------ a. the combine, word for word
AGGS_ALL = [("lat", SUM), ("lat", MIN), ("lat", MAX), ("lat", MEAN), ("calls", SUM), ("calls", MIN), ("calls", MAX),
            ("calls", MEAN), ("calls", COUNT), ("lat", COUNT)]


def random_shards(bydb, ctx, R, G=7, n_series=48, n_pts=300, seed=5):
    rng = np.random.default_rng(seed + R)
    sids, ts, ver = grid(n_series, n_pts)
    lat = np.round(rng.normal(30, 12, sids.size), 2)
    calls = rng.integers(-(1 << 40), 1 << 40, sids.size)
    usid = np.unique(sids)
    rank_of = np.arange(usid.size) % R
    parts, ss, gs = [], [], []
    for r in range(R):
        mine = usid[rank_of == r]
        m = np.isin(sids, mine)
        parts.append(build_part(sids[m], ts[m], ver[m], [("lat", F, lat[m], None), ("calls", I, calls[m], None)]))
        ss.append(mine)
        gs.append((np.nonzero(rank_of == r)[0] * 5 % G).astype(np.int32))
    return Shards(bydb, ctx, parts, ss, gs, G)


@gpu
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_combine_is_the_rank_order_fold_of_the_raw_tables(bydb, gpu_ctx, R):
    with random_shards(bydb, gpu_ctx, R) as sh:
        t, host, lay = sh.tables(AGGS_ALL)
        Fn, G = n_fields(AGGS_ALL), sh.G
        assert host.shape[1] * 8 == 8 * (7 * G * Fn + G + Fn)
        got = sh.combine(t, R, lay, AGGS_ALL)
        assert_same_table(got, fold(host, G, Fn), G, Fn, f"R={R}")
        if R == 1:
            assert (got == host[0]).all(), "one table: the combine leaves it untouched"
        # the tables behind the first are inputs: the combine writes only the first
        assert (t.cpu().numpy().view(np.uint64).reshape(R, -1)[1:] == host[1:]).all()
        check_oracle(sh.finalize(t, lay, AGGS_ALL), sh.oracle(AGGS_ALL), AGGS_ALL, {"lat": F, "calls": I}, f"R={R}")


# ------------------------------------------------------------------ b. boundaries in the data
G_B = 16
# group -> [(rank, i cells, f cells)]; None is a null cell, ABSENT a series whose blocks lack the fields
BOUNDARY = {
    0: [(0, [I64_MIN, 5], [1.5, 2.5]), (1, [I64_MAX, -3], [-0.5, 4.0])],          # MIN = INT64_MIN (~x), MAX = INT64_MAX elsewhere
    1: [(2, [I64_MAX, I64_MAX], [7.25, 7.25])],                                    # only minimum INT64_MAX: the empty notmin word
    2: [(0, [1 << 62, (1 << 62) - 1], [0.5, 0.25]), (1, [1 << 62, 3], [0.125, 0.125])],  # sum wraps across ranks; MEAN < 1
    3: [(1, [11, -4, 9], [3.0, 1.0, 2.0])],                                        # on one rank only
    4: [(0, [None, None], [None, None]), (1, [6, -2], [2.5, -1.5])],              # met only nulls + values
    5: [(0, [None, None, None], [None, None, None])],                              # met only nulls: the sentinels
    6: [(2, ABSENT, None), (0, [-9, -7], [-3.5, -2.0])],                           # never met + values (all negative)
    7: [(2, ABSENT, None)],                                                        # never met: the zero values
    8: [(0, [None], [None]), (2, ABSENT, None)],                                   # met only nulls + never met: the sentinels
    9: [(1, [None, 4], [None, 8.5]), (2, ABSENT, None)],                           # values beside a null + never met
    10: [(0, [1, 2], [-0.0, None]), (1, [3, 4], [0.0, None])],                     # -0 then +0 (Plain pages: a null cell)
    11: [(0, [1, 2], [0.0, None]), (1, [3, 4], [-0.0, None])],                     # +0 then -0
    12: [(0, [5, 6], [INF, None]), (2, [7, 8], [-INF, 1.0, ])],                   # +-Inf: SUM NaN, MIN -Inf, MAX +Inf
    13: [(0, [1, -1], [NAN, 2.0]), (1, [2, -2], [3.0, None])],                     # NaN first
    14: [(1, [-5, -6], [3.0, None]), (2, [7, 1], [NAN, 0.5])],                     # NaN last
    15: [(0, [-7, 2], [0.25, 0.5]), (2, [1, 0], [0.125, 0.75])],                  # MEAN below 1, int64 MEAN of a negative sum
}
B_AGGS = [("i", SUM), ("i", MIN), ("i", MAX), ("i", MEAN), ("i", COUNT), ("f", SUM), ("f", MIN), ("f", MAX), ("f", MEAN), ("f", COUNT)]
B_TYPES = {"i": I, "f": F}
# groups where a rank never met the column but another did: a node's zero value there is not the identity of MIN / MAX
NEVER_MET_BESIDE_MET = {g for g, ss in BOUNDARY.items() if any(c is ABSENT for _, c, _ in ss) and any(c is not ABSENT for _, c, _ in ss)}


def boundary_shards(bydb, ctx, cases=BOUNDARY, R=3):
    per_rank = [[] for _ in range(R)]
    gs = [[] for _ in range(R)]
    for g, series in cases.items():
        for k, (r, ic, fc) in enumerate(series):
            sid = 1 + r * 1000 + g * 10 + k        # series order = rank order: the oracle meets the ranks in rank order
            per_rank[r].append((sid, ic, fc))
            gs[r].append(g)
    parts = [rank_part(s) for s in per_rank]
    return Shards(bydb, ctx, parts, [[s[0] for s in ss] for ss in per_rank], gs, max(cases) + 1)


@gpu
@pytest.mark.parametrize("order", ["rank", "reversed"])
@pytest.mark.parametrize("row_path", [False, True])
def test_boundary_values_across_ranks(bydb, gpu_ctx, order, row_path):
    kw = dict(flags=ROW_PATH) if row_path else {}
    with boundary_shards(bydb, gpu_ctx) as sh:
        R = len(sh.parts)
        perm = list(range(R)) if order == "rank" else list(reversed(range(R)))
        t, host, lay = sh.tables(B_AGGS, perm, **kw)
        got_t = sh.combine(t, R, lay, B_AGGS, **kw)
        assert_same_table(got_t, fold(host, sh.G, 2), sh.G, 2, order)
        # the encodings at their edges, read from the combined table
        tb = got_t.view(np.int64)
        GF = sh.G * 2
        cnt, mx_i, notmin_i = tb[4 * GF:5 * GF].reshape(-1, 2), tb[5 * GF + sh.G:6 * GF + sh.G].reshape(-1, 2), tb[6 * GF + sh.G:7 * GF + sh.G].reshape(-1, 2)
        assert notmin_i[0, 0] == ~I64_MIN and mx_i[0, 0] == I64_MAX
        assert notmin_i[1, 0] == notmin_i[7, 0] == I64_MIN and cnt[1, 0] == 2 and cnt[7, 0] == 0, "INT64_MAX minimum vs empty: only cnt differs"
        assert (tb[7 * GF + sh.G:] == [I, F]).all(), "coltype: the types, no status"
        got = sh.finalize(t, lay, B_AGGS, **kw)
        check_oracle(got, sh.oracle(B_AGGS), B_AGGS, B_TYPES, f"{order}/row_path={row_path}", row_path)
        # met_column: never met -> zero values, only nulls -> the sentinels, anything else -> the values
        at = {g: k for k, g in enumerate(got.group_id.tolist())}
        imin, imax, fmin, fmax = (B_AGGS.index(a) for a in [("i", MIN), ("i", MAX), ("f", MIN), ("f", MAX)])
        for g, (vi_min, vi_max, vf_min, vf_max) in {7: (0, 0, 0.0, 0.0), 5: (I64_MAX, I64_MIN, 1.7976931348623157e308, -1.7976931348623157e308),
                                                      8: (I64_MAX, I64_MIN, 1.7976931348623157e308, -1.7976931348623157e308),
                                                      6: (-9, -7, -3.5, -2.0), 4: (-2, 6, -1.5, 2.5), 9: (4, 4, 8.5, 8.5)}.items():
            k = at[g]
            assert (got.val_i64[k, imin], got.val_i64[k, imax], got.val_f64[k, fmin], got.val_f64[k, fmax]) == (vi_min, vi_max, vf_min, vf_max), g
        # NaN: the reference's order of a NaN is ill-defined; the combined answer equals one context over the same parts
        check_same_answer(got, gpu_ctx.scan_agg(sh.q_whole(B_AGGS, **kw)), f"{order}: single context")


# ------------------------------------------------------------------ c. shapes
@gpu
def test_groups_of_32_and_33_series_give_bit_identical_tables(bydb, gpu_ctx):
    """group_reduce_small_kernel (every group <= 32 series) and the CTA reduce (a group of 33) sum in the same tree: a series
    that selects no block, appended to a 32-series group, switches the kernel and must leave the rank's table unchanged"""
    import torch
    rng = np.random.default_rng(33)
    spec = [(0, 32, 0), (0, 3, 1), (1, 5, 0), (1, 4, 2)]       # (rank, series, group)
    per_rank, gs, sid = [[], []], [[], []], 1
    for r, n, g in spec:
        for _ in range(n):
            per_rank[r].append((sid, rng.integers(-1000, 1000, 40).tolist(), np.round(rng.normal(7, 30, 40), 3).tolist()))
            gs[r].append(g)
            sid += 1
    parts = [rank_part(s) for s in per_rank]
    aggs = [("f", SUM), ("f", MEAN), ("f", MIN), ("i", SUM), ("i", MAX), ("i", COUNT)]
    with Shards(bydb, gpu_ctx, parts, [[s[0] for s in ss] for ss in per_rank], gs, 3) as sh:
        t, host, lay = sh.tables(aggs)
        nb = lay["total_bytes"]
        # rank 0 again, group 0 grown to 33 series by a series id no block holds (the largest id: the tree keeps its order)
        q33 = sh.q(0, aggs)
        q33.series_ids = np.append(q33.series_ids, np.uint64(10_000))
        q33.series_group = np.append(q33.series_group, np.int32(0))
        t33 = torch.zeros(nb // 8, dtype=torch.int64, device="cuda")
        gpu_ctx.scan_partials(q33, t33.data_ptr(), nb, sh.stream)
        assert (t33.cpu().numpy().view(np.uint64) == host[0]).all(), "32-series warp reduce vs 33-series CTA reduce"
        got_t = sh.combine(t, 2, lay, aggs)
        assert_same_table(got_t, fold(host, 3, 2), 3, 2, "32/33")
        check_oracle(sh.finalize(t, lay, aggs), sh.oracle(aggs), aggs, {"i": I, "f": F}, "32/33")


def topn_shards(bydb, ctx, G, R, seed):
    """groups of one or two series on neighbouring ranks, small values (ties across ranks), every 7th group never meets the
    column (a null Top-N key for MIN / MAX), every 11th meets only null cells"""
    rng = np.random.default_rng(seed)
    per_rank, gs = [[] for _ in range(R)], [[] for _ in range(R)]
    for g in range(G):
        for k in range(1 + g % 2):
            r = (g + k) % R
            sid = 1 + g * 4 + k
            if g % 7 == 3:
                per_rank[r].append((sid, ABSENT, None))
            elif g % 11 == 5:
                per_rank[r].append((sid, [None, None], [None, None]))
            else:
                per_rank[r].append((sid, rng.integers(-3, 4, 2).tolist(), rng.choice([0.5, 1.5, 2.5], 2).tolist()))
            gs[r].append(g)
    return Shards(bydb, ctx, [rank_part(s) for s in per_rank], [[s[0] for s in ss] for ss in per_rank], gs, G)


T_AGGS = [("i", SUM), ("i", MAX), ("f", MIN), ("i", COUNT), ("f", MEAN)]


@gpu
@pytest.mark.parametrize("G", [12, 2048, 2049])
def test_top_n_after_the_combine(bydb, gpu_ctx, G):
    """G <= 2048: every group goes through the bitonic sort; 2049: the radix select first.  Ties across ranks (the lower group
    id wins), null keys (groups that never met the column) in both directions, N above the competing groups"""
    with topn_shards(bydb, gpu_ctx, G, 3, seed=G) as sh:
        t, host, lay = sh.tables(T_AGGS)
        sh.combine(t, 3, lay, T_AGGS)
        big = min(G + 5, 2048)                               # the device's largest N
        for top_agg, desc, n in [(0, True, 5), (0, False, 9), (1, True, 7), (1, False, 11), (2, False, 4), (2, True, 6),
                                 (1, True, big), (1, False, big), (3, False, big)]:
            kw = dict(top_n=n, top_agg=top_agg, top_desc=desc)
            got = sh.finalize(t, lay, T_AGGS, **kw)        # finalisation reads the combined table; it does not change it
            want = sh.oracle(T_AGGS, **kw)
            check_oracle(got, want, T_AGGS, {"i": I, "f": F}, f"G={G} top {kw}")
            if G == 12:                                     # one context over every shard selects the same rows
                check_oracle(gpu_ctx.scan_agg(sh.q_whole(T_AGGS, **kw)), want, T_AGGS, {"i": I, "f": F}, f"single context top {kw}")


# ------------------------------------------------------------------ d. wire-shape rows
def _wrap(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


@gpu
def test_partial_rows_on_boundary_tables(bydb, gpu_ctx):
    """bydb_partials_rows per rank and on the combined table: Partial.Value (+ Partial.Count for MEAN) per function, typed like
    the field, the sentinels for groups that met only nulls; the liaison's fold over the ranks' rows gives the oracle's answer"""
    fns = (SUM, COUNT, MAX, MIN)
    with boundary_shards(bydb, gpu_ctx) as sh:
        t, host, lay = sh.tables(B_AGGS)
        nb = lay["total_bytes"]
        R = len(sh.parts)

        def expect(rows, parts, sids, groups, ctx):
            own = {fn: O.run_query(O.Query(parts, sids, [(f, fn) for f, _ in B_AGGS], groups=groups, n_groups=sh.G)) for fn in fns}
            assert rows["group_id"].tolist() == own[SUM].group_id.tolist(), ctx
            assert rows["is_float"].tolist() == [B_TYPES[f] == F for f, _ in B_AGGS], ctx
            for a, (f, fn) in enumerate(B_AGGS):
                isf = B_TYPES[f] == F
                gv = (rows["val_f64"] if isf else rows["val_i64"])[:, a].tolist()
                gc = (rows["cnt_f64"] if isf else rows["cnt_i64"])[:, a].tolist()
                src = own[SUM if fn == MEAN else fn]
                wv = (src.val_f64 if isf and fn != COUNT else src.val_i64)[:, a].tolist()
                wc = own[COUNT].val_i64[:, a].tolist() if fn == MEAN else [0] * len(gc)
                for k, (x, y) in enumerate(zip(gv, wv)):
                    assert (_float_eq(x, y, fn) if isf else x == y), f"{ctx}: group {rows['group_id'][k]} agg {a} ({f}, {fn}): {x!r} vs {y!r}"
                assert gc == wc, f"{ctx}: Partial.Count of agg {a}"

        node_rows = []
        for slot in range(R):
            rows = gpu_ctx.partials_rows(sh.q(slot, B_AGGS), t.data_ptr() + slot * nb, nb, sh.stream)
            o = np.argsort(sh.sids[slot], kind="stable")
            expect(rows, [sh.parts[slot]], sh.sids[slot][o], sh.groups[slot][o], f"rank {slot}")
            node_rows.append(rows)
        sh.combine(t, R, lay, B_AGGS)
        expect(gpu_ctx.partials_rows(sh.q_final(B_AGGS), t.data_ptr(), nb, sh.stream), sh.parts, sh.all_sids, sh.all_groups, "combined")
        # the liaison: reduceAccumulator.Combine over the nodes' rows, then Val() (function.go), int64 sums wrapping
        want = sh.oracle(B_AGGS)
        for gi, g in enumerate(want.group_id.tolist()):
            for a, (f, fn) in enumerate(B_AGGS):
                isf = B_TYPES[f] == F
                if fn in (MIN, MAX) and g in NEVER_MET_BESIDE_MET:
                    continue
                vals = []
                for rows in node_rows:
                    k = np.nonzero(rows["group_id"] == g)[0]
                    if k.size:
                        vals.append(((rows["val_f64"] if isf else rows["val_i64"])[k[0], a].item(), (rows["cnt_f64"] if isf else rows["cnt_i64"])[k[0], a].item()))
                assert vals, g
                if fn == MEAN:
                    s_, c_ = (sum(v for v, _ in vals), sum(c for _, c in vals)) if isf else (_wrap(sum(v for v, _ in vals)), sum(c for _, c in vals))
                    if c_ == 0:
                        val = 0.0 if isf else 0
                    elif isf:
                        val = s_ / c_
                    else:
                        val = abs(s_) // c_ * (1 if s_ >= 0 else -1)      # Go's integer division truncates toward zero
                    val = 1 if (c_ != 0 and val < 1) else val
                elif fn in (SUM, COUNT):
                    val = sum(v for v, _ in vals) if isf else _wrap(sum(v for v, _ in vals))
                elif fn == MAX:
                    val = max(v for v, _ in vals)
                else:
                    val = min(v for v, _ in vals)
                ref = want.val_f64[gi, a] if want.is_float[a] else want.val_i64[gi, a]
                ok = _float_eq(float(val), float(ref), fn, 1e-9) if isf else val == ref
                assert ok, (g, a, f, fn, val, ref)


# ------------------------------------------------------------------ e. peer mailboxes
@gpu
def test_scan_reduce_equals_combine_and_finalize(bydb, gpu_ctx):
    """bydb_scan_reduce over the boundary shards, three contexts on one device: the root's answer is bit-identical to
    bydb_partials_combine + bydb_reduce_finalize over the same tables (both combine in rank order; the mailbox slots have
    their own stride).  A field int64 on one rank and float64 on another fails the root with BYDB_EINVAL, and the
    mailboxes stay usable afterwards."""
    import faulthandler
    import gc
    import threading
    # as in test_gpu_parity's collective: a finaliser of an earlier test's object may free page-locked memory on a rank's thread
    # in the middle of the collective (an implicit device synchronisation that waits for the peers' spinning kernels)
    gc.collect()
    gc.disable()
    faulthandler.dump_traceback_later(25, exit=False)
    try:
        _scan_reduce_body(bydb, gpu_ctx)
    finally:
        faulthandler.cancel_dump_traceback_later()
        gc.enable()


def _collective(ctxs, call):
    R = len(ctxs)
    got, errs = [None] * R, [None] * R

    def run(r):
        try:
            got[r] = call(r)
        except Exception as e:  # noqa: BLE001
            errs[r] = e
    import threading
    th = [threading.Thread(target=run, args=(r,)) for r in range(R)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return got, errs


def _scan_reduce_body(bydb, gpu_ctx):
    import torch
    n_dev = torch.cuda.device_count()
    R = 3
    ms = M.type_mix_cases() + [M.Measure("vi2", np.arange(100, 104), 50, [("v", I)], [("default", [("region", O.VT_STR)])], seed=34)]
    mix_parts = [ms[0].own_part(), ms[1].own_part(), ms[2].own_part()]   # rank 0, 2: v int64; rank 1: v float64
    with boundary_shards(bydb, gpu_ctx) as sh:
        ctxs = [bydb.Context(device=r % n_dev) for r in range(R)]
        try:
            handles = [c.comm_export(1 << 20, R) for c in ctxs]
            for r, c in enumerate(ctxs):
                c.comm_connect(r, R, handles)
            hs = [c.register_part(1, p.files()) for c, p in zip(ctxs, sh.parts)]
            t, host, lay = sh.tables(B_AGGS)
            sh.combine(t, R, lay, B_AGGS)
            want = sh.finalize(t, lay, B_AGGS)
            def boundary(root):
                def call(r):
                    o = np.argsort(sh.sids[r], kind="stable")
                    return ctxs[r].scan_reduce(bydb.Query([hs[r]], sh.sids[r][o], B_AGGS, series_group=sh.groups[r][o], n_groups=sh.G), root=root)
                got, errs = _collective(ctxs, call)
                assert errs == [None] * R, errs
                g = got[root]
                assert g.group_id.tolist() == want.group_id.tolist() and g.rows.tolist() == want.rows.tolist(), root
                assert g.is_float.tolist() == want.is_float.tolist() and g.val_i64.tolist() == want.val_i64.tolist(), root
                assert g.val_f64.view(np.uint64).tolist() == want.val_f64.view(np.uint64).tolist(), f"root {root}: {g.val_f64} vs {want.val_f64}"
                assert all(got[r].group_id.size == 0 for r in range(R) if r != root)
            for root in (0, 2):
                boundary(root)
            # the type mix across ranks: v int64 on ranks 0 and 2, float64 on rank 1
            mix = [ctxs[r].register_part(2, mix_parts[r].files()) for r in range(R)]
            for root in (1, 0):
                got, errs = _collective(ctxs, lambda r: ctxs[r].scan_reduce(bydb.Query([mix[r]], ms[r].sids, MIX_AGGS), root=root))
                for r in range(R):
                    if r == root:
                        assert isinstance(errs[r], bydb.BydbError) and errs[r].code == EINVAL, f"root {root}: {errs[r]!r} {got[r]}"
                    else:
                        assert errs[r] is None, errs[r]
            # the mailboxes stay usable
            boundary(1)
        finally:
            for c in ctxs:
                c.close()


# ------------------------------------------------------------------ f. refusals
@gpu
def test_refusals_and_the_worst_status(bydb, gpu_ctx):
    import torch
    with random_shards(bydb, gpu_ctx, 3, seed=9) as sh:
        aggs = [("lat", SUM), ("calls", MAX)]
        t, host, lay = sh.tables(aggs)
        nb = lay["total_bytes"]
        qf = sh.q_final(aggs)
        for n, each in [(0, nb), (3, nb - 8), (3, nb + 8)]:
            with pytest.raises(bydb.BydbError) as e:
                gpu_ctx.partials_combine(qf, t.data_ptr(), n, each, sh.stream)
            assert e.value.code == EINVAL, (n, each)
        assert (t.cpu().numpy().view(np.uint64).reshape(3, -1) == host).all(), "a refused combine writes nothing"
        for call in (lambda: gpu_ctx.reduce_finalize(qf, t.data_ptr(), nb - 8, sh.stream),
                     lambda: gpu_ctx.partials_rows(qf, t.data_ptr(), nb - 8, sh.stream)):
            with pytest.raises(bydb.BydbError) as e:
                call()
            assert e.value.code == EINVAL
        # a device error of an asynchronous scan travels in its table; whatever that table's rank, the combined table fails
        part = build_part(*grid(6, 50, sid0=50_000), [("lat", F, np.full(300, 1.5), None), ("calls", I, np.arange(300), None)],
                          [("default", [("region", O.VT_STR, [b"r1"] * 300, None)])])
        h = gpu_ctx.register_part(_next_pid(), part.files())
        try:
            bad = bydb.Query([h], np.arange(50_000, 50_006, dtype=np.uint64), aggs, series_group=np.zeros(6, np.int32), n_groups=sh.G,
                             preds=[bydb.Pred("default", "region", O.OP_EQ, 5)])      # an int64 literal against a string tag
            for r in range(3):
                t2 = torch.zeros(3 * nb // 8, dtype=torch.int64, device="cuda")
                for slot in range(3):
                    if slot == r:
                        assert gpu_ctx.scan_partials(bad, t2.data_ptr() + slot * nb, nb, sh.stream, want_stats=False) is None
                    else:
                        gpu_ctx.scan_partials(sh.q(slot, aggs), t2.data_ptr() + slot * nb, nb, sh.stream)
                gpu_ctx.partials_combine(qf, t2.data_ptr(), 3, nb, sh.stream)
                for call in (lambda: gpu_ctx.reduce_finalize(qf, t2.data_ptr(), nb, sh.stream),
                             lambda: gpu_ctx.partials_rows(qf, t2.data_ptr(), nb, sh.stream)):
                    with pytest.raises(bydb.BydbError) as e:
                        call()
                    assert e.value.code == EINVAL, f"bad table at rank {r}"
        finally:
            gpu_ctx.release_part(h)


# ------------------------------------------------------------------ g. a field's type differs between tables
MIX_AGGS = [("v", SUM), ("v", COUNT), ("v", MIN), ("v", MAX), ("v", MEAN)]


def mix_measures():
    """v int64 ("vi"), v float64 ("vf"), and two measures without v ("none", "none2"); all series disjoint"""
    ms = {m.label: m for m in M.type_mix_cases()}
    for label, base in (("none", 500), ("none2", 600)):
        ms[label] = M.Measure(label, np.arange(base, base + 4), 50, [("w", I)], [("default", [("region", O.VT_STR)])], seed=base)
    return ms


@gpu
@pytest.mark.parametrize("order", [("vi", "vf"), ("vf", "vi"), ("vi", "none", "vf"), ("none", "vf", "none2", "vi")])
def test_type_mix_across_tables_fails(bydb, gpu_ctx, order):
    """v is int64 in one shard and float64 in another: one scan over both parts fails with BYDB_EINVAL (kErrTypeMix), and so
    must their combined tables, in finalisation and in the wire-shape rows"""
    ms = mix_measures()
    parts = [ms[k].own_part() for k in order]
    with Shards(bydb, gpu_ctx, parts, [ms[k].sids for k in order], [np.zeros(ms[k].sids.size, np.int32) for k in order], 1) as sh:
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg(sh.q_whole(MIX_AGGS))
        assert e.value.code == EINVAL
        t, host, lay = sh.tables(MIX_AGGS)
        got_t = sh.combine(t, len(parts), lay, MIX_AGGS)
        assert_same_table(got_t, fold(host, 1, 1), 1, 1, str(order))
        assert int(np.int64(got_t[-1])) >> 8 == K_ERR_TYPE_MIX
        for call in (lambda: sh.finalize(t, lay, MIX_AGGS),
                     lambda: gpu_ctx.partials_rows(sh.q_final(MIX_AGGS), t.data_ptr(), lay["total_bytes"], sh.stream)):
            with pytest.raises(bydb.BydbError) as e:
                call()
            assert e.value.code == EINVAL, order


@gpu
@pytest.mark.parametrize("order", [("none", "vf"), ("vi", "none"), ("none", "vi", "none2")])
def test_a_table_without_the_field_is_no_type_mix(bydb, gpu_ctx, order):
    """a table whose field met no block (type 0) next to a typed one: the typed table's type, no status"""
    ms = mix_measures()
    with Shards(bydb, gpu_ctx, [ms[k].own_part() for k in order], [ms[k].sids for k in order],
                [np.arange(ms[k].sids.size) % 2 for k in order], 2) as sh:
        t, host, lay = sh.tables(MIX_AGGS)
        got_t = sh.combine(t, len(order), lay, MIX_AGGS)
        assert_same_table(got_t, fold(host, 2, 1), 2, 1, str(order))
        typed = next(k for k in order if k != "none")
        assert int(np.int64(got_t[-1])) == (I if typed == "vi" else F)
        check_oracle(sh.finalize(t, lay, MIX_AGGS), sh.oracle(MIX_AGGS), MIX_AGGS, {"v": I if typed == "vi" else F}, str(order))


@gpu
def test_type_mix_inside_one_cold_path_call(bydb, gpu_ctx, monkeypatch, capfd):
    """bydb_scan_agg_host over ONE part whose first primary blocks hold v as int64 and whose last hold it as float64: the cold
    path parses the block index in slices and scans each into its own table; however the slices fall, the answer is
    BYDB_EINVAL, as for the same part registered and scanned at once"""
    n = 9000
    vi = M.Measure("vi", np.arange(1, n + 1), 2, [("v", I)], [("default", [("region", O.VT_STR)])], seed=41)
    vf = M.Measure("vf", np.arange(n + 1, 2 * n + 1), 2, [("v", F)], [("default", [("region", O.VT_STR)])], seed=42)
    part = M.mixed([vi, vf])
    files = part.files()
    assert len(M.primary_frames(files)) >= 3, "several primary blocks: the cold path parses them in several pieces"
    sids = np.arange(1, 2 * n + 1, dtype=np.uint64)
    h = gpu_ctx.register_part(_next_pid(), files)
    try:
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg(bydb.Query([h], sids, [("v", SUM), ("v", MAX)]))
        assert e.value.code == EINVAL
    finally:
        gpu_ctx.release_part(h)
    monkeypatch.setenv("BYDB_TRACE", "1")
    capfd.readouterr()
    with pytest.raises(bydb.BydbError) as e:
        gpu_ctx.scan_agg_host([files], bydb.Query([], sids, [("v", SUM), ("v", MAX), ("v", COUNT)]))
    slices = len(re.findall(r"\[bydb cold\] slice \d+ =", capfd.readouterr().err))
    assert e.value.code == EINVAL, f"{slices} slice(s): {e.value!r}"
    # each measure alone through the same path: its own answer
    monkeypatch.delenv("BYDB_TRACE")
    for m in (vi, vf):
        got = gpu_ctx.scan_agg_host([m.own_part().files()], bydb.Query([], m.sids, [("v", SUM), ("v", COUNT)]))
        want = O.run_query(O.Query([m.own_part()], m.sids, [("v", SUM), ("v", COUNT)]))
        check_oracle(got, want, [("v", SUM), ("v", COUNT)], {"v": m.fields[0][1]}, m.label)

"""Queries over many parts, and the version dedup, against the oracle at their boundaries (DESIGN.md 2, 4.3, 4.4).

A query may name up to 64 parts, in any order: a table snapshot lists a merged part, which covers older time, after the parts
it did not absorb.  What depends on the part count or order: series_reduce_kernel's overlap check (it raises an error when
series of disjoint parts look overlapping and the dedup did not run), detect_overlap_kernel's 8-slot span merge, the per-row
walk over the other parts in dedup_kernel phase 1, and the binary search that replaces the first-block table when
n_series x n_parts > 16 Mi.

Every query is checked three ways:
  - against the oracle (assert_parity);
  - against `model`: for each (series, timestamp) the highest version, the earliest part in the query on equal versions; then
    the time range, the predicates, and the fold rules of test_gpu_fallback.py over the stored (read back) float values;
  - against a survivor part: the rows the model keeps written into one part (rows that came from a part without the i column
    into a second part without it), the same query on the device over those alone -- rows, group ids, int64 values and float
    MIN / MAX exactly, float SUM / MEAN within 1e-9 * sum|x|.
An all-rows SUM takes the express lane over disjoint parts and never where parts overlap in the range.
"""
import dataclasses
import gc
import itertools
import struct
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_fallback import fold
from tests.test_gpu_keyed import KScan, build_keyed, mk
from tests.test_gpu_keyed_int64 import KScan64, mk64
from tests.test_gpu_masks import host_images
from tests.test_oracle_model_sweep import OPS

gpu = pytest.mark.gpu

SUM, COUNT, MIN, MAX, MEAN = O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FAM = "default"
AGGS = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("i", MEAN), ("f", SUM), ("f", COUNT), ("f", MIN), ("f", MAX), ("f", MEAN)]
EXPRESS = [("i", SUM), ("i", COUNT)]
BLOCK = 8193                     # the writer cuts a series into blocks of this many rows
EINVAL, ENOTSUP = -22, -95
FAIL6 = (0, 1, 2, 3, 5, 4)       # windows [0,9] [10,19] [20,29] [30,39] [50,59] [40,49]: a false overlap under a 4-slot merge
_pid = [500_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


# ------------------------------------------------------------------ parts and the model
class Part:
    """One part's rows in (series, timestamp) order: versions, int64 field i, float64 field f (the stored values), string tag
    region, int64 tag code.  A field left out of `fields` is not written: its cells read as nil."""

    def __init__(self, sid, ts, ver, seed=0, fields=("i", "f"), i=None, i_null=None, f=None, region=None, code=None):
        sid, ts, ver = np.asarray(sid, np.uint64), np.asarray(ts, np.int64), np.asarray(ver, np.int64)
        n = sid.size
        rng = np.random.default_rng(seed)
        o = np.lexsort((ts, sid))
        self.sid, self.ts, self.ver = sid[o], ts[o], ver[o]
        same = self.sid[1:] == self.sid[:-1]
        assert not (same & (self.ts[1:] == self.ts[:-1])).any(), "one row per (series, ts) in a part"
        self.i = (rng.integers(-1000, 1000, n) if i is None else np.asarray(i, np.int64))[o]
        self.i_null = (np.zeros(n, bool) if i_null is None else np.asarray(i_null, bool))[o]
        self.f = (np.round(rng.uniform(-50.0, 150.0, n), 2) if f is None else np.asarray(f, np.float64))[o]
        region = [b"r%d" % x for x in rng.integers(0, 3, n)] if region is None else region
        self.region = [region[k] for k in o]
        self.code = (rng.integers(0, 5, n) if code is None else np.asarray(code, np.int64))[o]
        self.fields = fields
        fl = []
        if "i" in fields:
            fl.append(("i", O.VT_INT64, self.i, self.i_null.astype(np.uint8) if self.i_null.any() else None))
        if "f" in fields:
            fl.append(("f", O.VT_FLOAT64, self.f, None))
        self.part = build_part(self.sid, self.ts, self.ver, fl,
                               [(FAM, [("region", O.VT_STR, self.region, None), ("code", O.VT_INT64, self.code, None)])])
        if "f" in fields:   # the decimal float page is lossy for long inputs: the model reads what the part holds
            back = O.scan_rows(O.Query([self.part], np.unique(self.sid), [("f", SUM)]))
            assert back["sid"].size == n
            self.f = back["fields"][0][2]

    @property
    def n(self):
        return self.sid.size

    def row(self, k):
        return dict(i=None if "i" not in self.fields or self.i_null[k] else int(self.i[k]),
                    f=None if "f" not in self.fields else float(self.f[k]), region=self.region[k], code=int(self.code[k]))

    def take(self, mask):
        m = np.asarray(mask, bool)
        return Part(self.sid[m], self.ts[m], self.ver[m], fields=self.fields, i=self.i[m], i_null=self.i_null[m], f=self.f[m],
                    region=[r for r, k in zip(self.region, m) if k], code=self.code[m])


def best_rows(parts, order):
    """{(series, ts): (part, row)}: the highest version, the earliest part in the query on equal versions"""
    best = {}
    for q, pi in enumerate(order):
        p = parts[pi]
        for k, (key, v) in enumerate(zip(zip(p.sid.tolist(), p.ts.tolist()), p.ver.tolist())):
            b = best.get(key)
            if b is None or (v, -q) > b[0]:
                best[key] = ((v, -q), pi, k)
    return {key: (pi, k) for key, (_, pi, k) in best.items()}


def survivor_parts(parts, keep):
    """the rows the model keeps: those from parts with the i column in one part (a nil i cell becomes a null cell), those
    from parts without it in a second part without it, so that a group still meets the column exactly where it did (every
    part here writes f).  The two hold different (series, ts), so their dedup keeps every row."""
    assert all("f" in p.fields for p in parts)
    out = []
    for with_i in (True, False):
        rows = [(parts[pi], k) for _, (pi, k) in sorted(keep.items()) if ("i" in parts[pi].fields) == with_i]
        if not rows:
            continue
        cells = [p.row(k) for p, k in rows]
        out.append(Part([p.sid[k] for p, k in rows], [p.ts[k] for p, k in rows], [p.ver[k] for p, k in rows],
                        fields=("i", "f") if with_i else ("f",), i=[c["i"] or 0 for c in cells], i_null=[c["i"] is None for c in cells],
                        f=[c["f"] for c in cells], region=[c["region"] for c in cells], code=[c["code"] for c in cells]))
    return out


def model(parts, keep, sids, groups, tmin, tmax, preds, aggs, top):
    """-> [(group, rows, [(value, x) per agg], fields met)] in result order.  A group meets a field column when one of its kept rows comes
    from a part that has it, null cell or not (aggregation.go:290-312); a group that never met it keeps the zero value for
    MIN / MAX and is null to Top-N (nulls sort lowest: last for desc, first for asc, top.go:88-117)."""
    gid = dict(zip((int(s) for s in sids), (int(g) for g in groups)))
    acc = {}
    for (s, t), (pi, k) in sorted(keep.items()):
        g = gid.get(s)
        if g is None or t < tmin or t > tmax:
            continue
        row = parts[pi].row(k)
        if not all(OPS[op](row[tag] is not None, 0 if row[tag] is None else (row[tag] > lit) - (row[tag] < lit)) for tag, op, lit in preds):
            continue
        e = acc.setdefault(g, [0, [], [], set()])
        e[0] += 1
        e[3].update(parts[pi].fields)
        if row["i"] is not None:
            e[1].append(row["i"])
        if row["f"] is not None:
            e[2].append(row["f"])
    out = []
    for g in sorted(acc):
        rows, iv, fv, met = acc[g]
        x = {"i": np.array(iv, np.int64), "f": np.array(fv, np.float64)}
        vals = [(fold(O.VT_INT64 if f == "i" else O.VT_FLOAT64, fn, x[f]) if f in met or fn not in (MIN, MAX) else 0, x[f]) for f, fn in aggs]
        out.append((g, rows, vals, met))
    if top:
        n, a, desc = top
        f, fn = aggs[a]
        null = [e for e in out if fn != COUNT and f not in e[3]]
        vals = sorted((e for e in out if fn == COUNT or f in e[3]), key=lambda e: e[2][a][0], reverse=desc)   # stable: ties keep group order
        out = (vals + null if desc else null + vals)[:n]
    return out


def check_model(got, exp, aggs, ctx, what="model"):
    assert got.group_id.tolist() == [e[0] for e in exp], f"{ctx}: group ids {got.group_id.tolist()[:12]} vs {what} {[e[0] for e in exp][:12]}"
    assert got.rows.tolist() == [e[1] for e in exp], f"{ctx}: rows {got.rows.tolist()[:12]} vs {what} {[e[1] for e in exp][:12]}"
    for i, (g, _, vals, _) in enumerate(exp):
        for a, ((f, fn), (m, x)) in enumerate(zip(aggs, vals)):
            where = f"{ctx}: group {g} agg {a} ({f},{fn}) vs {what}"
            if not got.is_float[a]:
                assert int(got.val_i64[i, a]) == m, f"{where}: {got.val_i64[i, a]} vs {m}"
            elif fn in (MIN, MAX):
                assert got.val_f64[i:i + 1, a].view(np.uint64)[0] == np.array([m]).view(np.uint64)[0], f"{where}: {got.val_f64[i, a]!r} vs {m!r}"
            else:
                tol = 1e-9 * float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1)
                assert abs(float(got.val_f64[i, a]) - float(m)) <= tol, f"{where}: {got.val_f64[i, a]!r} vs {m!r}"


def check_survivor(got, ref, exp, aggs, ctx):
    """the device over the parts against the device over the survivor part (exp: the model, for the float tolerances)"""
    assert got.group_id.tolist() == ref.group_id.tolist() and got.rows.tolist() == ref.rows.tolist(), f"{ctx}: survivor groups / rows"
    check_model(ref, exp, aggs, ctx, "model (survivor part)")
    for a, (_, fn) in enumerate(aggs):
        if not got.is_float[a]:
            assert got.val_i64[:, a].tolist() == ref.val_i64[:, a].tolist(), f"{ctx}: agg {a} vs survivor part"
        elif fn in (MIN, MAX):
            assert got.val_f64[:, a].view(np.uint64).tolist() == ref.val_f64[:, a].view(np.uint64).tolist(), f"{ctx}: agg {a} vs survivor part"
        else:
            for i, (_, _, vals, _) in enumerate(exp):
                x = vals[a][1]
                tol = 1e-9 * float(np.abs(x).sum()) / (max(x.size, 1) if fn == MEAN else 1)
                assert abs(float(got.val_f64[i, a]) - float(ref.val_f64[i, a])) <= tol, f"{ctx}: agg {a} group {i} vs survivor part"


class Case:
    """Parts registered once; queries over any order of their handles, each checked three ways."""

    def __init__(self, bydb, ctx, parts):
        self.bydb, self.ctx, self.parts = bydb, ctx, parts
        pid = _next_pid()
        self.h = [ctx.register_part(pid + i, p.part.files()) for i, p in enumerate(parts)]
        self.usid = np.unique(np.concatenate([p.sid for p in parts]))
        self.surv = {}

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for h in self.h + [h for hs in self.surv.values() for h in hs]:
            self.ctx.release_part(h)

    def query(self, order, sids=None, groups=None, n_groups=None, tmin=I64_MIN, tmax=I64_MAX, preds=(), aggs=AGGS, top=None):
        sids = self.usid if sids is None else np.asarray(sids, np.uint64)
        groups = (sids % 3).astype(np.int32) if groups is None else np.asarray(groups, np.int32)
        tn, ta, td = top or (0, 0, True)
        oq = O.Query([self.parts[i].part for i in order], sids, list(aggs), groups=groups, n_groups=n_groups or int(groups.max()) + 1,
                     tmin=tmin, tmax=tmax, preds=[O.Pred(FAM, t, op, v) for t, op, v in preds], top_n=tn, top_agg=ta, top_desc=td)
        return oq, to_gpu_query(self.bydb, [self.h[i] for i in order], oq)

    def survivor(self, keep):
        key = frozenset(keep.items())
        if key not in self.surv:
            pid = _next_pid()
            self.surv[key] = [self.ctx.register_part(pid + i, p.part.files()) for i, p in enumerate(survivor_parts(self.parts, keep))]
        return self.surv[key]

    def check(self, got, order, oq, q, ctx, express=None):
        assert_parity(got, O.run_query(oq), oq.aggs, ctx)
        keep = best_rows(self.parts, order)
        top = (oq.top_n, oq.top_agg, oq.top_desc) if oq.top_n else None
        preds = [(p.tag, p.op, p.value) for p in oq.preds]
        exp = model(self.parts, keep, oq.sids, oq.groups, oq.tmin, oq.tmax, preds, oq.aggs, top)
        check_model(got, exp, oq.aggs, ctx)
        ref = self.ctx.scan_agg(dataclasses.replace(q, parts=self.survivor(keep)))
        check_survivor(got, ref, exp, oq.aggs, ctx)
        if express is not None:
            n = got.stats.blocks_express_lane
            assert (n > 0) if express else (n == 0), f"{ctx}: {n} express-lane blocks"

    def run(self, order, ctx="", express=None, **kw):
        oq, q = self.query(order, **kw)
        got = self.ctx.scan_agg(q)
        self.check(got, order, oq, q, f"{ctx}/order {list(order)}", express)
        return got

    def sweep(self, order, ctx=""):
        """the standard pair: every function over three groups, and the all-rows SUM of the express lane"""
        self.run(order, ctx)
        self.run(order, ctx + "/express", express=not parts_overlap([self.parts[i] for i in order]), aggs=EXPRESS,
                 groups=np.zeros(self.usid.size))


def parts_overlap(parts):
    """capi.cu parts_overlap over the full time range: two non-empty parts whose [min_ts, max_ts] meet"""
    spans = [(int(p.ts.min()), int(p.ts.max())) for p in parts if p.n]
    return any(max(a[0], b[0]) <= min(a[1], b[1]) for a, b in itertools.combinations(spans, 2))


# ------------------------------------------------------------------ the part sets
def disjoint_parts(n, seed, width=10):
    """n parts, part w holding time window w (`width` steps): series 1..5 in every part, series 6 in parts 1 and n - 2 only,
    series 7 in part n // 2 only; 1..width rows per series and part at random steps of the window"""
    rng = np.random.default_rng(seed)
    parts = []
    for w in range(n):
        sids, ts = [], []
        for s in [1, 2, 3, 4, 5] + ([6] if w in (1, n - 2) else []) + ([7] if w == n // 2 else []):
            k = int(rng.integers(1, width + 1))
            sids += [s] * k
            ts += (T0 + (width * w + np.sort(rng.choice(width, size=k, replace=False))) * STEP).tolist()
        parts.append(Part(sids, ts, np.ones(len(sids)), seed=seed * 1000 + w))
    return parts


def many_orders(n, seed):
    rng = np.random.default_rng(seed)
    out = [tuple(range(n)), tuple(range(n - 1, -1, -1)), tuple(list(range(0, n, 2)) + list(range(1, n, 2)))]
    return out + [tuple(int(x) for x in rng.permutation(n)) for _ in range(3)]


def grid_parts(n, scheme, seed, npts=24, density=0.8):
    """n parts over one grid (series 1..3 at npts steps, each point present with probability `density`), series 9 in part 0 only;
    each part its own values and one version: `perm` a permutation of the part index, `ties` the top version on up to three
    parts, `equal` the same version everywhere"""
    rng = np.random.default_rng(seed)
    if scheme == "perm":
        vers = rng.permutation(n)
    elif scheme == "ties":
        vers = rng.integers(0, 3, n)
        vers[rng.choice(n, size=min(n, 3), replace=False)] = 7
    else:
        vers = np.full(n, 4)
    parts = []
    for j in range(n):
        sids, ts = [], []
        for s in (1, 2, 3):
            t = np.nonzero(rng.random(npts) < density)[0]
            sids += [s] * t.size
            ts += (T0 + t * STEP).tolist()
        if j == 0:
            sids += [9] * 5
            ts += (T0 + np.arange(5) * STEP).tolist()
        parts.append(Part(sids, ts, np.full(len(sids), vers[j]), seed=seed * 1000 + j))
    return parts


# ------------------------------------------------------------------ A. many parts, no overlap (the dedup does not run)
@gpu
@pytest.mark.parametrize("n", [5, 6])
def test_disjoint_parts_in_every_order(bydb, gpu_ctx, n):
    """Six time-disjoint parts in all 720 orders (a four-slot span merge in series_reduce_kernel takes 240 of them for an
    overlap and fails the query), five in all 120 (no order can fail a four-slot merge)."""
    with Case(bydb, gpu_ctx, disjoint_parts(n, seed=n)) as c:
        failed = []
        for order in itertools.permutations(range(n)):
            try:
                c.sweep(order, f"{n} parts")
            except bydb.BydbError as e:
                failed.append((order, e.code, str(e)))
        assert not failed, f"{len(failed)} of {len(list(itertools.permutations(range(n))))} orders fail, first {failed[:2]}"


@gpu
@pytest.mark.parametrize("n", [7, 8, 9, 16, 33, 64])
def test_disjoint_part_counts(bydb, gpu_ctx, n):
    """time order, reverse, interleaved (even windows first) and three shuffles, plus a range cut and predicates"""
    with Case(bydb, gpu_ctx, disjoint_parts(n, seed=100 + n)) as c:
        for order in many_orders(n, n):
            c.sweep(order, f"{n} parts")
            c.run(order, f"{n} parts/cut", tmin=T0 + 13 * STEP, tmax=T0 + (10 * n - 14) * STEP, preds=[("region", O.OP_NE, b"r1")])


@gpu
def test_65_parts_is_einval(bydb, gpu_ctx):
    parts = disjoint_parts(64, seed=7) + [Part([1], [T0 - STEP], [1])]
    with Case(bydb, gpu_ctx, parts) as c:
        _, q = c.query(range(65))
        with pytest.raises(bydb.BydbError) as e:
            gpu_ctx.scan_agg(q)
        assert e.value.code == EINVAL, e.value
        c.sweep(range(64), "64 of the 65 parts")


@gpu
def test_disjoint_out_of_order_keyed(bydb, gpu_ctx):
    """bydb_scan_agg_keyed over the failing six-part order, string and int64 key: insertion order follows time, not part order"""
    def windows(make):
        ws = []
        for w in range(6):
            ss = [make(s, w) for s in (1, 2, 3)] + ([make(4, w)] if w in (1, 4) else []) + ([make(5, w)] if w == 2 else [])
            ws.append((build_keyed(ss), ss))
        return ws
    keys = lambda s, w: [b"k%d" % ((s + w + r) % 3) for r in range(10)]   # noqa: E731
    with KScan(bydb, gpu_ctx, windows(lambda s, w: mk(s, keys(s, w), row0=10 * w))) as k:
        k.query(order=list(FAIL6), ctx="string key")
        k.query(order=list(FAIL6), tmin=T0 + 5 * STEP, tmax=T0 + 44 * STEP, ctx="string key, cut")
        k.query(order=list(FAIL6), top=(3, 0, True), ctx="string key, top")
    cells = lambda s, w: [(s * 7 + w + r) % 4 - 1 for r in range(10)]   # noqa: E731
    with KScan64(bydb, gpu_ctx, windows(lambda s, w: mk64(s, cells(s, w), row0=10 * w))) as k:
        k.query(order=list(FAIL6), ctx="int64 key")


@gpu
def test_disjoint_out_of_order_graph_and_host(bydb, gpu_ctx):
    """the prepared graph (capture, then replays) and bydb_scan_agg_host (pageable and pinned) over the failing order"""
    with Case(bydb, gpu_ctx, disjoint_parts(6, seed=6)) as c:
        for kw in (dict(), dict(aggs=EXPRESS, groups=np.zeros(c.usid.size))):
            oq, q = c.query(FAIL6, **kw)
            plain = gpu_ctx.scan_agg(q)
            c.check(plain, FAIL6, oq, q, "plain")
            g = gpu_ctx.prepare_graph(q)
            try:
                for it in range(4):
                    r = g.run()
                    assert r.group_id.tolist() == plain.group_id.tolist() and r.rows.tolist() == plain.rows.tolist(), it
                    assert r.val_i64.tolist() == plain.val_i64.tolist(), it
                    assert r.val_f64.view(np.uint64).tolist() == plain.val_f64.view(np.uint64).tolist(), it
            finally:
                g.close()
            for pinned in (False, True):
                got = gpu_ctx.scan_agg_host(host_images([c.parts[i].part for i in FAIL6], pinned), dataclasses.replace(q, parts=[]))
                c.check(got, FAIL6, oq, q, f"host images, pinned={pinned}")


@gpu
def test_disjoint_out_of_order_scan_reduce(bydb, gpu_ctx):
    """bydb_scan_reduce: three ranks as threads, each holding the failing six-part order of its series shard"""
    import faulthandler

    import torch
    R = 3
    n_dev = torch.cuda.device_count()
    parts = disjoint_parts(6, seed=16)
    gc.collect()
    gc.disable()
    faulthandler.dump_traceback_later(50, exit=False)
    ctxs = []
    try:
        with Case(bydb, gpu_ctx, parts) as c:
            shard = {int(s): k % R for k, s in enumerate(c.usid.tolist())}
            ctxs = [bydb.Context(device=r % n_dev) for r in range(R)]
            handles = [x.comm_export(1 << 20, R) for x in ctxs]
            for r, x in enumerate(ctxs):
                x.comm_connect(r, R, handles)
            pid = _next_pid()
            hs = [[x.register_part(pid + i, parts[i].take([shard[int(s)] == r for s in parts[i].sid]).part.files()) for i in FAIL6]
                  for r, x in enumerate(ctxs)]
            for kw in (dict(), dict(tmin=T0 + 7 * STEP, tmax=T0 + 52 * STEP, preds=[("code", O.OP_LT, 3)])):
                oq, q = c.query(FAIL6, **kw)
                got, errs = [None] * R, []

                def run(r):
                    try:
                        mine = np.array([shard[int(s)] == r for s in c.usid.tolist()])
                        got[r] = ctxs[r].scan_reduce(dataclasses.replace(q, parts=hs[r], series_ids=c.usid[mine],
                                                                         series_group=np.asarray(q.series_group)[mine]), root=0)
                    except Exception as e:  # noqa: BLE001
                        errs.append(repr(e))
                th = [threading.Thread(target=run, args=(r,)) for r in range(R)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                assert not errs, errs
                c.check(got[0], FAIL6, oq, q, f"scan_reduce {kw}")
                assert all(got[r].group_id.size == 0 for r in range(1, R))
    finally:
        for x in ctxs:
            x.close()
        faulthandler.cancel_dump_traceback_later()
        gc.enable()


@gpu
@pytest.mark.parametrize("overlap", [False, True])
def test_binary_search_fallback(bydb, gpu_ctx, overlap):
    """64 parts and 262 145 query series (most absent from every part): n_series x n_parts > 16 Mi, so the scan finds each
    series' first block by binary search instead of the first-block table"""
    parts = grid_parts(64, "ties", seed=64) if overlap else disjoint_parts(64, seed=65)
    sids = np.arange(1, 262_146, dtype=np.uint64)
    assert sids.size * 64 > 16 << 20
    with Case(bydb, gpu_ctx, parts) as c:
        for order in many_orders(64, 3)[3:4]:
            c.run(order, "fallback", sids=sids)
            c.run(order, "fallback/express", express=not overlap, sids=sids, aggs=EXPRESS, groups=np.zeros(sids.size))


# ------------------------------------------------------------------ B. the version dedup at its boundaries (the dedup runs)
@gpu
@pytest.mark.parametrize("n", [2, 3, 8, 9, 10, 64])
@pytest.mark.parametrize("scheme", ["perm", "ties", "equal"])
def test_same_grid(bydb, gpu_ctx, n, scheme):
    with Case(bydb, gpu_ctx, grid_parts(n, scheme, seed=n * 10 + len(scheme))) as c:
        for order in many_orders(n, n)[:2] + many_orders(n, n)[3:4]:
            c.sweep(order, f"{n} parts {scheme}")
        c.run(tuple(range(n)), "cut", tmin=T0 + 3 * STEP, tmax=T0 + 17 * STEP, preds=[("code", O.OP_GE, 2)])


def slot_parts(n, case):
    """n parts, part j in window win[j] (series 1..3, 10 steps each); series 8 overlaps in parts 0 and 1 so that the dedup runs.
    `first`: the last part repeats window 0.  `gap`: the 9th part is merged into detect_overlap's 8th slot, and the last part
    falls in the gap that merge covers (n = 10); at n = 9 the last part lies between the 7th and the 8th slot."""
    if case == "first":
        win = list(range(n - 1)) + [0]
    else:
        win = [0, 1, 2, 3, 4, 5, 6, 8, 10, 9][:n] if n == 10 else [0, 1, 2, 3, 4, 5, 6, 8, 7]
    rng = np.random.default_rng(n + len(case))
    parts = []
    for j, w in enumerate(win):
        sids, ts = [], []
        for s in (1, 2, 3):
            sids += [s] * 10
            ts += (T0 + (10 * w + np.arange(10)) * STEP).tolist()
        if j < 2:
            sids += [8] * 4
            ts += (T0 + np.arange(4) * 3 * STEP).tolist()
        parts.append(Part(sids, ts, np.full(len(sids), 1 + int(rng.integers(0, 3))), seed=200 + j))
    return parts


@gpu
@pytest.mark.parametrize("n", [9, 10])
@pytest.mark.parametrize("case", ["first", "gap"])
def test_eight_slot_merge(bydb, gpu_ctx, n, case):
    with Case(bydb, gpu_ctx, slot_parts(n, case)) as c:
        for order in (tuple(range(n)), tuple(range(n - 1, -1, -1))):
            c.sweep(order, f"{n} parts {case}")


POSITIONS = (0, 1, 31, 32, 33)
SIZES = (1, 2, 31, 32, 33, 8192, 8193)


def position_parts():
    """Part 0: series 10 + j of SIZES[j] rows (one block each) and series 20 of BLOCK + 40 rows (two blocks), at even steps.
    Part 1: for each series a duplicate at rows 0, 1, 31, 32, 33, count - 2, count - 1 of its block (versions alternate above
    and below part 0's), and rows that fall between the two blocks of series 20, before all of part 0's rows, after all of
    them, and on odd steps; series 20 also duplicates the ts_min / ts_max of both its blocks."""
    sids0, ts0, dup = [], [], {}
    for j, size in enumerate(list(SIZES) + [BLOCK + 40]):
        s = 10 + j if j < len(SIZES) else 20
        sids0 += [s] * size
        ts0 += (T0 + 2 * np.arange(size) * STEP).tolist()
        if s == 20:
            rows = {0, 1, 31, 32, 33, BLOCK - 2, BLOCK - 1, BLOCK, BLOCK + 1, size - 2, size - 1}
        else:
            rows = {r for r in POSITIONS + (size - 2, size - 1) if 0 <= r < size}
        dup[s] = sorted(rows)
    p0 = Part(sids0, ts0, np.full(len(sids0), 5), seed=300)
    sids1, ts1, ver1 = [], [], []
    for s, rows in dup.items():
        n = sids0.count(s)
        extra = [-2, 2 * n, 2 * n + 6, 3, 2 * n - 3] + ([2 * BLOCK - 1] if s == 20 else [])   # odd steps, before, after
        for k, r in enumerate(rows):
            sids1.append(s)
            ts1.append(T0 + 2 * r * STEP)
            ver1.append(7 if k % 2 == 0 else 3)
        for e in extra:
            if 0 <= e < 2 * n and e % 2 == 0:
                continue
            sids1.append(s)
            ts1.append(T0 + e * STEP)
            ver1.append(6)
    return [p0, Part(sids1, ts1, ver1, seed=301)], dup


@gpu
def test_duplicate_positions(bydb, gpu_ctx):
    """duplicates at rows 0, 1, 31, 32, 33 (the first shadow words) and count - 2, count - 1 (a partial last word) of blocks of
    1, 2, 31, 32, 33, 8192 and 8193 rows; between two blocks, on a block's ts_min / ts_max, before and after all rows"""
    parts, _ = position_parts()
    with Case(bydb, gpu_ctx, parts) as c:
        for order in ((0, 1), (1, 0)):
            c.sweep(order, "positions")
            groups = np.arange(c.usid.size)
            c.run(order, "positions/per series", groups=groups)
            for r in (0, 31, 32, 33, BLOCK - 1):   # time range cut at rows of series 20's first block
                t = T0 + 2 * r * STEP
                c.run(order, f"positions/from row {r}", groups=groups, tmin=t)
                c.run(order, f"positions/to row {r}", groups=groups, tmax=t)


def kind_parts():
    """Part 0, series by series (timestamp page, version page): 1 (DeltaConst, Const), 2 (DoD: irregular ascending steps, the
    encoder's choice for any non-constant ascending list, so no timestamp page is Delta; DeltaConst), 3 (a one-row block:
    Const, Const), 4 (negative timestamps, DoD; DoD versions), 5 (a block ending at INT64_MAX; Delta versions cycling 0, -1,
    INT64_MAX, INT64_MIN), 6 (DeltaConst; Delta versions going negative).  Part 1 repeats every third row of each series (and
    the one row of series 3) with versions cycling INT64_MIN, -1, 0, 1, INT64_MAX."""
    rng = np.random.default_rng(77)
    n = 40
    ts = {1: T0 + np.arange(n) * STEP, 2: T0 + np.cumsum(rng.integers(1, 9, n)) * STEP, 3: np.array([T0 + 5 * STEP]),
          4: -T0 + np.cumsum(rng.integers(1, 5, n)) * STEP, 5: I64_MAX - (n - 1 - np.arange(n)) * 3, 6: T0 + np.arange(n) * STEP}
    ver = {1: np.full(n, 4), 2: 3 + np.arange(n), 3: np.array([2]), 4: 1 + np.cumsum(rng.integers(1, 9, n)),
           5: np.tile([0, -1, I64_MAX, I64_MIN], n // 4), 6: np.concatenate([[6], rng.integers(-9, 9, n - 1)])}
    p0 = Part(np.concatenate([np.full(ts[s].size, s) for s in ts]), np.concatenate(list(ts.values())),
              np.concatenate(list(ver.values())), seed=400)
    lim = [I64_MIN, -1, 0, 1, I64_MAX]
    m = np.zeros(p0.n, bool)
    m[::3] = True
    m[p0.sid == 3] = True
    p1 = Part(p0.sid[m], p0.ts[m], [lim[k % 5] for k in range(int(m.sum()))], seed=401)
    return [p0, p1]


KINDS = {1: (O.ENC_DELTA_CONST, O.ENC_CONST), 2: (O.ENC_DELTA_OF_DELTA, O.ENC_DELTA_CONST), 3: (O.ENC_CONST, O.ENC_CONST),
         4: (O.ENC_DELTA_OF_DELTA, O.ENC_DELTA_OF_DELTA), 5: (O.ENC_DELTA_CONST, O.ENC_DELTA), 6: (O.ENC_DELTA_CONST, O.ENC_DELTA)}


@gpu
def test_page_kinds(bydb, gpu_ctx):
    with Case(bydb, gpu_ctx, kind_parts()) as c:
        for order in ((0, 1), (1, 0)):
            c.sweep(order, "kinds")
            c.run(order, "kinds/per series", groups=np.arange(c.usid.size))
            c.run(order, "kinds/range", groups=np.arange(c.usid.size), tmin=-T0 + 20 * STEP, tmax=I64_MAX - 30)


def hidden_parts():
    """Part 0 (version 1) and part 1 (version 2) over series 1..4 at 100 steps, part 1 on every other step: series 1's newer
    rows fail `region == r0` where the older pass it, series 2's newer i cells are null, part 1 holds no i column for series 3
    (it is a part of its own, part 2), series 4 is only in part 0 (no overlap) next to the overlapping ones."""
    n = 100
    t = T0 + np.arange(n) * STEP
    s0 = np.repeat([1, 2, 3, 4], n)
    p0 = Part(s0, np.tile(t, 4), np.ones(4 * n), seed=500, region=[b"r0"] * (4 * n))
    even = t[::2]
    p1 = Part(np.repeat([1, 2], even.size), np.tile(even, 2), np.full(2 * even.size, 2), seed=501, region=[b"r1"] * (2 * even.size),
              i_null=np.concatenate([np.zeros(even.size, bool), np.ones(even.size, bool)]))
    p2 = Part(np.full(even.size, 3), even, np.full(even.size, 2), seed=502, fields=("f",))
    return [p0, p1, p2]


@gpu
def test_hidden_rows(bydb, gpu_ctx):
    """a newer version hides an older row: failing a predicate, with a null cell, without the field column; time range cuts at
    rows 0, 31, 32, 33 and count - 1 of an overlapping block"""
    with Case(bydb, gpu_ctx, hidden_parts()) as c:
        per = np.arange(c.usid.size)
        for order in itertools.permutations(range(3)):
            c.sweep(order, "hidden")
            c.run(order, "hidden/pred", groups=per, preds=[("region", O.OP_EQ, b"r0")])
            c.run(order, "hidden/ne", groups=per, preds=[("region", O.OP_NE, b"r1"), ("code", O.OP_LE, 3)])
        # at the cut `to 0` series 3 keeps one row, from the part without the i column: its group never meets the column
        for r in (0, 31, 32, 33, 99):
            for order in ((0, 1, 2), (2, 1, 0)):
                c.run(order, f"hidden/from {r}", groups=per, tmin=T0 + r * STEP)
                c.run(order, f"hidden/to {r}", groups=per, tmax=T0 + r * STEP)
                for a, desc in ((2, True), (3, False), (0, True)):   # the never-met group is null to Top-N
                    c.run(order, f"hidden/to {r}/top {a} desc={desc}", groups=per, tmax=T0 + r * STEP, top=(3, a, desc))


@gpu
def test_groups_that_never_meet_the_column(bydb, gpu_ctx):
    """A group whose kept rows all come from blocks without the aggregated column keeps the zero value for MIN / MAX and is
    null to Top-N; a group that met only null cells keeps the empty-fold sentinels and competes with them.  One part without
    the column, then next to a part with it (no overlap, and overlapping so that the older rows with values are hidden)."""
    n = 40
    t = T0 + np.arange(n) * STEP
    bare = Part(np.repeat([1, 2], n), np.tile(t, 2), np.ones(2 * n), seed=600, fields=("f",))
    with Case(bydb, gpu_ctx, [bare]) as c:
        c.run((0,), "one part without i", groups=np.arange(2))
        c.run((0,), "one part without i/top", groups=np.arange(2), top=(2, 2, True))
    nulls = Part(np.repeat([3, 4], n), np.tile(t, 2), np.ones(2 * n), seed=601, i_null=np.arange(2 * n) >= n)
    older = Part(np.repeat([1, 2], n), np.tile(t, 2), np.zeros(2 * n), seed=602)
    with Case(bydb, gpu_ctx, [bare, nulls, older]) as c:
        per = np.arange(c.usid.size)
        for order in ((0, 1), (1, 0), (0, 1, 2), (2, 1, 0)):
            c.sweep(order, "without i")
            c.run(order, "without i/per series", groups=per)
            c.run(order, "without i/cut", groups=per, tmin=T0 + 3 * STEP, tmax=T0 + 31 * STEP)
            for a in (0, 2, 3, 4, 7):
                for desc in (True, False):
                    c.run(order, f"without i/top {a} desc={desc}", groups=per, top=(4, a, desc))


@gpu
def test_top_n_over_deduplicated_groups(bydb, gpu_ctx):
    """Top-N over groups whose rows come out of the dedup, both directions; COUNT ties on every series (no nulls, same grid)"""
    with Case(bydb, gpu_ctx, grid_parts(4, "ties", seed=90, npts=30, density=1.0)) as c:
        per = np.arange(c.usid.size)
        for order in ((0, 1, 2, 3), (3, 1, 0, 2)):
            for desc in (True, False):
                for a in (0, 1, 5, 8):
                    c.run(order, f"top {a} desc={desc}", groups=per, top=(2, a, desc))
                c.run(order, f"top all desc={desc}", groups=per, top=(10, 1, desc))


# ------------------------------------------------------------------ C. what the cases rest on (no GPU)
def part_blocks(part):
    """(series, count, ts_min, ts_max, timestamp encode type, version encode type) of every block, read from the part's
    meta.bin (primaryBlockMetadata, 40 bytes each) and primary.bin (blockMetadata records, block_metadata.go:133-168)"""
    files = part.files()
    meta, out = O.zstd_decompress(files["meta.bin"]), []
    for k in range(0, len(meta), 40):
        off, size = struct.unpack(">QQ", meta[k + 24:k + 40])
        buf, pos = O.zstd_decompress(files["primary.bin"][off:off + size]), 0

        def take(fmt):
            nonlocal pos
            v = struct.unpack_from(fmt, buf, pos)[0]
            pos += struct.calcsize(fmt)
            return v

        def varu():
            nonlocal pos
            v = s = 0
            while True:
                b = buf[pos]
                pos += 1
                v |= (b & 0x7f) << s
                s += 7
                if b < 0x80:
                    return v

        while pos < len(buf):
            sid = take(">Q")
            varu()
            count = varu()
            varu()
            varu()
            ts_min, ts_max, enc = take(">q"), take(">q"), take("B")
            varu()
            take(">q")
            ver_enc = take("B")
            for _ in range(varu()):   # tag families: name, offset, size
                ln = varu()
                pos += ln
                varu()
                varu()
            for _ in range(varu()):   # fields: name, value type, offset, size
                ln = varu()
                pos += ln
                take("B")
                varu()
                varu()
            out.append((sid, count, ts_min, ts_max, enc - 4, ver_enc))
    return out


def four_slot_overlap(spans):
    """series_reduce_kernel's former check: spans kept in four slots, a fifth part and later merged into the last slot"""
    slots, hit = [], False
    for lo, hi in spans:
        hit = hit or any(not (hi < a or lo > b) for a, b in slots)
        if len(slots) < 4:
            slots.append([lo, hi])
        else:
            slots[3] = [min(lo, slots[3][0]), max(hi, slots[3][1])]
    return hit


def test_case_foundations():
    # the four-slot merge fails 0 of 120 orders of five disjoint windows, 240 of 720 at six (FAIL6 among them), 3360 of 5040 at seven
    for n, want in ((5, 0), (6, 240), (7, 3360)):
        w = [(10 * k, 10 * k + 9) for k in range(n)]
        assert sum(four_slot_overlap([w[i] for i in p]) for p in itertools.permutations(range(n))) == want
    assert four_slot_overlap([(10 * k, 10 * k + 9) for k in FAIL6])
    # the case-A windows are pairwise disjoint, part by part (the directory's min / max) and series by series
    for n, seed in ((5, 5), (6, 6), (6, 16), (64, 65), (64, 7)):
        parts = disjoint_parts(n, seed)
        assert not parts_overlap(parts)
        metas = [p.part.meta() for p in parts]
        assert all(m["min_ts"] == int(p.ts.min()) and m["max_ts"] == int(p.ts.max()) for m, p in zip(metas, parts))
        assert all(a["max_ts"] < b["min_ts"] for a, b in zip(metas, metas[1:]))
        assert {6} <= set(parts[1].sid.tolist()) and sum(7 in p.sid.tolist() for p in parts) == 1
    for n, case in ((9, "first"), (10, "gap")):
        assert parts_overlap(slot_parts(n, case))
    # the timestamp and version pages have the encode types claimed, as the part's block directory records them
    p0 = kind_parts()[0]
    blocks = part_blocks(p0.part)
    assert [b[0] for b in blocks] == sorted(KINDS)
    for s, count, ts_min, ts_max, ts_enc, ver_enc in blocks:
        t = p0.ts[p0.sid == s]
        assert (count, ts_min, ts_max) == (t.size, int(t[0]), int(t[-1])) and (ts_enc, ver_enc) == KINDS[s], s
    assert {I64_MIN, I64_MAX, -1, 0} <= set(p0.ver[p0.sid == 5].tolist()) and p0.ts[p0.sid == 5].max() == I64_MAX
    assert p0.ts[p0.sid == 4].max() < 0
    # the planted duplicates sit on the claimed rows and blocks: one block per series, two for series 20, each block's
    # ts_min / ts_max duplicated in part 1 (the directory's blocks)
    (q0, q1), dup = position_parts()
    blocks = part_blocks(q0.part)
    assert [(b[0], b[1]) for b in blocks] == [(10 + j, n) for j, n in enumerate(SIZES)] + [(20, BLOCK), (20, 40)]
    for s, _, ts_min, ts_max, _, _ in blocks:
        assert {ts_min, ts_max} <= set(q1.ts[q1.sid == s].tolist()), s
    for s, rows in dup.items():
        t0, t1 = q0.ts[q0.sid == s], set(q1.ts[q1.sid == s].tolist())
        assert {int(t0[r]) for r in rows} == t1 & set(t0.tolist()), s
        assert {r for r, t in enumerate(t0.tolist()) if t in t1} == set(rows), s
    t20 = q0.ts[q0.sid == 20]
    assert int(t20[BLOCK - 1]) + STEP in set(q1.ts[q1.sid == 20].tolist())   # between the two blocks
    # the survivor parts hold exactly the model's rows, and the i column exactly where the model's rows had it
    for parts, order in ((hidden_parts(), (1, 0, 2)), (grid_parts(3, "ties", seed=5), (2, 0, 1))):
        keep = best_rows(parts, order)
        sps = survivor_parts(parts, keep)
        assert [sp.fields for sp in sps] == [("i", "f")] + ([("f",)] if any(p.fields == ("f",) for p in parts) else [])
        assert {(int(s), int(t)) for sp in sps[1:] for s, t in zip(sp.sid, sp.ts)} == \
            {key for key, (pi, _) in keep.items() if parts[pi].fields == ("f",)}
        sp = sps[0]
        keep = {key: v for key, v in keep.items() if "i" in parts[v[0]].fields}
        got = O.scan_rows(O.Query([sp.part], np.unique(sp.sid), [("i", SUM), ("f", SUM)]))
        want = sorted(keep.items())
        assert list(zip(got["sid"].tolist(), got["ts"].tolist())) == [k for k, _ in want]
        assert got["version"].tolist() == [int(parts[pi].ver[k]) for _, (pi, k) in want]
        (_, _, iv, inull), (_, _, fv, _) = got["fields"]
        rows = [parts[pi].row(k) for _, (pi, k) in want]
        assert [None if nl else int(v) for v, nl in zip(iv.tolist(), inull.tolist())] == [r["i"] for r in rows]
        assert fv.tolist() == [r["f"] for r in rows]

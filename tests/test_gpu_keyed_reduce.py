"""Group-by on a stored tag across ranks (bydb_scan_reduce_keyed, DESIGN.md 5): R = 3 ranks as threads, one context each on
device r % device_count (a one-GPU box exercises the host-polled shared-device waits, a multi-GPU box the device-side waits).
Every rank passes the same query but its parts.  Each answer of the root is checked
  - against the oracle with group_key over all ranks' parts (for an int64 key: keyed on its string twin);
  - against bydb_scan_agg_keyed on one context, over one part holding every rank's rows (series shards) or over the ranks'
    parts themselves (time shards): group ids, key bytes, rows and int64 values exactly and in order, floats within 1e-12;
  - on n_keys, on rows_matched summed over the ranks, and on every other rank: no rows, no keys, and the blocks of its own passes
    (V_r x its selected blocks, as bydb_scan_agg_keyed over its shard counts them).
"""
import dataclasses
import faulthandler
import gc
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, to_gpu_query
from tests.test_gpu_fallback import COUNT, MAX, MEAN, MIN, SUM, Series
from tests.test_gpu_keyed import AGGS, FAM, KT, build_keyed, mk, std_fields
from tests.test_gpu_keyed_int64 import KX, int_tag, twin
from tests.test_gpu_masks import I64_MAX, I64_MIN

gpu = pytest.mark.gpu

R = 3
ENOMEM, EINVAL, ENOTSUP = -12, -22, -95
_pid = [300_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


@pytest.fixture
def quiet():
    # Ranks may share one device: a finaliser of an unrelated object that frees page-locked memory on a rank's thread in the middle
    # of a collective would synchronise with a peer's wait.  Nothing unrelated may be torn down here; a stall shows every thread.
    gc.collect()
    gc.disable()
    faulthandler.dump_traceback_later(50, exit=False)
    yield
    faulthandler.cancel_dump_traceback_later()
    gc.enable()


class Ranks:
    """R contexts with connected mailboxes of `slot` bytes; each rank's shard (a list of parts) registered on its context"""

    def __init__(self, bydb, slot, shards=None):
        import torch
        n_dev = torch.cuda.device_count()
        self.bydb = bydb
        self.ctxs = [bydb.Context(device=r % n_dev) for r in range(R)]
        handles = [c.comm_export(slot, R) for c in self.ctxs]
        for r, c in enumerate(self.ctxs):
            c.comm_connect(r, R, handles)
        self.hs = [[] for _ in range(R)]
        if shards:
            self.register(shards)

    def register(self, shards):
        pid = _next_pid()
        self.hs = [[c.register_part(pid + i, p.files()) for i, p in enumerate(shard)] for c, shard in zip(self.ctxs, shards)]

    def run(self, fn):
        """fn(r) on R threads -> (results, codes): codes[r] = 0 or the BydbError code of rank r"""
        res, codes, errs = [None] * R, [0] * R, []

        def body(r):
            try:
                res[r] = fn(r)
            except self.bydb.BydbError as e:
                codes[r] = e.code
            except Exception as e:  # noqa: BLE001
                errs.append(repr(e))
        th = [threading.Thread(target=body, args=(r,)) for r in range(R)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        return res, codes

    def keyed(self, qs, root, key=KT, max_values=256, vt=0):
        return self.run(lambda r: self.ctxs[r].scan_reduce_keyed(qs[r], FAM, key, root=root, max_values=max_values, value_type=vt))

    def close(self):
        for c in self.ctxs:
            c.close()


class Case:
    """Shards of one data set: `shards[r]` are rank r's parts, `whole` the parts one context scans for the same answer"""

    def __init__(self, shards, whole, gid):
        self.shards, self.whole, self.gid = shards, whole, gid
        self.sids = np.array(sorted(gid), dtype=np.uint64)

    def oquery(self, parts, aggs=AGGS, preds=(), tmin=I64_MIN, tmax=I64_MAX, top=None, sids=None):
        sids = self.sids if sids is None else np.array(sorted(sids), dtype=np.uint64)
        tn, ta, td = top or (0, 0, True)
        return O.Query(parts, sids, list(aggs), groups=np.array([self.gid[int(s)] for s in sids], np.int32),
                       n_groups=max(self.gid.values()) + 1, tmin=tmin, tmax=tmax, preds=list(preds), top_n=tn, top_agg=ta, top_desc=td)


def same(got, want, ctx):
    """group ids, key bytes, rows and int64 values exactly and in order; floats within 1e-12 relative"""
    assert got.group_id.tolist() == want.group_id.tolist(), f"{ctx}: group ids {got.group_id[:12]} vs {want.group_id[:12]}"
    assert got.key == want.key, f"{ctx}: keys {got.key[:12]} vs {want.key[:12]}"
    assert got.rows.tolist() == want.rows.tolist(), f"{ctx}: rows"
    assert got.is_float.tolist() == want.is_float.tolist(), f"{ctx}: typing"
    assert got.val_i64.tolist() == want.val_i64.tolist(), f"{ctx}: int64 values"
    assert np.allclose(got.val_f64, want.val_f64, rtol=1e-12, atol=0, equal_nan=True), f"{ctx}: float values"


def check(bydb, gpu_ctx, ranks, case, root, key=KT, vt=0, twin=None, max_values=256, label="", **kw):
    """one keyed collective against the oracle, the single-context call and the counters; -> the root's result"""
    ctx = f"{label}/root{root}/{kw}"
    qs = [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], **kw)) for r in range(R)]
    res, codes = ranks.keyed(qs, root, key, max_values, vt)
    assert codes == [0] * R, f"{ctx}: {codes}"
    got = res[root]
    pid = _next_pid()
    whole = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(case.whole)]
    try:
        one = gpu_ctx.scan_agg_keyed(to_gpu_query(bydb, whole, case.oquery(case.whole, **kw)), FAM, key, max_values, vt)
    finally:
        for h in whole:
            gpu_ctx.release_part(h)
    same(got, one, ctx)
    want = O.run_query(dataclasses.replace(case.oquery([p for s in case.shards for p in s], **kw), group_key=(FAM, twin or key)))
    if got.group_id.size or want.group_id.size:
        assert_parity(got, want, kw.get("aggs", AGGS), ctx)
    assert got.key == want.key, f"{ctx}: keys vs oracle"
    assert got.n_keys == one.n_keys, f"{ctx}: n_keys {got.n_keys} vs {one.n_keys}"
    assert sum(res[r].stats.rows_matched for r in range(R)) == one.stats.rows_matched, ctx
    for r in range(R):
        if r == root:
            continue
        assert res[r].group_id.size == 0 and res[r].n_keys == 0, f"{ctx}: rank {r} got rows"
        alone = ranks.ctxs[r].scan_agg_keyed(qs[r], FAM, key, max_values, vt)
        assert res[r].stats.blocks_scanned == alone.stats.blocks_scanned, f"{ctx}: rank {r} blocks"
    return got


# ------------------------------------------------------------------ data
S_TAG = "s"


def split(pieces, gid, int64=False):
    """pieces: (rank, sid, cells, row0), each a contiguous window of one series' rows.  -> Case whose rank r holds one part with its
    pieces, and whose `whole` is one part with every series in full (the fields of std_fields over the whole series, sliced)"""
    by_sid = {}
    for r, sid, cells, row0 in pieces:
        by_sid.setdefault(sid, []).append((row0, list(cells), r))
    per_rank, whole = [[] for _ in range(R)], []

    def series(sid, cells, row0, fields, stag):
        tags = {KT: int_tag(cells), KX: twin(cells)} if int64 else {KT: cells}
        return Series(sid, fields, {**tags, S_TAG: stag}, row0=row0)
    for sid, ps in sorted(by_sid.items()):
        ps.sort(key=lambda p: p[0])
        lo = ps[0][0]
        n = ps[-1][0] + len(ps[-1][1]) - lo
        f = std_fields(sid, n)
        stag = [b"x" if (i + sid) % 3 else b"y" for i in range(n)]
        cells = [None] * n
        for row0, cs, r in ps:
            a = row0 - lo
            cells[a:a + len(cs)] = cs
            per_rank[r].append(series(sid, cs, row0, {k: (vt, v[a:a + len(cs)], None) for k, (vt, v, _) in f.items()},
                                      stag[a:a + len(cs)]))
        assert sum(len(p[1]) for p in ps) == n, f"series {sid}: windows must tile its rows"
        whole.append(series(sid, cells, lo, f, stag))
    return Case([[build_keyed(ss)] for ss in per_rank], [build_keyed(whole)], gid)


def series_case(pool_of=None):
    """12 series by series range (4 per rank), a string key with values shared by all ranks, values unique to one rank, nil on
    rank 0 and "" on rank 1; group 3 lives on rank 2 only, group 2 starts on rank 1"""
    rng = np.random.default_rng(11)
    pieces = []
    for r in range(R):
        pool = pool_of(r) if pool_of else [b"a", b"b", b"c", b"u%d" % r] + ([None] if r == 0 else [b""] if r == 1 else [b"z" * 64])
        for sid in range(4 * r + 1, 4 * r + 5):
            n = 300 + 37 * sid
            cells = [pool[(i + sid) % len(pool)] for i in range(n)] if sid % 2 else [pool[int(x)] for x in rng.integers(0, len(pool), n)]
            pieces.append((r, sid, cells, 0))
    gid = {1: 0, 2: 1, 3: 0, 4: 1, 5: 1, 6: 2, 7: 2, 8: 1, 9: 3, 10: 2, 11: 3, 12: 3}
    return split(pieces, gid)


def time_case():
    """6 series, each cut into three time windows, window r on rank r; an int64 key with nil (rank 0) next to 0 (rank 1); value
    99 first seen on rank 2 by series 1, whose earlier windows on ranks 0 and 1 do not hold it"""
    pieces = []
    for sid in range(1, 7):
        row0 = 0
        for r in range(R):
            pool = [7, -3, 1 << 40, None if r == 0 else 0] + ([99] if r == 2 and sid == 1 else [5 + r])
            n = 200 + 10 * sid + 7 * r
            pieces.append((r, sid, [pool[(i * (sid + 1) + r) % len(pool)] for i in range(n)], row0))
            row0 += n
    return split(pieces, {sid: sid % 2 for sid in range(1, 7)}, int64=True)


def order_case():
    """series 1 holds `p` on ranks 0 and 1 and first shows `late` in its window on rank 2; `only2` lives on rank 2 alone; group 2's
    only series (4) and group 1's second series (3) live on rank 2, group 1's first (2) on rank 1"""
    p = [(0, 1, [b"p"] * 40, 0), (1, 1, [b"p", b"q"] * 20, 40), (2, 1, [b"p"] * 5 + [b"late"] * 5 + [b"q"] * 5, 80),
         (1, 2, [b"q", b"p"] * 10, 0), (2, 3, [b"only2", b"p"] * 10, 0), (2, 4, [b"p", b"q"] * 10, 0)]
    return split(p, {1: 0, 2: 1, 3: 1, 4: 2})


def slot_for(bydb, case, max_values=256, **kw):
    q = to_gpu_query(bydb, [], case.oquery([], **kw))
    return bydb.keyed_reduce_slot_bytes(q, FAM, KT, max_values)


QUERIES = [
    dict(),
    dict(aggs=[("i", COUNT), ("f", SUM)], top=(5, 0, True)),
    dict(aggs=[("i", COUNT), ("f", MIN)], top=(4, 0, False)),
    dict(aggs=[("f", MEAN), ("i", MAX), ("i", SUM)], tmin=T0 + 50 * STEP, tmax=T0 + 700 * STEP),
    dict(aggs=[("i", SUM), ("f", MAX), ("i", MIN)], preds=[O.Pred(FAM, S_TAG, O.OP_EQ, b"x")]),
]


def plain_ok(bydb, gpu_ctx, ranks, case, root):
    """a plain bydb_scan_reduce over the same shards answers like one context: the epochs stayed in step"""
    aggs = [("i", SUM), ("f", SUM), ("i", COUNT)]
    qs = [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r], aggs=aggs)) for r in range(R)]
    res, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce(qs[r], root=root))
    assert codes == [0] * R, codes
    pid = _next_pid()
    whole = [gpu_ctx.register_part(pid + i, p.files()) for i, p in enumerate(case.whole)]
    try:
        want = gpu_ctx.scan_agg(to_gpu_query(bydb, whole, case.oquery(case.whole, aggs=aggs)))
    finally:
        for h in whole:
            gpu_ctx.release_part(h)
    got = res[root]
    assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist()
    assert got.val_i64.tolist() == want.val_i64.tolist() and np.allclose(got.val_f64, want.val_f64, rtol=1e-12, atol=0)


def refused(bydb, ranks, case, root, want_codes, qs=None, **keyed):
    qs = qs or [to_gpu_query(bydb, ranks.hs[r], case.oquery(case.shards[r])) for r in range(R)]
    _, codes = ranks.keyed(qs, root, **keyed)
    assert codes == want_codes, (codes, want_codes)


# ------------------------------------------------------------------ tests
@gpu
def test_series_and_time_shards(bydb, gpu_ctx, quiet):
    """sharding by series range (string key) and by time window (int64 key): aggregates, Top-N both ways with COUNT ties, a time
    cut and a dictionary predicate, roots 0 and 2"""
    sc, tc = series_case(), time_case()
    ranks = Ranks(bydb, max(slot_for(bydb, sc), slot_for(bydb, tc)))
    try:
        ranks.register(sc.shards)
        for root in (0, 2):
            for kw in QUERIES:
                check(bydb, gpu_ctx, ranks, sc, root, label="series", **kw)
        ranks.register(tc.shards)
        for root in (0, 2):
            for kw in QUERIES:
                check(bydb, gpu_ctx, ranks, tc, root, vt=bydb.VT_INT64, twin=KX, label="time", **kw)
    finally:
        ranks.close()


@gpu
def test_insertion_order_across_ranks(bydb, gpu_ctx, quiet):
    """a value first seen on a later rank in a series' later window, a value on one rank only, a group whose first series is on a
    later rank, and Top-N ties resolved by the insertion order of the whole scan"""
    case = order_case()
    ranks = Ranks(bydb, slot_for(bydb, case), case.shards)
    try:
        for root in (0, 2):
            got = check(bydb, gpu_ctx, ranks, case, root, label="order")
            assert list(zip(got.group_id.tolist(), got.key))[:3] == [(0, b"p"), (0, b"q"), (0, b"late")], got.key
            check(bydb, gpu_ctx, ranks, case, root, label="order-top", aggs=[("i", COUNT)], top=(4, 0, True))
            check(bydb, gpu_ctx, ranks, case, root, label="order-top-asc", aggs=[("i", COUNT)], top=(3, 0, False))
    finally:
        ranks.close()


@gpu
def test_union_edges(bydb, gpu_ctx, quiet):
    """a rank without a selected block, all ranks empty, a union of exactly 256 values, and one of max_values + 1 with every rank
    under the cap (ENOMEM at the root only)"""
    big = split([(r, r + 1, [b"v%03d" % v for v in range(78 * r, 78 * r + 100)], 0) for r in range(R)], {1: 0, 2: 1, 3: 0})
    cap = split([(r, r + 1, [b"a%02d" % v for v in range(7 * r, 7 * r + 7)] * 3, 0) for r in range(R)], {1: 0, 2: 0, 3: 1})
    ranks = Ranks(bydb, slot_for(bydb, big))
    try:
        ranks.register(big.shards)
        for root in (0, 2):
            got = check(bydb, gpu_ctx, ranks, big, root, label="256")
            assert got.n_keys == 256
            # rank 1 selects no block (its series is not asked for): V_r = 0
            got = check(bydb, gpu_ctx, ranks, big, root, label="rank1-empty", sids=[1, 3])
            assert got.n_keys == 200 and b"v100" not in got.key
            got = check(bydb, gpu_ctx, ranks, big, root, label="all-empty", tmin=T0 + 10**6 * STEP, tmax=T0 + 2 * 10**6 * STEP)
            assert got.n_keys == 0 and got.group_id.size == 0
        ranks.register(cap.shards)
        for root in (0, 2):
            want = [0] * R
            want[root] = ENOMEM
            refused(bydb, ranks, cap, root, want, max_values=20)
            got = check(bydb, gpu_ctx, ranks, cap, root, max_values=21, label="cap21")
            assert got.n_keys == 21
    finally:
        ranks.close()


@gpu
def test_refusals_keep_the_epochs_in_step(bydb, gpu_ctx, quiet):
    """every refusal is followed by a plain and a keyed collective that answer correctly"""
    sc = series_case()
    ranks = Ranks(bydb, slot_for(bydb, sc), sc.shards)
    try:
        def after(root):
            ranks.register(sc.shards)
            plain_ok(bydb, gpu_ctx, ranks, sc, root)
            check(bydb, gpu_ctx, ranks, sc, root, label="after", **QUERIES[1])
        # series 1 also on rank 1, over times that intersect its rows on rank 0
        st = {S_TAG: [b"x"] * 50}
        inter = Case([[build_keyed([mk(1, [b"a"] * 50, tags=st)])], [build_keyed([mk(1, [b"b"] * 50, row0=49, tags=st), mk(2, [b"a"] * 50, tags=st)])],
                      [build_keyed([mk(3, [b"c"] * 50, tags=st)])]], None, {1: 0, 2: 0, 3: 0})
        for root in (0, 2):
            ranks.register(inter.shards)
            want = [0] * R
            want[root] = ENOTSUP
            refused(bydb, ranks, inter, root, want)
            after(root)
        # two parts of rank 2 that overlap in time
        ranks.register(sc.shards)
        ranks.hs[2].append(ranks.ctxs[2].register_part(_next_pid(), build_keyed([mk(13, [b"a"] * 20, tags={S_TAG: [b"x"] * 20})]).files()))
        refused(bydb, ranks, sc, 0, [ENOTSUP, 0, ENOTSUP])
        after(0)
        # the key declared int64 on a string tag: every rank's discovery refuses it
        refused(bydb, ranks, sc, 1, [EINVAL] * R, vt=bydb.VT_INT64)
        after(1)
        # ranks that disagree on the series or on max_values
        qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r], sids=sc.sids[:-1] if r == 2 else None)) for r in range(R)]
        refused(bydb, ranks, sc, 0, [EINVAL, 0, 0], qs=qs)
        after(0)
        qs = [to_gpu_query(bydb, ranks.hs[r], sc.oquery(sc.shards[r])) for r in range(R)]
        _, codes = ranks.run(lambda r: ranks.ctxs[r].scan_reduce_keyed(qs[r], FAM, KT, root=2, max_values=128 if r == 1 else 256))
        assert codes == [0, 0, EINVAL], codes
        after(2)
    finally:
        ranks.close()
    # mailboxes sized for 4 values; rank 1 finds 6 (EINVAL on rank 1 and at the root), the others 2 and 3
    small = series_case(lambda r: [[b"a", b"b", b"c"], [b"a", b"b", b"c", b"d", b"e", b"f"], [b"a", b"g"]][r])
    ranks = Ranks(bydb, slot_for(bydb, small, max_values=4), small.shards)
    try:
        refused(bydb, ranks, small, 0, [EINVAL, EINVAL, 0])
        plain_ok(bydb, gpu_ctx, ranks, small, 0)
        got = check(bydb, gpu_ctx, ranks, small, 0, label="small-fits", sids=[s for s in range(1, 13) if not 5 <= s <= 8])
        assert got.n_keys == 4 and set(got.key) == {b"a", b"b", b"c", b"g"}
    finally:
        ranks.close()


@gpu
def test_keyed_and_plain_collectives_alternate(bydb, gpu_ctx, quiet):
    """keyed and plain collectives alternating over rotating roots reuse both slot parities of every root"""
    sc = series_case()
    ranks = Ranks(bydb, slot_for(bydb, sc), sc.shards)
    try:
        for it in range(8):
            root = it % R
            if it % 2:
                plain_ok(bydb, gpu_ctx, ranks, sc, root)
            else:
                check(bydb, gpu_ctx, ranks, sc, root, label=f"seq{it}", **QUERIES[it % len(QUERIES)])
    finally:
        ranks.close()

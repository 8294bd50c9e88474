"""-m gpu: a prepared query's replays run in device memory the query owns (partial table, step scratch, finalisation scratch),
start with one reset kernel and end with one read-back that carries the result rows and the step's zero page.

Every replay must give the plain call's answer and counters, however often it runs, whatever other prepared queries run in
between, and whatever happens to the context's parts meanwhile."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, build_part, grid

pytestmark = pytest.mark.gpu

COUNTERS = ("rows_scanned", "rows_matched", "page_bytes", "blocks_scanned", "blocks_slow_lane", "slow_lane_reasons", "blocks_express_lane")
_pid = [9_500_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def _assert_same(got, want, what):
    assert {k: getattr(got.stats, k) for k in COUNTERS} == {k: getattr(want.stats, k) for k in COUNTERS}, what
    assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), what
    assert got.is_float.tolist() == want.is_float.tolist(), what
    assert got.val_i64.tolist() == want.val_i64.tolist(), what
    assert got.val_f64.view(np.uint64).tolist() == want.val_f64.view(np.uint64).tolist(), what


def _part(rng, n_series=24, n_pts=3000, shift=0):
    """delta int64, decimal floats, a non-decimal float field (raw-cell pages: the slow lane) and a dictionary tag"""
    sids, ts, ver = grid(n_series, n_pts)
    n = sids.size
    calls = rng.integers(-500, 500, n) + shift
    lat = np.round(rng.normal(30, 6, n), 2)
    raw = rng.standard_normal(n) * 1e6
    region = [b"r%d" % v for v in rng.integers(0, 4, n)]
    part = build_part(sids, ts, ver, [("calls", O.VT_INT64, calls, None), ("latency", O.VT_FLOAT64, lat, None), ("raw", O.VT_FLOAT64, raw, None)],
                      [("default", [("region", O.VT_STR, region, None)])])
    return part, np.unique(sids)


def _express(bydb, h, usid, n_groups=5):
    groups = (np.arange(usid.size) % n_groups).astype(np.int32)
    return bydb.Query([h], usid, [("calls", O.AGG_SUM), ("latency", O.AGG_SUM), ("calls", O.AGG_COUNT)], series_group=groups, n_groups=n_groups)


def _masked(bydb, h, usid):
    groups = (np.arange(usid.size) % 5).astype(np.int32)
    return bydb.Query([h], usid, [("calls", O.AGG_MIN), ("latency", O.AGG_MAX), ("calls", O.AGG_MEAN)], preds=[bydb.Pred("default", "region", O.OP_EQ, b"r2")],
                      tmin=T0 + 300 * STEP + 1, tmax=T0 + 2500 * STEP, series_group=groups, n_groups=5)


def test_replays_keep_giving_the_plain_calls_answer_and_counters(bydb, gpu_ctx):
    part, usid = _part(np.random.default_rng(31))
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        shapes = [("express", _express(bydb, h, usid), lambda s: s.blocks_express_lane > 0),
                  ("masked", _masked(bydb, h, usid), lambda s: 0 < s.rows_matched < s.rows_scanned and s.blocks_express_lane == 0),
                  ("slow lane", bydb.Query([h], usid, [("raw", O.AGG_MAX), ("raw", O.AGG_SUM)]), lambda s: s.blocks_slow_lane > 0),
                  # series in descending block order within the list: first_block must be written afresh by every replay
                  ("top 3 of 24 groups", bydb.Query([h], usid, [("calls", O.AGG_SUM)], series_group=np.arange(24, dtype=np.int32)[::-1].copy(), n_groups=24, top_n=3),
                   lambda s: s.blocks_scanned > 0)]
        for name, q, reached in shapes:
            want = gpu_ctx.scan_agg(q)
            assert reached(want.stats), name
            g = gpu_ctx.prepare_graph(q)
            try:
                for run in range(12):   # plain path, capture + first replay, ten more replays
                    _assert_same(g.run(), want, (name, run))
            finally:
                g.close()
    finally:
        gpu_ctx.release_part(h)


def test_a_replay_reports_what_it_launched_and_copied(bydb, gpu_ctx):
    part, usid = _part(np.random.default_rng(32))
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        q = _express(bydb, h, usid)
        plain = gpu_ctx.scan_agg(q).stats
        g = gpu_ctx.prepare_graph(q)
        try:
            for _ in range(2):
                g.run()
            s = g.run().stats
        finally:
            g.close()
        # reset + the plain call's kernels; nothing goes up; one copy comes back: the plain call's two (rows, then the 256 B zero page) in one
        assert s.kernel_launches == plain.kernel_launches + 1
        assert s.h2d_bytes == 0 and plain.h2d_bytes > 0
        assert s.d2h_bytes == plain.d2h_bytes and s.d2h_bytes > 256
        assert s.device_ms > 0 and s.scan_kernel_ms == 0
    finally:
        gpu_ctx.release_part(h)


def test_released_and_newly_registered_parts_between_replays(bydb, gpu_ctx):
    rng = np.random.default_rng(33)
    part, usid = _part(rng)
    other, _ = _part(rng, n_series=40, n_pts=500, shift=10_000)
    h = gpu_ctx.register_part(_next_pid(), part.files())
    g = gpu_ctx.prepare_graph(_express(bydb, h, usid))
    try:
        want = gpu_ctx.scan_agg(_express(bydb, h, usid))
        for run in range(4):
            _assert_same(g.run(), want, run)
        # another part comes and goes: the captured step's parts are checked again and still stand
        h2 = gpu_ctx.register_part(_next_pid(), other.files())
        _assert_same(g.run(), want, "after a registration")
        gpu_ctx.release_part(h2)
        _assert_same(g.run(), want, "after a release of another part")
        # its own part goes: the replay fails like the plain call, every time, and the prepared query can still be released
        gpu_ctx.release_part(h)
        for _ in range(2):
            with pytest.raises(bydb.BydbError) as ei:
                g.run()
            assert ei.value.code == bydb.capi.ENOENT
    finally:
        g.close()
    # the same part id registered again with other data: a handle of its own, and a prepared query over it answers for the new data
    h = gpu_ctx.register_part(_pid[0] - 100, other.files())
    try:
        usid2 = np.arange(1, 41, dtype=np.uint64)
        want = gpu_ctx.scan_agg(_express(bydb, h, usid2))
        assert want.val_i64[:, 0].sum() > 10_000 * 500
        g = gpu_ctx.prepare_graph(_express(bydb, h, usid2))
        try:
            for run in range(4):
                _assert_same(g.run(), want, ("new data", run))
        finally:
            g.close()
    finally:
        gpu_ctx.release_part(h)


def test_two_prepared_queries_over_one_part_keep_their_own_state(bydb, gpu_ctx):
    part, usid = _part(np.random.default_rng(34))
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        qa = _express(bydb, h, usid, n_groups=5)
        qb = _express(bydb, h, usid[3:17], n_groups=3)
        qc = _masked(bydb, h, usid[::2])
        wants = [gpu_ctx.scan_agg(q) for q in (qa, qb, qc)]
        gs = [gpu_ctx.prepare_graph(q) for q in (qa, qb, qc)]
        try:
            for rnd in range(6):
                for i, (g, want) in enumerate(zip(gs, wants)):
                    _assert_same(g.run(), want, (rnd, i))
        finally:
            for g in gs:
                g.close()
    finally:
        gpu_ctx.release_part(h)


def test_replays_that_select_nothing(bydb, gpu_ctx):
    part, usid = _part(np.random.default_rng(35))
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        groups = (np.arange(usid.size) % 5).astype(np.int32)
        aggs = [("calls", O.AGG_SUM), ("calls", O.AGG_COUNT)]
        for name, q in (("series the part does not hold", bydb.Query([h], usid + 1000, aggs, series_group=groups, n_groups=5)),
                        ("time range before the part", bydb.Query([h], usid, aggs, tmin=T0 - 100 * STEP, tmax=T0 - STEP)),
                        ("tmin > tmax", bydb.Query([h], usid, aggs, series_group=groups, n_groups=5, tmin=T0 + 10 * STEP, tmax=T0 + 5 * STEP)),
                        ("no series", bydb.Query([h], np.zeros(0, np.uint64), aggs))):
            want = gpu_ctx.scan_agg(q)
            assert want.stats.rows_matched == 0, name
            g = gpu_ctx.prepare_graph(q)
            try:
                for run in range(5):
                    _assert_same(g.run(), want, (name, run))
            finally:
                g.close()
    finally:
        gpu_ctx.release_part(h)

"""-m gpu: every counter of a scan step's zero page comes out the same whichever entry point ran the step.

The entry points share one reader of the read-back zero page: bydb_scan_agg, the prepared graph (run 1 = plain path, run 2 =
capture, runs 3.. = replays), the cold host path (bydb_scan_agg_host) and the prepared collective (bydb_scan_reduce_prepared).
A device error read from a replay must carry the same code and message as the plain call's."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, build_part, grid

pytestmark = pytest.mark.gpu

COUNTERS = ("rows_scanned", "rows_matched", "page_bytes", "blocks_scanned", "blocks_slow_lane", "slow_lane_reasons", "blocks_express_lane")
_pid = [9_000_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def _counters(r):
    return {k: getattr(r.stats, k) for k in COUNTERS}


def _assert_same(got, want, what, float_bits=True):
    assert _counters(got) == _counters(want), what
    assert got.group_id.tolist() == want.group_id.tolist() and got.rows.tolist() == want.rows.tolist(), what
    assert got.val_i64.tolist() == want.val_i64.tolist(), what
    if float_bits:
        assert got.val_f64.view(np.uint64).tolist() == want.val_f64.view(np.uint64).tolist(), what
    else:
        assert np.allclose(got.val_f64, want.val_f64, rtol=1e-12, atol=0), what


def _parts(rng, n_series=24, n_pts=3000):
    """A main part (delta int64, decimal floats, a non-decimal float field that is unpacked into raw-cell pages, a dictionary tag)
    and a second part that rewrites the even series over the same time span with a newer version (the parts overlap)."""
    sids, ts, ver = grid(n_series, n_pts)
    n = sids.size
    calls = rng.integers(-500, 500, n)
    lat = np.round(rng.normal(30, 6, n), 2)
    raw = rng.standard_normal(n) * 1e6
    region = [b"r%d" % v for v in rng.integers(0, 4, n)]
    main = build_part(sids, ts, ver, [("calls", O.VT_INT64, calls, None), ("latency", O.VT_FLOAT64, lat, None), ("raw", O.VT_FLOAT64, raw, None)],
                      [("default", [("region", O.VT_STR, region, None)])])
    m = (sids % 2 == 0) & (rng.random(n) < 0.4)
    newer = build_part(sids[m], ts[m], np.full(m.sum(), 7, np.int64),
                       [("calls", O.VT_INT64, calls[m] + 1000, None), ("latency", O.VT_FLOAT64, lat[m] + 100, None), ("raw", O.VT_FLOAT64, raw[m], None)],
                       [("default", [("region", O.VT_STR, [x for x, k in zip(region, m) if k], None)])])
    return main, newer, np.unique(sids)


def _queries(bydb, h_main, h_newer, usid):
    """(name, query, check on the plain call's stats): each query reaches the lane or path its name says."""
    groups = (np.arange(usid.size) % 5).astype(np.int32)
    return [
        ("express", bydb.Query([h_main], usid, [("calls", O.AGG_SUM), ("latency", O.AGG_SUM), ("calls", O.AGG_COUNT)], series_group=groups, n_groups=5),
         lambda s: s.blocks_express_lane > 0),
        ("masked", bydb.Query([h_main], usid, [("calls", O.AGG_MIN), ("latency", O.AGG_MAX), ("calls", O.AGG_MEAN)],
                              preds=[bydb.Pred("default", "region", O.OP_EQ, b"r2")], tmin=T0 + 300 * STEP + 1, tmax=T0 + 2500 * STEP,
                              series_group=groups, n_groups=5),
         lambda s: 0 < s.rows_matched < s.rows_scanned and s.blocks_express_lane == 0),
        ("slow lane", bydb.Query([h_main], usid, [("raw", O.AGG_MAX), ("raw", O.AGG_SUM)]),
         lambda s: s.blocks_slow_lane > 0 and s.slow_lane_reasons != 0),
        ("overlapping parts", bydb.Query([h_main, h_newer], usid, [("calls", O.AGG_SUM), ("latency", O.AGG_MAX)], series_group=groups, n_groups=5),
         lambda s: s.blocks_scanned > 0),
    ]


def test_prepared_runs_report_the_plain_calls_counters(bydb, gpu_ctx):
    main, newer, usid = _parts(np.random.default_rng(2024))
    h_main = gpu_ctx.register_part(_next_pid(), main.files())
    h_newer = gpu_ctx.register_part(_next_pid(), newer.files())
    try:
        for name, q, reached in _queries(bydb, h_main, h_newer, usid):
            want = gpu_ctx.scan_agg(q)
            assert reached(want.stats), (name, _counters(want))
            g = gpu_ctx.prepare_graph(q)
            try:
                for run in range(5):   # plain path, capture, three replays (overlapping parts: the plain path every time)
                    _assert_same(g.run(), want, (name, run))
            finally:
                g.close()
    finally:
        gpu_ctx.release_part(h_main)
        gpu_ctx.release_part(h_newer)


def test_cold_host_path_reports_the_resident_counters(bydb, gpu_ctx):
    main, newer, usid = _parts(np.random.default_rng(2025))
    files = [{k: np.frombuffer(v, dtype=np.uint8) for k, v in p.files().items()} for p in (main, newer)]
    h_main = gpu_ctx.register_part(_next_pid(), main.files())
    h_newer = gpu_ctx.register_part(_next_pid(), newer.files())
    try:
        for name, q, _ in _queries(bydb, h_main, h_newer, usid):
            want = gpu_ctx.scan_agg(q)
            # the same images as host buffers: one part takes the sliced gather path (its slices are combined, so float sums
            # may round differently), two parts the transient resident path
            q.parts = []
            got = gpu_ctx.scan_agg_host(files if name == "overlapping parts" else files[:1], q)
            _assert_same(got, want, name, float_bits=False)
    finally:
        gpu_ctx.release_part(h_main)
        gpu_ctx.release_part(h_newer)


def test_replayed_device_error_reads_like_the_plain_call(bydb, gpu_ctx):
    # one block, so the block index in the message is the same whichever warp reports first
    sids, ts, ver = grid(1, 500)
    part = build_part(sids, ts, ver, [("calls", O.VT_INT64, np.arange(500), None)], [("default", [("region", O.VT_STR, [b"r1"] * 500, None)])])
    h = gpu_ctx.register_part(_next_pid(), part.files())
    try:
        bad = bydb.Query([h], np.unique(sids), [("calls", O.AGG_SUM)], preds=[bydb.Pred("default", "region", O.OP_EQ, 5)])
        with pytest.raises(bydb.BydbError) as plain:
            gpu_ctx.scan_agg(bad)
        assert plain.value.code == bydb.capi.EINVAL and "#" in plain.value.msg
        g = gpu_ctx.prepare_graph(bad)
        try:
            for run in range(5):
                with pytest.raises(bydb.BydbError) as ei:
                    g.run()
                assert (ei.value.code, ei.value.msg) == (plain.value.code, plain.value.msg), run
        finally:
            g.close()
    finally:
        gpu_ctx.release_part(h)


def test_prepared_collective_reports_the_plain_collectives_counters(bydb):
    # bydb_scan_reduce_prepared against bydb_scan_reduce, rank by rank, on whatever devices are present.  With one GPU the two
    # ranks share it, and the prepared collective then always takes the plain path: only a box with two or more GPUs replays graphs.
    import gc
    import threading
    import torch
    n_dev = torch.cuda.device_count()
    rng = np.random.default_rng(2026)
    R = 2
    sids, ts, ver = grid(24, 3000)
    usid = np.unique(sids)
    shard_of = (np.arange(usid.size) * R) // usid.size
    calls = rng.integers(-500, 500, sids.size)
    region = [b"r%d" % v for v in rng.integers(0, 4, sids.size)]
    shards = []
    for r in range(R):
        m = np.isin(sids, usid[shard_of == r])
        shards.append(build_part(sids[m], ts[m], ver[m], [("calls", O.VT_INT64, calls[m], None)],
                                 [("default", [("region", O.VT_STR, [x for x, k in zip(region, m) if k], None)])]))
    gc.collect()
    gc.disable()   # no finaliser may free page-locked memory on a rank's thread in the middle of a collective (see test_gpu_parity)
    ctxs = [bydb.Context(device=r % n_dev) for r in range(R)]
    try:
        handles = [c.comm_export(1 << 20, R) for c in ctxs]
        for r, c in enumerate(ctxs):
            c.comm_connect(r, R, handles)
        hs = [c.register_part(1, p.files()) for c, p in zip(ctxs, shards)]
        groups = (np.arange(usid.size) % 3).astype(np.int32)
        for kw in (dict(aggs=[("calls", O.AGG_SUM), ("calls", O.AGG_COUNT)]),
                   dict(aggs=[("calls", O.AGG_MAX)], preds=[bydb.Pred("default", "region", O.OP_NE, b"r1")], tmin=T0 + 100 * STEP, tmax=T0 + 2000 * STEP)):
            qs = [bydb.Query([hs[r]], usid[shard_of == r], series_group=groups[shard_of == r], n_groups=3, **kw) for r in range(R)]

            def collective(call):
                got, errs = [None] * R, []

                def run(r):
                    try:
                        got[r] = call(r)
                    except Exception as e:  # noqa: BLE001
                        errs.append(repr(e))
                th = [threading.Thread(target=run, args=(r,)) for r in range(R)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                assert not errs, errs
                return got

            want = collective(lambda r: ctxs[r].scan_reduce(qs[r], root=0))
            assert all(w.stats.blocks_scanned > 0 for w in want)
            gqs = [ctxs[r].prepare_graph(qs[r]) for r in range(R)]
            try:
                for run in range(5):   # run 1 plain, then one capture per slot parity, then replays
                    got = collective(lambda r: gqs[r].run_reduce(root=0))
                    for r in range(R):
                        _assert_same(got[r], want[r], (kw["aggs"], run, r))
            finally:
                for gq in gqs:
                    gq.close()
    finally:
        for c in ctxs:
            c.close()
        gc.enable()

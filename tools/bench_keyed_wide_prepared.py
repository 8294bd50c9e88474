#!/usr/bin/env python
"""bench_keyed_wide_prepared.py -- a wide group-by on a stored tag, unprepared (bydb_scan_agg_keyed_wide) against prepared
(bydb_query_prepare_keyed_wide + bydb_scan_agg_keyed_prepared, one captured graph per step), on one GPU.

Shapes:
  - dashboard_1000 / dashboard_4096: 300 series x 1440 points (a day at one point a minute), sum(latency), count(calls),
    max(calls) per (10 series groups, key) on an int64 tag with up to 1,000 / 4,096 values (at most 206 per block): the step an
    interactive panel refresh pays, where the unprepared call's host sequence (memsets, stream-ordered allocations, four
    synchronised read-backs) is a large share of it;
  - bench: bench.py's part -- its series, points, seed, region tag and latency field, without the three fields the query does not
    read -- 10 000 series x 100 000 points (1e9 datapoints), sum + count of latency GROUP BY region: the scan dominates the step.

Each shape is warmed up on both forms (the prepared handle captures on its second run), then timed over --steps steps that
alternate the two forms, each step timed with the wall clock around a call that ends in a device synchronise; the medians and
the spread (min, max) are reported.  The answers of the two forms are compared field by field (rows, series groups, key bytes,
values as bit patterns, scan counters).  Prints one JSON line per shape, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_keyed_prepared import COUNTERS, SEED, STEP, T0, card, stats_of  # noqa: E402


def identical(a, b):
    return (a.key == b.key and a.n_keys == b.n_keys and a.group_id.tolist() == b.group_id.tolist() and a.rows.tolist() == b.rows.tolist()
            and a.is_float.tolist() == b.is_float.tolist() and a.val_i64.tolist() == b.val_i64.tolist()
            and a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist()
            and all(getattr(a.stats, k) == getattr(b.stats, k) for k in COUNTERS))


def dashboard_part(S, capi, n_series, n_points, V):
    n = n_series * n_points
    sid = np.repeat(np.arange(1, n_series + 1, dtype=np.uint64), n_points)
    r = np.tile(np.arange(n_points, dtype=np.int64), n_series)
    rng = np.random.default_rng(11)
    lat = rng.integers(500, 9000, n)   # latency in hundredths: a decimal column of 2 digits
    calls = rng.integers(0, 1000, n)
    key = ((sid.astype(np.int64) * 97 + r // 7) % V).astype(np.int64)
    return S.write_part(sid, T0 + r * STEP, np.ones(n, np.int64), [("latency", capi.VT_FLOAT64, lat, 2), ("calls", capi.VT_INT64, calls)],
                        tag_family="default", tags=[("key", capi.VT_INT64, key)]), n


def timed(ctx, q, tag, cap, vt, steps, warmup):
    g = ctx.prepare_keyed_wide(q, "default", tag, cap, vt)
    try:
        for _ in range(max(warmup, 3)):   # the handle's unprepared run, its capture, then replays
            plain, prep = ctx.scan_agg_keyed_wide(q, "default", tag, cap, vt), g.run()
        t_plain, t_prep, same = [], [], True
        for _ in range(steps):
            t = time.perf_counter()
            plain = ctx.scan_agg_keyed_wide(q, "default", tag, cap, vt)
            t_plain.append((time.perf_counter() - t) * 1e3)
            t = time.perf_counter()
            prep = g.run()
            t_prep.append((time.perf_counter() - t) * 1e3)
            same = same and identical(plain, prep)
    finally:
        g.release()
    mp, mq = statistics.median(t_plain), statistics.median(t_prep)
    return {"n_keys": plain.n_keys, "rows_out": int(plain.group_id.size), "steps": steps,
            "plain_ms_per_step": round(mp, 4), "plain_ms_min_max": [round(min(t_plain), 4), round(max(t_plain), 4)],
            "prepared_ms_per_step": round(mq, 4), "prepared_ms_min_max": [round(min(t_prep), 4), round(max(t_prep), 4)],
            "speedup": round(mp / mq, 3), "plain": stats_of(plain), "prepared": stats_of(prep), "identical": bool(same)}, plain


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bench-series", type=int, default=10_000)
    ap.add_argument("--bench-points", type=int, default=100_000)
    ap.add_argument("--dash-series", type=int, default=300)
    ap.add_argument("--dash-points", type=int, default=1440)
    args = ap.parse_args()
    if args.steps < 20:
        raise SystemExit("--steps must be >= 20 (medians of at least 20 steps)")
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import capi, synth as S
    gpu = card()
    timing = "median wall ms of synchronised calls, unprepared and prepared alternating"
    with pkg.Context(device=0) as ctx:
        for pid, V in ((1, 1000), (2, 4096)):
            part, n = dashboard_part(S, capi, args.dash_series, args.dash_points, V)
            h = ctx.register_part(pid, part.files())
            try:
                sids = np.arange(1, args.dash_series + 1, dtype=np.uint64)
                q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("calls", pkg.AGG_COUNT), ("calls", pkg.AGG_MAX)],
                              series_group=((sids - 1) % 10).astype(np.int32), n_groups=10)
                res, plain = timed(ctx, q, "key", V, pkg.VT_INT64, args.steps, args.warmup)
                res["identical"] = res["identical"] and int(plain.val_i64[:, 1].sum()) == n
            finally:
                ctx.release_part(h)
            print(json.dumps({"shape": f"dashboard_{V}", "datapoints": n, **res, "gpu": gpu[0], "power_limit": gpu[1], "timing": timing}), flush=True)
        part = S.synth_part(args.bench_series, args.bench_points, [("latency", S.F_LATENCY)], sid0=1, sid_step=1, t0=T0, t_step=STEP,
                            region_values=8, region_run=16, seed=SEED)
        n, _ = part.counts()
        h = ctx.register_part(3, part.files())
        try:
            q = pkg.Query(parts=[h], series_ids=np.arange(1, args.bench_series + 1, dtype=np.uint64),
                          aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)])
            res, plain = timed(ctx, q, "region", 0, 0, args.steps, args.warmup)
            res["identical"] = res["identical"] and int(plain.rows.sum()) == int(n)
        finally:
            ctx.release_part(h)
        print(json.dumps({"shape": "bench", "datapoints": int(n), **res, "gpu": gpu[0], "power_limit": gpu[1], "timing": timing}), flush=True)


if __name__ == "__main__":
    main()

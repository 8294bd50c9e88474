#!/usr/bin/env python
"""bench_keys_wide_prepared.py -- a group-by on a tuple of stored tags, unprepared (bydb_scan_agg_keys_wide) against prepared
(bydb_query_prepare_keys_wide + bydb_scan_agg_keys_prepared, one captured graph per step), on one GPU.

Shapes: the dashboard part of bench_keyed_wide_prepared.py -- 300 series x 1440 points (a day at one point a minute),
sum(latency), count(calls), max(calls) per (10 series groups, tuple) -- grouped by a (string endpoint, int64 status code) tuple of
about 1,000 (dashboard_1000: 100 endpoints x 10 codes) and 4,096 (dashboard_4096: 256 x 16) tuples, at most 206 per block.  This is
the step an interactive panel grouped by two tags pays on every refresh, where the unprepared call's host sequence (K + 1 discovery
tables, memsets, stream-ordered allocations, synchronised read-backs) is a large share of it.

Each shape is warmed up on both forms (the prepared handle captures on its second run), then timed over --steps steps that
alternate the two forms, each step timed with the wall clock around a call that ends in a device synchronise; the medians and the
spread (min, max) are reported.  The answers of the two forms are compared field by field (rows, series groups, each tag's key
bytes, values as bit patterns, n_tuples, each tag's value count, scan counters).  Prints one JSON line per shape, with the card's
name and power limit read in the same run.
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

from bench_keyed_prepared import COUNTERS, STEP, T0, card, stats_of  # noqa: E402


def identical(a, b):
    return (a.key == b.key and a.n_tuples == b.n_tuples and [len(t) for t in a.key_tables] == [len(t) for t in b.key_tables]
            and a.group_id.tolist() == b.group_id.tolist() and a.rows.tolist() == b.rows.tolist()
            and a.is_float.tolist() == b.is_float.tolist() and a.val_i64.tolist() == b.val_i64.tolist()
            and a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist()
            and all(getattr(a.stats, k) == getattr(b.stats, k) for k in COUNTERS))


def dashboard_part(S, capi, n_series, n_points, n_endpoints, n_codes):
    """tuple u = (sid * 97 + r // 7) mod (n_endpoints * n_codes) of row r: endpoint u // n_codes, status code 200 + u % n_codes"""
    n = n_series * n_points
    sid = np.repeat(np.arange(1, n_series + 1, dtype=np.uint64), n_points)
    r = np.tile(np.arange(n_points, dtype=np.int64), n_series)
    rng = np.random.default_rng(11)
    lat = rng.integers(500, 9000, n)   # latency in hundredths: a decimal column of 2 digits
    calls = rng.integers(0, 1000, n)
    u = (sid.astype(np.int64) * 97 + r // 7) % (n_endpoints * n_codes)
    endpoints = [b"/api/v1/endpoint-%03d" % e for e in range(n_endpoints)]
    tags = [("endpoint", capi.VT_STR, (u // n_codes).astype(np.uint32), endpoints), ("code", capi.VT_INT64, 200 + u % n_codes)]
    return S.write_part(sid, T0 + r * STEP, np.ones(n, np.int64), [("latency", capi.VT_FLOAT64, lat, 2), ("calls", capi.VT_INT64, calls)],
                        tag_family="default", tags=tags), n


def timed(ctx, q, keys, cap, steps, warmup):
    g = ctx.prepare_keys_wide(q, keys, cap)
    try:
        for _ in range(max(warmup, 3)):   # the handle's unprepared run, its capture, then replays
            plain, prep = ctx.scan_agg_keys_wide(q, keys, cap), g.run()
        t_plain, t_prep, same = [], [], True
        for _ in range(steps):
            t = time.perf_counter()
            plain = ctx.scan_agg_keys_wide(q, keys, cap)
            t_plain.append((time.perf_counter() - t) * 1e3)
            t = time.perf_counter()
            prep = g.run()
            t_prep.append((time.perf_counter() - t) * 1e3)
            same = same and identical(plain, prep)
    finally:
        g.release()
    mp, mq = statistics.median(t_plain), statistics.median(t_prep)
    return {"n_tuples": plain.n_tuples, "tag_values": [len(t) for t in plain.key_tables], "rows_out": int(plain.group_id.size),
            "steps": steps, "plain_ms_per_step": round(mp, 4), "plain_ms_min_max": [round(min(t_plain), 4), round(max(t_plain), 4)],
            "prepared_ms_per_step": round(mq, 4), "prepared_ms_min_max": [round(min(t_prep), 4), round(max(t_prep), 4)],
            "speedup": round(mp / mq, 3), "plain": stats_of(plain), "prepared": stats_of(prep), "identical": bool(same)}, plain


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
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
    keys = [("default", "endpoint", pkg.VT_STR), ("default", "code", pkg.VT_INT64)]
    with pkg.Context(device=0) as ctx:
        for pid, (n_endpoints, n_codes) in ((1, (100, 10)), (2, (256, 16))):
            T = n_endpoints * n_codes
            part, n = dashboard_part(S, capi, args.dash_series, args.dash_points, n_endpoints, n_codes)
            h = ctx.register_part(pid, part.files())
            try:
                sids = np.arange(1, args.dash_series + 1, dtype=np.uint64)
                q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("calls", pkg.AGG_COUNT), ("calls", pkg.AGG_MAX)],
                              series_group=((sids - 1) % 10).astype(np.int32), n_groups=10)
                res, plain = timed(ctx, q, keys, T, args.steps, args.warmup)
                res["identical"] = res["identical"] and int(plain.val_i64[:, 1].sum()) == n
            finally:
                ctx.release_part(h)
            print(json.dumps({"shape": f"dashboard_{T}", "datapoints": n, **res, "gpu": gpu[0], "power_limit": gpu[1], "timing": timing}), flush=True)


if __name__ == "__main__":
    main()

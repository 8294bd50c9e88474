#!/usr/bin/env python
"""bench_keyed_prepared.py -- a group-by on a stored tag, plain (bydb_scan_agg_keyed) against prepared
(bydb_query_prepare_keyed + bydb_scan_agg_keyed_prepared, one captured graph per step), on one GPU.

Query: sum(latency), count(latency) GROUP BY region (the synthetic parts' dictionary tag, 8 values: 8 scan passes), over two
shapes of part:
  - bench: bench.py's part -- its series, points, seed, region tag and latency field, without the three fields the query does not
    read -- 10 000 series x 100 000 points (1e9 datapoints): the scan dominates the step;
  - dashboard: 300 series x 1440 points (a day at one point a minute): the step an interactive panel refresh pays, where the
    plain call's host sequence (discovery, a synchronised round trip per pass, ordering, two read-backs) is most of it.

Each shape is warmed up on both forms (the prepared handle captures on its second run), then timed over --steps steps that
alternate the two forms, each step timed with the wall clock around a call that ends in a device synchronise (the call returns
its result on the host); the medians are reported.  The answers of the two forms are compared field by field (rows, keys, values
as bit patterns, scan counters).  Prints one JSON line per shape, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

T0 = 1_700_000_000_000_000_000
STEP = 60_000_000_000
SEED = 0xB200   # bench.py's
COUNTERS = ("rows_scanned", "rows_matched", "page_bytes", "blocks_scanned", "blocks_slow_lane", "slow_lane_reasons", "blocks_express_lane")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=60)
    if out.returncode != 0:
        raise SystemExit("nvidia-smi failed: " + out.stderr)
    name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
    return name, power


def identical(a, b):
    return (a.key == b.key and a.n_keys == b.n_keys and a.group_id.tolist() == b.group_id.tolist() and a.rows.tolist() == b.rows.tolist()
            and a.is_float.tolist() == b.is_float.tolist() and a.val_i64.tolist() == b.val_i64.tolist()
            and a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist()
            and all(getattr(a.stats, k) == getattr(b.stats, k) for k in COUNTERS))


def stats_of(r):
    s = r.stats
    return {"kernel_launches": int(s.kernel_launches), "device_ms": round(s.device_ms, 4), "h2d_bytes": int(s.h2d_bytes),
            "d2h_bytes": int(s.d2h_bytes)}


def shape(pkg, ctx, part_id, name, n_series, n_points, steps, warmup, gpu):
    from bydb_b200 import synth as S
    part = S.synth_part(n_series, n_points, [("latency", S.F_LATENCY)], sid0=1, sid_step=1, t0=T0, t_step=STEP, region_values=8,
                        region_run=16, seed=SEED)
    n_rows, _ = part.counts()
    h = ctx.register_part(part_id, part.files())
    try:
        q = pkg.Query(parts=[h], series_ids=np.arange(1, n_series + 1, dtype=np.uint64), aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)])
        g = ctx.prepare_keyed(q, "default", "region")
        try:
            for _ in range(max(warmup, 3)):   # the handle's plain run, its capture, then replays
                plain, prep = ctx.scan_agg_keyed(q, "default", "region"), g.run()
            t_plain, t_prep, same = [], [], True
            for _ in range(steps):
                t = time.perf_counter()
                plain = ctx.scan_agg_keyed(q, "default", "region")
                t_plain.append((time.perf_counter() - t) * 1e3)
                t = time.perf_counter()
                prep = g.run()
                t_prep.append((time.perf_counter() - t) * 1e3)
                same = same and identical(plain, prep)
        finally:
            g.release()
    finally:
        ctx.release_part(h)
    mp, mq = statistics.median(t_plain), statistics.median(t_prep)
    return {"shape": name, "datapoints": int(n_rows), "series": n_series, "points": n_points, "n_keys": plain.n_keys, "steps": steps,
            "plain_ms_per_step": round(mp, 4), "prepared_ms_per_step": round(mq, 4), "speedup": round(mp / mq, 3),
            "plain_ms_outside_device": round(mp - plain.stats.device_ms, 4),
            "plain": stats_of(plain), "prepared": stats_of(prep), "identical": bool(same and int(prep.rows.sum()) == int(n_rows)),
            "gpu": gpu[0], "power_limit": gpu[1], "timing": "median wall ms of synchronised calls, plain and prepared alternating"}


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
    gpu = card()
    with pkg.Context(device=0) as ctx:
        for pid, (name, ns, npts) in enumerate((("dashboard", args.dash_series, args.dash_points), ("bench", args.bench_series, args.bench_points)), 1):
            print(json.dumps(shape(pkg, ctx, pid, name, ns, npts, args.steps, args.warmup, gpu)), flush=True)


if __name__ == "__main__":
    main()

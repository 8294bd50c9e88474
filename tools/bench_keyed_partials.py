#!/usr/bin/env python
"""bench_keyed_partials.py -- the map-phase rows of a stored-tag group-by (bydb_scan_partials_keyed) against the finalised keyed
call (bydb_scan_agg_keyed) on one GPU.

Part: bench.py's part (10,000 series x 100,000 points = 1e9 datapoints by default, region tag of 8 values).  Query: sum(latency),
count(latency) by (series group of bench.py's 1000 services, region).  The two calls are timed in --rounds rounds alternated in one
process, --steps calls each, with the wall clock around calls that end in a device synchronise (both return their rows on the
host); the JSON line gives each call's median and spread in ms per call, the d2h_bytes of each next to the size of the composite
table (which the partial form never copies), and a check that Val() of the partial rows equals the finalised values.  With
--profile (a separate run under torch.profiler, after the timing) it adds the device time of keyed_partial_rows_kernel and of
the other kernels per call.  The card's name and power limit are read in the same run.
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

import bench  # noqa: E402  (make_part, T0, STEP: the bench's own part)


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=60)
    if out.returncode != 0:
        raise SystemExit("nvidia-smi failed: " + out.stderr)
    name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
    return name, power


def kernel_ms(fn, calls):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0)
        name = e.key.split("(")[0].replace("void ", "").replace("bydb::", "")
        if us and "kernel" in name:
            out[name] = round(out.get(name, 0.0) + us / 1e3 / calls, 4)
    if "keyed_partial_rows_kernel" not in out:
        raise SystemExit("torch.profiler did not record keyed_partial_rows_kernel")
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--services", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", type=int, default=0, help="calls of the partial form under torch.profiler after the timing (0 = none)")
    args = ap.parse_args()
    import __graft_entry__ as ge
    pkg = ge.load_package()
    part = bench.make_part(pkg, args.series, args.points, 1)
    n_rows, _ = part.counts()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    groups = ((sids - 1) % args.services).astype(np.int32)
    q = pkg.Query(parts=[], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)], series_group=groups,
                  n_groups=args.services)
    out = {"datapoints": int(n_rows), "series": args.series, "groups": args.services, "steps": args.steps, "rounds": args.rounds}
    with pkg.Context(device=0) as ctx:
        q.parts = [ctx.register_part(1, part.files())]
        legs = {"scan_agg_keyed": lambda: ctx.scan_agg_keyed(q, "default", "region"),
                "scan_partials_keyed": lambda: ctx.scan_partials_keyed(q, "default", "region")}
        for fn in legs.values():
            for _ in range(args.warmup):
                fn()
        times = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                t = time.perf_counter()
                for _ in range(args.steps):
                    r = fn()
                times[k].append((time.perf_counter() - t) * 1e3 / args.steps)
        fin, rows = legs["scan_agg_keyed"](), legs["scan_partials_keyed"]()
        assert list(zip(fin.group_id.tolist(), fin.key)) == list(zip(rows["group_id"].tolist(), rows["key"])), "row order"
        assert (fin.val_f64[:, 0] == rows["val_f64"][:, 0]).all() and (fin.val_i64[:, 1] == rows["val_f64"][:, 1]).all(), "values"
        assert int(fin.rows.sum()) == n_rows, "every row in a group"
        V, G = rows["n_keys"], args.services
        for k in legs:
            st = fin.stats if k == "scan_agg_keyed" else rows["stats"]
            out[k] = {"ms_per_call_median": round(statistics.median(times[k]), 3), "ms_per_call_rounds": [round(x, 3) for x in times[k]],
                      "d2h_bytes": int(st.d2h_bytes), "kernel_launches": int(st.kernel_launches), "rows_out": int(len(rows["key"]))}
        out["composite_table_bytes"] = 8 * (G * V * (7 * 1 + 1) + 1)
        out["n_keys"] = V
        if args.profile:
            out["kernels_ms_per_call_partials"] = kernel_ms(legs["scan_partials_keyed"], args.profile)
        ctx.release_part(q.parts[0])
    name, power = card()
    out.update(gpu=name, power_limit=power, checked="same (group, key) order; SUM and COUNT partials equal the finalised values")
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_partials_prepared.py -- a data node's partial answer, unprepared against prepared, on one GPU.

In a cluster the liaison pushes every aggregation down with agg_return_partial, and each data node answers with map-phase rows:
  - plain: sum(latency), count(latency) GROUP BY service (1000 series groups, bench.py's grouping): bydb_scan_partials into a
    device table + bydb_partials_rows, against bydb_scan_partials_prepared;
  - keyed: the same GROUP BY service, region (the synthetic parts' dictionary tag, 8 values: 8 scan passes):
    bydb_scan_partials_keyed, against bydb_scan_partials_keyed_prepared.
Two shapes of part, as tools/bench_keyed_prepared.py:
  - dashboard: 300 series x 1440 points (a day at one point a minute), where the unprepared call's host sequence is most of a step;
  - bench: bench.py's part without the fields the query does not read, 10 000 series x 100 000 points (1e9 datapoints).
Each shape is warmed up on every form (a prepared handle captures on its second run), then timed over --steps steps alternating
unprepared and prepared calls, each call timed with the wall clock around a call that ends in a device synchronise; medians are
reported, with each form's d2h_bytes and kernel_launches.  bydb_partials_rows alone over the bench shape's filled table is timed
the same way.  The two forms' answers are compared array by array (floats as bit patterns) and counter by counter.  Prints one
JSON line per shape, with the card's name and power limit read in the same run.
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
SERVICES = 1000
COUNTERS = ("rows_scanned", "rows_matched", "page_bytes", "blocks_scanned", "blocks_slow_lane", "slow_lane_reasons", "blocks_express_lane")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=60)
    if out.returncode != 0:
        raise SystemExit("nvidia-smi failed: " + out.stderr)
    name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
    return name, power


def identical(a, b):
    keys = ("group_id", "is_float", "val_i64", "cnt_i64") + (("key", "n_keys") if "key" in a else ())
    return (all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in keys)
            and all(a[k].view(np.uint64).tolist() == b[k].view(np.uint64).tolist() for k in ("val_f64", "cnt_f64"))
            and all(getattr(a["stats"], k) == getattr(b["stats"], k) for k in COUNTERS))


def timed(call):
    t = time.perf_counter()
    r = call()
    return (time.perf_counter() - t) * 1e3, r


def stats_of(s):
    return {"kernel_launches": int(s.kernel_launches), "device_ms": round(s.device_ms, 4), "h2d_bytes": int(s.h2d_bytes),
            "d2h_bytes": int(s.d2h_bytes)}


def shape(pkg, ctx, part_id, name, n_series, n_points, steps, warmup, gpu):
    import torch
    from bydb_b200 import synth as S
    part = S.synth_part(n_series, n_points, [("latency", S.F_LATENCY)], sid0=1, sid_step=1, t0=T0, t_step=STEP, region_values=8,
                        region_run=16, seed=SEED)
    n_rows, _ = part.counts()
    h = ctx.register_part(part_id, part.files())
    sids = np.arange(1, n_series + 1, dtype=np.uint64)
    q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)],
                  series_group=((sids - 1) % SERVICES).astype(np.int32), n_groups=SERVICES)
    nb = ctx.partials_layout(q)["total_bytes"]
    table = torch.zeros(nb // 8, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def unprepared_plain():
        st = ctx.scan_partials(q, table.data_ptr(), nb, stream)
        out = dict(ctx.partials_rows(q, table.data_ptr(), nb, stream))
        out["stats"] = st
        return out

    def unprepared_keyed():
        return ctx.scan_partials_keyed(q, "default", "region")

    out = {"shape": name, "datapoints": int(n_rows), "series": n_series, "points": n_points, "groups": SERVICES, "steps": steps,
           "gpu": gpu[0], "power_limit": gpu[1], "timing": "median wall ms of synchronised calls, unprepared and prepared alternating"}
    try:
        g, kg = ctx.prepare_graph(q), ctx.prepare_keyed(q, "default", "region")
        try:
            for form, plain_call, prep_call in (("plain", unprepared_plain, g.run_partials), ("keyed", unprepared_keyed, kg.run_partials)):
                for _ in range(max(warmup, 3)):   # the handle's unprepared run, its capture, then replays
                    plain_call(), prep_call()
                t_plain, t_prep, same = [], [], True
                for _ in range(steps):
                    dt, a = timed(plain_call)
                    t_plain.append(dt)
                    dt, b = timed(prep_call)
                    t_prep.append(dt)
                    same = same and identical(a, b)
                mp, mq = statistics.median(t_plain), statistics.median(t_prep)
                # the plain form's unprepared stats are bydb_scan_partials' alone: bydb_partials_rows reports none
                out[form] = {"unprepared_ms": round(mp, 4), "prepared_ms": round(mq, 4), "speedup": round(mp / mq, 3),
                             "rows": int(len(b["group_id"])), "n_keys": int(b.get("n_keys", 0)), "identical": bool(same),
                             "unprepared": stats_of(a["stats"]), "prepared": stats_of(b["stats"])}
            unprepared_plain()   # the table holds this shape's partials
            t_rows = [timed(lambda: ctx.partials_rows(q, table.data_ptr(), nb, stream))[0] for _ in range(steps)]
            out["partials_rows_ms"] = round(statistics.median(t_rows), 4)
        finally:
            g.close()
            kg.release()
    finally:
        ctx.release_part(h)
    return out


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

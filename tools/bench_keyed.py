#!/usr/bin/env python
"""bench_keyed.py -- group-by on a stored tag (bydb_scan_agg_keyed) on one GPU: the int64 key against the string key.

Part: the C5 shape (SURVEY.md 8d) -- 4 int64 fields (delta, small fluctuations, random < 100, counter) and 4 float64 fields
(latency, walk, integers, uniform), a region dictionary tag, the int64 tag "code" (6 values) and the string tag "zone"
(5 values) -- at 1e8 datapoints by default.  Query: sum(latency), count(latency), max(delta) grouped by (series group of 100
services, key), keyed once on "code" (value_type BYDB_VT_INT64, 6 passes) and once on "zone" (5 passes).

Each leg is warmed up, then timed over --steps calls with the wall clock around calls that end in a device synchronise
(the call returns its result on the host).  Checks: both answers hold every row of the selected series, and each key value's
rows and aggregates equal a plain bydb_scan_agg with the predicate "tag == value".  Prints one JSON line with the card's name
and power limit read in the same run, and (after the timing, profiler on) the device time per call of each kernel of the
keyed call, so key discovery can be told from the per-value scan passes.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

T0 = 1_700_000_000_000_000_000
STEP = 60_000_000_000
SERVICES = 100


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=60)
    if out.returncode != 0:
        raise SystemExit("nvidia-smi failed: " + out.stderr)
    name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
    return name, power


def kernel_ms(ctx, q, tag, vt, calls):
    """device time per call of each kernel of the keyed call, from torch.profiler (CUDA activity) over `calls` calls made after
    the timed ones: key discovery next to the per-value scan passes"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.scan_agg_keyed(q, "default", tag, 0, vt)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0)
        name = e.key.split("(")[0].replace("void ", "").replace("bydb::", "")
        if us and "kernel" in name:
            out[name] = round(out.get(name, 0.0) + us / 1e3 / calls, 3)
    if not out:
        raise SystemExit("torch.profiler recorded no kernel of the keyed call")
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-calls", type=int, default=3, help="calls per leg under torch.profiler after the timing (0 = none)")
    args = ap.parse_args()
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import synth as S
    fields = [("delta", S.I_DELTA), ("fluct", S.I_FLUCT), ("rand", S.I_RANDOM100), ("counter", S.I_COUNTER),
              ("latency", S.F_LATENCY), ("walk", S.F_WALK3), ("ints", S.F_INT1000), ("uniform", S.F_UNIFORM)]
    part = S.synth_part(args.series, args.points, fields, t0=T0, t_step=STEP, region_values=8, region_run=16, code_tag=True, zone_tag=True)
    n_rows, _ = part.counts()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    groups = ((sids - 1) % SERVICES).astype(np.int32)
    aggs = [("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)]
    legs = {"code": (pkg.VT_INT64, lambda k: int.from_bytes(k, "little", signed=True)), "zone": (0, bytes)}
    out = {"datapoints": int(n_rows), "series": args.series, "steps": args.steps}
    with pkg.Context(device=0) as ctx:
        h = ctx.register_part(1, part.files())
        q = pkg.Query(parts=[h], series_ids=sids, aggs=aggs, series_group=groups, n_groups=SERVICES)
        for tag, (vt, lit) in legs.items():
            for _ in range(args.warmup):
                r = ctx.scan_agg_keyed(q, "default", tag, 0, vt)
            t = time.perf_counter()
            for _ in range(args.steps):
                r = ctx.scan_agg_keyed(q, "default", tag, 0, vt)
            ms = (time.perf_counter() - t) * 1e3 / args.steps
            assert int(r.rows.sum()) == n_rows, f"{tag}: {int(r.rows.sum())} rows of {n_rows}"
            keys = r.key
            # the keyed pass of the int64 key 0 matches nil cells too (kOpEqOrNil); OP_EQ 0 is the same predicate here only
            # because the synthetic tags hold no nil cell
            for k in sorted(set(keys)):
                p = ctx.scan_agg(pkg.Query(parts=[h], series_ids=sids, aggs=aggs, series_group=groups, n_groups=SERVICES,
                                           preds=[pkg.Pred("default", tag, pkg.OP_EQ, lit(k))]))
                sel = np.array([x == k for x in keys])
                assert r.group_id[sel].tolist() == p.group_id.tolist() and r.rows[sel].tolist() == p.rows.tolist(), tag
                assert (r.val_i64[sel] == p.val_i64).all() and (r.val_f64[sel][:, 2] == p.val_f64[:, 2]).all(), tag
                assert np.allclose(r.val_f64[sel][:, 0], p.val_f64[:, 0], rtol=1e-9, atol=0), tag
            out[tag] = {"ms_per_call": round(ms, 3), "n_keys": r.n_keys, "passes": r.n_keys, "rows_out": int(r.rows.size),
                        "datapoints_per_s": round(n_rows / (ms / 1e3)), "passes_scan_kernel_ms": round(r.stats.scan_kernel_ms, 3),
                        "passes_device_ms": round(r.stats.device_ms, 3), "blocks_slow_lane": r.stats.blocks_slow_lane,
                        "blocks_scanned": r.stats.blocks_scanned}
        if args.profile_calls:
            out["kernels_ms_per_call"] = {tag: kernel_ms(ctx, q, tag, vt, args.profile_calls) for tag, (vt, _) in legs.items()}
        ctx.release_part(h)
    name, power = card()
    out.update(gpu=name, power_limit=power, checked="rows and per-value predicate scans agree")
    print(json.dumps(out))


if __name__ == "__main__":
    main()

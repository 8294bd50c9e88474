#!/usr/bin/env python
"""bench_keyed_wide.py -- group-by on a stored tag in one scan pass (bydb_scan_agg_keyed_wide) against the per-value passes of
bydb_scan_agg_keyed, on one GPU, in one process.

Legs (each: warm-up, then --steps rounds that time one narrow call and one wide call back to back, wall clock around calls that
end in a device synchronise):
  - bench:  the 1e9-datapoint part of bench.py (10,000 series x 100,000 points), sum + count of latency GROUP BY region (8 values);
  - c5:     the C5-shaped part of bench_keyed.py (1e8 datapoints), sum(latency), count(latency), max(delta) per (100 services,
            key), keyed on the int64 tag code (6 values) and on the string tag zone (5 values);
  - wide:   a part written with synth.write_part (2,000 series x 10,000 points) carrying the int64 tag wide (4,096 values, at
            most 249 per block; the wide call only: the passes take at most 256 values) and the tags one and two (1 and 2 values,
            both calls, for the small-V end).
Checks, wherever both calls run: the same rows in the same order, the same keys, equal int64 values, floats within 1e-9.  For the
4,096-value leg: every row of the selected series is accounted for and n_keys = 4,096.  After the timing, torch.profiler (CUDA
activity) gives the device time per call of every kernel of the wide call.  Prints one JSON line with the card's name and power
limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_keyed import card  # noqa: E402

T0 = 1_700_000_000_000_000_000
STEP = 60_000_000_000


def same(n, w, label):
    assert n.group_id.tolist() == w.group_id.tolist() and n.key == w.key and n.rows.tolist() == w.rows.tolist(), f"{label}: rows"
    assert (n.val_i64 == w.val_i64).all(), f"{label}: int64 values"
    a, b = n.val_f64, w.val_f64
    assert ((a.view(np.uint64) == b.view(np.uint64)) | np.isclose(a, b, rtol=1e-9, atol=0)).all(), f"{label}: float values"


def alternate(ctx, q, tag, vt, cap, steps, warmup, narrow=True):
    """-> (narrow ms per call or None, wide ms per call, last wide result)"""
    calls = [("wide", lambda: ctx.scan_agg_keyed_wide(q, "default", tag, cap, vt))]
    if narrow:
        calls.insert(0, ("narrow", lambda: ctx.scan_agg_keyed(q, "default", tag, min(cap, 256), vt)))
    last = {}
    for _ in range(warmup):
        for name, fn in calls:
            last[name] = fn()
    spent = {name: 0.0 for name, _ in calls}
    for _ in range(steps):
        for name, fn in calls:
            t = time.perf_counter()
            last[name] = fn()
            spent[name] += time.perf_counter() - t
    if narrow:
        same(last["narrow"], last["wide"], tag)
    ms = {name: round(s * 1e3 / steps, 3) for name, s in spent.items()}
    return ms.get("narrow"), ms["wide"], last["wide"]


def leg(ctx, q, tag, vt, cap, n_rows, args, narrow=True):
    n_ms, w_ms, r = alternate(ctx, q, tag, vt, cap, args.steps, args.warmup, narrow)
    assert int(r.rows.sum()) == r.stats.rows_matched == n_rows, f"{tag}: {int(r.rows.sum())} rows of {n_rows}"
    out = {"n_keys": r.n_keys, "rows_out": int(r.rows.size), "wide_ms_per_call": w_ms, "wide_scan_kernel_ms": round(r.stats.scan_kernel_ms, 3),
           "wide_device_ms": round(r.stats.device_ms, 3), "wide_datapoints_per_s": round(n_rows / (w_ms / 1e3))}
    if narrow:
        out.update(narrow_ms_per_call=n_ms, speedup=round(n_ms / w_ms, 2))
    return out


def kernel_ms(ctx, q, tag, vt, cap, calls):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.scan_agg_keyed_wide(q, "default", tag, cap, vt)
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
        raise SystemExit("torch.profiler recorded no kernel of the wide call")
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def wide_part(S, capi, n_series, n_points):
    n = n_series * n_points
    sid = np.repeat(np.arange(1, n_series + 1, dtype=np.uint64), n_points)
    r = np.tile(np.arange(n_points, dtype=np.int64), n_series)
    ts = T0 + r * STEP
    rng = np.random.default_rng(11)
    lat = rng.integers(500, 9000, n)   # latency in hundredths: a decimal column of 2 digits
    calls = rng.integers(0, 1000, n)
    wide = ((sid.astype(np.int64) * 97 + r // 33) % 4096).astype(np.int64)   # 8,193-row blocks hold at most 249 values
    one = np.full(n, 7, np.int64)
    two = (r // 33 % 2).astype(np.int64)
    return S.write_part(sid, ts, np.ones(n, np.int64), [("latency", capi.VT_FLOAT64, lat, 2), ("calls", capi.VT_INT64, calls)],
                        tag_family="default", tags=[("wide", capi.VT_INT64, wide), ("one", capi.VT_INT64, one), ("two", capi.VT_INT64, two)]), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-calls", type=int, default=3)
    ap.add_argument("--bench-series", type=int, default=10_000)
    ap.add_argument("--bench-points", type=int, default=100_000)
    ap.add_argument("--c5-series", type=int, default=1000)
    ap.add_argument("--c5-points", type=int, default=100_000)
    ap.add_argument("--wide-series", type=int, default=2000)
    ap.add_argument("--wide-points", type=int, default=10_000)
    args = ap.parse_args()
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import capi
    from bydb_b200 import synth as S
    import bench
    out = {"steps": args.steps, "checked": "narrow and wide answers agree wherever both run; every row accounted for"}
    kernels = {}
    with pkg.Context(device=0) as ctx:
        # 1. the bench part, GROUP BY region
        part = bench.make_part(pkg, args.bench_series, args.bench_points, 1)
        n_rows, _ = part.counts()
        h = ctx.register_part(1, part.files())
        sids = np.arange(1, args.bench_series + 1, dtype=np.uint64)
        q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)])
        out["bench_region"] = {"datapoints": int(n_rows), **leg(ctx, q, "region", 0, 64, int(n_rows), args)}
        if args.profile_calls:
            kernels["bench_region"] = kernel_ms(ctx, q, "region", 0, 64, args.profile_calls)
        ctx.release_part(h)
        del part
        # 2. the C5 part, keyed on code (int64) and zone
        fields = [("delta", S.I_DELTA), ("fluct", S.I_FLUCT), ("rand", S.I_RANDOM100), ("counter", S.I_COUNTER),
                  ("latency", S.F_LATENCY), ("walk", S.F_WALK3), ("ints", S.F_INT1000), ("uniform", S.F_UNIFORM)]
        part = S.synth_part(args.c5_series, args.c5_points, fields, t0=T0, t_step=STEP, region_values=8, region_run=16, code_tag=True, zone_tag=True)
        n_rows, _ = part.counts()
        h = ctx.register_part(2, part.files())
        sids = np.arange(1, args.c5_series + 1, dtype=np.uint64)
        q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)],
                      series_group=((sids - 1) % 100).astype(np.int32), n_groups=100)
        out["c5_code"] = {"datapoints": int(n_rows), **leg(ctx, q, "code", pkg.VT_INT64, 64, int(n_rows), args)}
        out["c5_zone"] = {"datapoints": int(n_rows), **leg(ctx, q, "zone", 0, 64, int(n_rows), args)}
        ctx.release_part(h)
        del part
        # 3. an int64 tag of 4,096 values (wide only), and the small-V end on the same part
        part, n = wide_part(S, capi, args.wide_series, args.wide_points)
        h = ctx.register_part(3, part.files())
        sids = np.arange(1, args.wide_series + 1, dtype=np.uint64)
        q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("calls", pkg.AGG_COUNT), ("calls", pkg.AGG_MAX)],
                      series_group=((sids - 1) % 100).astype(np.int32), n_groups=100)
        out["wide_4096"] = {"datapoints": n, **leg(ctx, q, "wide", pkg.VT_INT64, 4096, n, args, narrow=False)}
        assert out["wide_4096"]["n_keys"] == 4096
        for tag in ("one", "two"):
            out[f"wide_part_{tag}"] = {"datapoints": n, **leg(ctx, q, tag, pkg.VT_INT64, 64, n, args)}
        if args.profile_calls:
            kernels["wide_4096"] = kernel_ms(ctx, q, "wide", pkg.VT_INT64, 4096, args.profile_calls)
        ctx.release_part(h)
    if kernels:
        out["wide_kernels_ms_per_call"] = kernels
    name, power = card()
    out.update(gpu=name, power_limit=power)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

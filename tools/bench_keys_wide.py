#!/usr/bin/env python
"""bench_keys_wide.py -- group-by on a tuple of stored tags in one scan pass (bydb_scan_agg_keys_wide) on one GPU, in one process.

The C5-shaped part of bench_keyed.py (1,000 series x 100,000 points = 1e8 datapoints), sum(latency), count(latency), max(delta)
per (100 service groups, key), grouped by (code, zone) (int64 + string, 6 x 5 values), by (code, zone, region) (8 more) and, on
the same part in the same run, by code alone through bydb_scan_agg_keyed_wide.  Warm-up, then --steps rounds that call the three
back to back (wall clock around calls that end in a device synchronise); per leg ms/call, the scan kernel's ms and the device ms
of the last call.  Checks: every leg's rows sum to rows_matched = all datapoints, and the (code, zone) rows folded over zone
equal the code call's rows.  Prints one JSON line with the card's name and power limit read in the same run.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--series", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100_000)
    args = ap.parse_args()
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import synth as S
    fields = [("delta", S.I_DELTA), ("fluct", S.I_FLUCT), ("rand", S.I_RANDOM100), ("counter", S.I_COUNTER),
              ("latency", S.F_LATENCY), ("walk", S.F_WALK3), ("ints", S.F_INT1000), ("uniform", S.F_UNIFORM)]
    part = S.synth_part(args.series, args.points, fields, t0=T0, t_step=STEP, region_values=8, region_run=16, code_tag=True, zone_tag=True)
    n_rows, _ = part.counts()
    out = {"datapoints": int(n_rows), "steps": args.steps}
    with pkg.Context(device=0) as ctx:
        h = ctx.register_part(1, part.files())
        sids = np.arange(1, args.series + 1, dtype=np.uint64)
        q = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)],
                      series_group=((sids - 1) % 100).astype(np.int32), n_groups=100)
        pair = [("default", "code", pkg.VT_INT64), ("default", "zone", 0)]
        triple = pair + [("default", "region", 0)]
        legs = {"code_keyed_wide": lambda: ctx.scan_agg_keyed_wide(q, "default", "code", 64, pkg.VT_INT64),
                "code_zone": lambda: ctx.scan_agg_keys_wide(q, pair, 4096),
                "code_zone_region": lambda: ctx.scan_agg_keys_wide(q, triple, 4096)}
        last = {}
        for _ in range(args.warmup):
            for name, fn in legs.items():
                last[name] = fn()
        spent = dict.fromkeys(legs, 0.0)
        for _ in range(args.steps):
            for name, fn in legs.items():
                t = time.perf_counter()
                last[name] = fn()
                spent[name] += time.perf_counter() - t
        ctx.release_part(h)
    for name, r in last.items():
        assert int(r.rows.sum()) == r.stats.rows_matched == n_rows, f"{name}: {int(r.rows.sum())} rows of {n_rows}"
        out[name] = {"rows_out": int(r.rows.size), "ms_per_call": round(spent[name] * 1e3 / args.steps, 3),
                     "scan_kernel_ms": round(r.stats.scan_kernel_ms, 3), "device_ms": round(r.stats.device_ms, 3),
                     "keys": getattr(r, "n_tuples", getattr(r, "n_keys", None))}
    one, two = last["code_keyed_wide"], last["code_zone"]
    folded = {}
    for g, k, n in zip(two.group_id.tolist(), two.key, two.rows.tolist()):
        folded[(g, k[0])] = folded.get((g, k[0]), 0) + n
    assert folded == {(g, k): n for g, k, n in zip(one.group_id.tolist(), one.key, one.rows.tolist())}, "(code, zone) folded over zone != code"
    out["checked"] = "rows sum to rows_matched on every leg; (code, zone) folded over zone equals the code call"
    name, power = card()
    out.update(gpu=name, power_limit=power)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_keys_wide_reduce.py -- the tuple collective (bydb_scan_reduce_keys_wide) against bydb_scan_agg_keys_wide on one context over
the same rows.

Two legs, each sharded by time window over --ranks ranks (rank r holds one part with window r of every series; one context per
GPU, ranks share a GPU when there are fewer), mailboxes sized with bydb_keys_wide_reduce_slot_bytes, and one more context holding
all the ranks' parts (time-disjoint, so one context scans them as one data set):
  - c5: bench_keys_wide.py's C5-shaped data (synth_part with the code and zone tags; --series x --points in all), sum(latency),
    count(latency), max(delta) per (100 service groups, code, zone);
  - high: --hi-series x --hi-points rows with two int64 tags that make a few thousand distinct pairs (at most 128 per block).
After --warmup rounds, --steps rounds each time one collective (every rank's call on its own thread; wall clock from the release of
the threads to the last return, every call ending in a device synchronise) and one single-context call, alternating; medians are
reported.  Checks: the root's answer equals the single-context answer (the same rows in the same order by their key bytes, equal
int64 values, floats within 1e-9, the same n_tuples).  Prints one JSON line with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_keyed import card  # noqa: E402

T0 = 1_700_000_000_000_000_000
STEP = 60_000_000_000


def collective(ctxs, qs, keys, root, cap):
    """-> (seconds, the root's answer): every rank's call on its own thread"""
    res, errs = [None] * len(ctxs), []
    go = threading.Barrier(len(ctxs) + 1)

    def body(r):
        go.wait()
        try:
            res[r] = ctxs[r].scan_reduce_keys_wide(qs[r], keys, root=root, max_values=cap)
        except Exception as e:  # noqa: BLE001
            errs.append(repr(e))
    th = [threading.Thread(target=body, args=(r,)) for r in range(len(ctxs))]
    for t in th:
        t.start()
    go.wait()
    t0 = time.perf_counter()
    for t in th:
        t.join()
    dt = time.perf_counter() - t0
    if errs:
        raise SystemExit(f"collective failed: {errs}")
    return dt, res[root]


def same(one, got, what):
    assert got.group_id.tolist() == one.group_id.tolist(), f"{what}: group ids"
    assert got.key == one.key, f"{what}: keys"
    assert got.rows.tolist() == one.rows.tolist() and got.val_i64.tolist() == one.val_i64.tolist(), f"{what}: rows / int64 values"
    assert np.allclose(got.val_f64, one.val_f64, rtol=1e-9, atol=0, equal_nan=True), f"{what}: float values"
    assert got.n_tuples == one.n_tuples, f"{what}: n_tuples"


def run_leg(pkg, ctxs, one_ctx, parts, sids, aggs, keys, cap, args, pid):
    """register rank r's part on rank r and every part on one_ctx; time the collective and the single-context call"""
    R = len(ctxs)
    groups = ((sids - 1) % 100).astype(np.int32)
    hs = [ctxs[r].register_part(pid + r, parts[r].files()) for r in range(R)]
    hw = [one_ctx.register_part(pid + 50 + r, parts[r].files()) for r in range(R)]
    qs = [pkg.Query(parts=[hs[r]], series_ids=sids, aggs=aggs, series_group=groups, n_groups=100) for r in range(R)]
    q1 = pkg.Query(parts=hw, series_ids=sids, aggs=aggs, series_group=groups, n_groups=100)
    t_coll, t_one = [], []
    got = one = None
    for step in range(args.warmup + args.steps):
        dt, got = collective(ctxs, qs, keys, args.root, cap)
        t = time.perf_counter()
        one = one_ctx.scan_agg_keys_wide(q1, keys, cap)
        d1 = time.perf_counter() - t
        if step >= args.warmup:
            t_coll.append(dt)
            t_one.append(d1)
    same(one, got, "collective vs one context")
    for r in range(R):
        ctxs[r].release_part(hs[r])
        one_ctx.release_part(hw[r])
    return {"n_tuples": got.n_tuples, "tag_values": [len(t) for t in got.key_tables], "rows_out": int(got.rows.size),
            "collective_ms_median": round(statistics.median(t_coll) * 1e3, 3), "one_context_ms_median": round(statistics.median(t_one) * 1e3, 3),
            "one_context_scan_kernel_ms": round(one.stats.scan_kernel_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--series", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--hi-series", type=int, default=2000)
    ap.add_argument("--hi-points", type=int, default=10_000)
    ap.add_argument("--root", type=int, default=0)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import capi
    from bydb_b200 import synth as S
    n_dev = max(torch.cuda.device_count(), 1)
    R = args.ranks
    cap = 4096
    ctxs = [pkg.Context(device=r % n_dev) for r in range(R)]
    one_ctx = pkg.Context(device=0)
    out = {"ranks": R, "gpus": n_dev, "steps": args.steps}
    try:
        # mailboxes for the larger of the two legs: every tag and the tuples at the cap, 100 groups x cap present groups
        q0 = pkg.Query(parts=[], series_ids=np.arange(1, max(args.series, args.hi_series) + 1, dtype=np.uint64),
                       aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)],
                       series_group=None, n_groups=1)
        slot = pkg.keys_wide_reduce_slot_bytes(q0, [("default", "code", pkg.VT_INT64), ("default", "zone", 0)], cap, 100 * cap)
        handles = [c.comm_export(slot, R) for c in ctxs]
        for r, c in enumerate(ctxs):
            c.comm_connect(r, R, handles)
        # ---- c5: window r of every series on rank r
        fields = [("delta", S.I_DELTA), ("fluct", S.I_FLUCT), ("rand", S.I_RANDOM100), ("counter", S.I_COUNTER),
                  ("latency", S.F_LATENCY), ("walk", S.F_WALK3), ("ints", S.F_INT1000), ("uniform", S.F_UNIFORM)]
        ppr = args.points // R
        parts = [S.synth_part(args.series, ppr, fields, t0=T0 + r * ppr * STEP, t_step=STEP, region_values=8, region_run=16,
                              code_tag=True, zone_tag=True, seed=0xB200 + r) for r in range(R)]
        out["c5"] = run_leg(pkg, ctxs, one_ctx, parts, np.arange(1, args.series + 1, dtype=np.uint64),
                            [("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)],
                            [("default", "code", pkg.VT_INT64), ("default", "zone", 0)], cap, args, 100)
        out["c5"]["datapoints"] = args.series * ppr * R
        del parts
        # ---- high: two int64 tags, a few thousand pairs
        n_s, n_p = args.hi_series, args.hi_points
        sid = np.repeat(np.arange(1, n_s + 1, dtype=np.uint64), n_p)
        row = np.tile(np.arange(n_p, dtype=np.int64), n_s)
        rng = np.random.default_rng(11)
        lat = rng.integers(500, 9000, sid.size)
        calls = rng.integers(0, 1000, sid.size)
        j = row // 64
        hi = ((sid.astype(np.int64) * 7 + j) % 64).astype(np.int64)
        lo = ((sid.astype(np.int64) + j // 2) % 50).astype(np.int64)
        bounds = [n_p * r // R for r in range(R + 1)]
        parts = []
        for r in range(R):
            m = (row >= bounds[r]) & (row < bounds[r + 1])
            parts.append(S.write_part(sid[m], T0 + row[m] * STEP, np.ones(int(m.sum()), np.int64),
                                      [("latency", capi.VT_FLOAT64, lat[m], 2), ("delta", capi.VT_INT64, calls[m])],
                                      tag_family="default", tags=[("code", capi.VT_INT64, hi[m]), ("zone", capi.VT_INT64, lo[m])]))
        out["high"] = run_leg(pkg, ctxs, one_ctx, parts, np.arange(1, n_s + 1, dtype=np.uint64),
                              [("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT), ("delta", pkg.AGG_MAX)],
                              [("default", "code", pkg.VT_INT64), ("default", "zone", pkg.VT_INT64)], cap, args, 200)
        out["high"]["datapoints"] = int(sid.size)
        out["checked"] = "the root's answer equals the single-context answer on both legs"
        name, power = card()
        out.update(gpu=name, power_limit=power)
        print(json.dumps(out))
    finally:
        for c in ctxs + [one_ctx]:
            c.close()


if __name__ == "__main__":
    main()

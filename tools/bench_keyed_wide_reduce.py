#!/usr/bin/env python
"""bench_keyed_wide_reduce.py -- the wide keyed collective (bydb_scan_reduce_keyed_wide) against bydb_scan_agg_keyed_wide on one
context over the same rows.

The part is bench_keyed_wide.py's 4,096-value leg (synth.write_part, --series x --points, the int64 tag `wide` with at most 249
values per block), sharded by series range over --ranks ranks: rank r holds one part with its range of series, one context per
GPU (ranks share a GPU when there are fewer), connected mailboxes sized with bydb_keyed_wide_reduce_slot_bytes.  One context also
holds the whole part.  After --warmup rounds, --steps rounds each time one collective (every rank's call on its own thread; wall
clock from the release of the threads to the last return) and one single-context call, alternating; the medians are reported.
Checks: the root's answer equals the single-context answer (same rows in the same order, same keys, equal int64 values, floats
within 1e-9) and n_keys = 4,096.  Prints one JSON line with the card's name and power limit read in the same run.
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
from bench_keyed_wide import STEP, T0, same  # noqa: E402


def columns(n_series, n_points):
    """bench_keyed_wide.wide_part's rows, as arrays that can be cut by series"""
    n = n_series * n_points
    sid = np.repeat(np.arange(1, n_series + 1, dtype=np.uint64), n_points)
    r = np.tile(np.arange(n_points, dtype=np.int64), n_series)
    rng = np.random.default_rng(11)
    lat = rng.integers(500, 9000, n)
    calls = rng.integers(0, 1000, n)
    wide = ((sid.astype(np.int64) * 97 + r // 33) % 4096).astype(np.int64)   # 8,193-row blocks hold at most 249 values
    return dict(sid=sid, ts=T0 + r * STEP, lat=lat, calls=calls, wide=wide)


def write(S, capi, c, rows):
    return S.write_part(c["sid"][rows], c["ts"][rows], np.ones(int(np.asarray(c["sid"][rows]).size), np.int64),
                        [("latency", capi.VT_FLOAT64, c["lat"][rows], 2), ("calls", capi.VT_INT64, c["calls"][rows])],
                        tag_family="default", tags=[("wide", capi.VT_INT64, c["wide"][rows])])


def collective(ctxs, qs, root, cap, vt):
    """-> (seconds, the root's answer): every rank's call on its own thread"""
    res, errs = [None] * len(ctxs), []
    go = threading.Barrier(len(ctxs) + 1)

    def body(r):
        go.wait()
        try:
            res[r] = ctxs[r].scan_reduce_keyed_wide(qs[r], "default", "wide", root=root, max_values=cap, value_type=vt)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=0, help="0 = one per visible GPU (at least 2)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--series", type=int, default=2000)
    ap.add_argument("--points", type=int, default=10_000)
    ap.add_argument("--root", type=int, default=0)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    from bydb_b200 import capi
    from bydb_b200 import synth as S
    n_dev = max(torch.cuda.device_count(), 1)
    R = args.ranks or max(n_dev, 2)
    cap, vt = 4096, pkg.VT_INT64
    cols = columns(args.series, args.points)
    n = int(cols["sid"].size)
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    groups = ((sids - 1) % 100).astype(np.int32)
    aggs = [("latency", pkg.AGG_SUM), ("calls", pkg.AGG_COUNT), ("calls", pkg.AGG_MAX)]
    bounds = [round(args.series * r / R) for r in range(R + 1)]   # rank r: the series [bounds[r], bounds[r + 1]) by position
    ctxs = [pkg.Context(device=r % n_dev) for r in range(R)]
    try:
        q0 = pkg.Query(parts=[], series_ids=sids, aggs=aggs, series_group=groups, n_groups=100)
        slot = pkg.keyed_wide_reduce_slot_bytes(q0, "default", "wide", cap, 100 * cap, vt)
        handles = [c.comm_export(slot, R) for c in ctxs]
        for r, c in enumerate(ctxs):
            c.comm_connect(r, R, handles)
        qs, parts = [], []   # a part image owns the buffers its files() point into: keep it while it is registered
        for r in range(R):
            parts.append(write(S, capi, cols, slice(bounds[r] * args.points, bounds[r + 1] * args.points)))
            h = ctxs[r].register_part(10 + r, parts[-1].files())
            qs.append(pkg.Query(parts=[h], series_ids=sids, aggs=aggs, series_group=groups, n_groups=100))
        one_ctx = ctxs[0]
        parts.append(write(S, capi, cols, slice(0, n)))
        hw = one_ctx.register_part(1, parts[-1].files())
        q1 = pkg.Query(parts=[hw], series_ids=sids, aggs=aggs, series_group=groups, n_groups=100)
        t_coll, t_one = [], []
        for step in range(args.warmup + args.steps):
            dt, got = collective(ctxs, qs, args.root, cap, vt)
            t = time.perf_counter()
            one = one_ctx.scan_agg_keyed_wide(q1, "default", "wide", cap, vt)
            d1 = time.perf_counter() - t
            if step >= args.warmup:
                t_coll.append(dt)
                t_one.append(d1)
        same(one, got, "collective vs one context")
        assert got.n_keys == cap == one.n_keys, (got.n_keys, one.n_keys)
        name, power = card()
        print(json.dumps({
            "ranks": R, "gpus": n_dev, "datapoints": n, "n_keys": got.n_keys, "rows_out": int(got.rows.size), "steps": args.steps,
            "collective_ms_median": round(statistics.median(t_coll) * 1e3, 3), "one_context_ms_median": round(statistics.median(t_one) * 1e3, 3),
            "checked": "the root's answer equals the single-context answer",
            "gpu": name, "power_limit": power}))
    finally:
        for c in ctxs:
            c.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_keyed_reduce.py -- group-by on a stored tag sharded over ranks (bydb_scan_reduce_keyed) against one GPU (bydb_scan_agg_keyed).

Workload: bench.py's 1e9 part (10 000 series x 100 000 points, the region tag with 8 values), query sum(latency), count(latency)
GROUP BY region.  The series are sharded by series range over R = 1, 2, 4 and 8 ranks, as many as there are GPUs: one context
and one thread per rank, rank r on GPU r.  Each shard holds exactly the whole part's rows of its series (bench.make_part seeds
its generators by series id).

Per R: --warmup collectives, then --steps timed ones (wall clock around calls that end in a device synchronise; a collective's
time is its slowest rank's).  Reported: ms per call, datapoints/s, each rank's pass time (CUDA events of its scan passes,
stats.device_ms), and the root's union-and-combine time per call (key_union, rank_span_check, combine_keyed and merge_first
kernels, from torch.profiler's CUDA activity over --profile-calls further collectives).  Every answer must equal the one-GPU
answer: keys, rows and int64 values exactly, floats within 1e-12 relative.  One JSON line, with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ROOT_KERNELS = ("key_union_kernel", "rank_span_check_kernel", "combine_keyed_kernel", "merge_first_kernel")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=60)
    if out.returncode != 0:
        raise SystemExit("nvidia-smi failed: " + out.stderr)
    name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
    return name, power


def equal(got, want):
    assert got.key == want.key, (got.key, want.key)
    assert got.rows.tolist() == want.rows.tolist() and got.val_i64.tolist() == want.val_i64.tolist()
    assert np.allclose(got.val_f64, want.val_f64, rtol=1e-12, atol=0)


def collective(ctxs, qs, root):
    """one keyed collective on len(ctxs) threads -> (root result, per-rank results, wall seconds)"""
    R = len(ctxs)
    res, errs = [None] * R, []
    go = threading.Barrier(R + 1)

    def body(r):
        go.wait()
        try:
            res[r] = ctxs[r].scan_reduce_keyed(qs[r], "default", "region", root=root)
        except Exception as e:  # noqa: BLE001
            errs.append(repr(e))
    th = [threading.Thread(target=body, args=(r,)) for r in range(R)]
    for t in th:
        t.start()
    go.wait()
    t0 = time.perf_counter()
    for t in th:
        t.join()
    dt = time.perf_counter() - t0
    if errs:
        raise SystemExit(f"collective failed: {errs}")
    return res[root], res, dt


def root_kernels_ms(ctxs, qs, calls):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            collective(ctxs, qs, 0)
        for d in range(len(ctxs)):
            torch.cuda.synchronize(d)
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0)
        name = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("bydb::", "")
        if name in ROOT_KERNELS:
            out[name] = round(us / 1e3 / calls, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ranks", default="1,2,4,8")
    ap.add_argument("--profile-calls", type=int, default=2)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    from bench import make_part
    pkg = ge.load_package()
    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("no GPU")
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    aggs = [("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)]
    n_rows = args.series * args.points
    out = {"workload": f"{n_rows:.0e} datapoints ({args.series} series x {args.points} points), sum(latency), count(latency) GROUP BY region",
           "steps": args.steps, "gpus_present": n_dev}
    # ---- one GPU: bydb_scan_agg_keyed over the whole part
    whole = make_part(pkg, args.series, args.points, 1)
    with pkg.Context(device=0) as ctx:
        h = ctx.register_part(1, whole.files())
        q = pkg.Query(parts=[h], series_ids=sids, aggs=aggs)
        for _ in range(args.warmup):
            want = ctx.scan_agg_keyed(q, "default", "region")
        t = time.perf_counter()
        for _ in range(args.steps):
            want = ctx.scan_agg_keyed(q, "default", "region")
        ms = (time.perf_counter() - t) * 1e3 / args.steps
        ctx.release_part(h)
    del whole
    assert int(want.rows.sum()) == n_rows
    out["one_gpu_scan_agg_keyed"] = {"ms_per_call": round(ms, 3), "datapoints_per_s": round(n_rows / (ms / 1e3)), "n_keys": want.n_keys,
                                     "passes_device_ms": round(want.stats.device_ms, 3)}
    # ---- R ranks on R GPUs: bydb_scan_reduce_keyed over series-range shards
    legs = {}
    for R in [int(x) for x in args.ranks.split(",")]:
        if R > n_dev:
            legs[str(R)] = "not measured: fewer GPUs present"
            continue
        bounds = [(r * args.series // R, (r + 1) * args.series // R) for r in range(R)]
        ctxs = [pkg.Context(device=r) for r in range(R)]
        try:
            probe = pkg.Query(parts=[], series_ids=sids, aggs=aggs)
            slot = pkg.keyed_reduce_slot_bytes(probe, "default", "region")
            handles = [c.comm_export(slot, R) for c in ctxs]
            for r, c in enumerate(ctxs):
                c.comm_connect(r, R, handles)
            qs = []
            for r, (lo, hi) in enumerate(bounds):
                part = make_part(pkg, hi - lo, args.points, lo + 1)
                qs.append(pkg.Query(parts=[ctxs[r].register_part(1, part.files())], series_ids=sids, aggs=aggs))
                del part
            for _ in range(args.warmup):
                got, _, _ = collective(ctxs, qs, 0)
            times, per_rank = [], []
            for _ in range(args.steps):
                got, res, dt = collective(ctxs, qs, 0)
                times.append(dt)
                per_rank = [round(x.stats.device_ms, 3) for x in res]
            equal(got, want)
            cms = sum(times) * 1e3 / args.steps
            legs[str(R)] = {"ms_per_call": round(cms, 3), "datapoints_per_s": round(n_rows / (cms / 1e3)),
                            "rank_pass_device_ms": per_rank,
                            "root_union_combine_ms": root_kernels_ms(ctxs, qs, args.profile_calls) if args.profile_calls else None}
        finally:
            for c in ctxs:
                c.close()
    out["scan_reduce_keyed_by_ranks"] = legs
    name, power = card()
    out.update(gpu=name, power_limit=power, checked="every collective answer equals the one-GPU answer")
    print(json.dumps(out))


if __name__ == "__main__":
    main()

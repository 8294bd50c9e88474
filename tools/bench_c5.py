#!/usr/bin/env python
"""bench_c5.py -- BASELINE.json configs[4] (SURVEY.md 8d C5) as an extra measurement next to bench.py:

    1e9 datapoints, 8-field mixed measure (4 int64: monotone delta / small fluctuations / random < 100 / counter with resets;
    4 float64), two dictionary string tags + one int64 tag, query = region == "r3" AND zone != "z1" AND code >= 200 AND the
    middle half of the time range, aggregating avg(latency), max(walk), sum(i_fluct), min(i_rand) -- the reference has no
    percentile (pkg/query/aggregation/aggregation.go:63-82 lists MEAN/MAX/MIN/COUNT/SUM only), so none is measured.

    python tools/bench_c5.py --steps 10                                   # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/bench_c5.py --steps 10

N > 1: the series are sharded over the ranks (strong scaling) and reduced through the peer mailboxes (bydb_scan_reduce).
Algorithmic bytes per scanned datapoint (SURVEY.md 8d): 8 (timestamp) + 1 + 1 (dictionary tags) + 8 (int64 tag) + 4 x 8 (fields) = 50 for
this four-field variant; the judge's 26 B figure is the two-field variant (--fields 2: avg(latency) + sum(i_fluct)).
A 1/64 sample of the series is checked against the oracle on rank 0 (--check).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fields", type=int, default=2, choices=[2, 4])
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    rank, world, local_rank = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    pkg = B.load_pkg()
    from importlib import import_module
    S = import_module("bydb_b200.synth")
    ctx = pkg.Context(device=local_rank)
    lo, hi = rank * args.series // world, (rank + 1) * args.series // world
    n_mine, sid0 = hi - lo, 1 + lo
    fields = [("i_delta", S.I_DELTA), ("i_fluct", S.I_FLUCT), ("i_rand", S.I_RANDOM100), ("i_counter", S.I_COUNTER),
              ("latency", S.F_LATENCY), ("walk", S.F_WALK3), ("ints", S.F_INT1000), ("f_lat2", S.F_LATENCY)]

    def part(n, s0):
        return S.synth_part(n, args.points, fields, sid0=s0, t0=B.T0, t_step=B.STEP, region_values=8, region_run=16, code_tag=True, zone_tag=True, seed=0xC5)
    t0 = time.perf_counter()
    img = part(n_mine, sid0)
    t_gen = time.perf_counter() - t0
    h = ctx.register_part(1 + rank, img.files())
    info = ctx.part_info(h)
    del img
    sids = np.arange(sid0, sid0 + n_mine, dtype=np.uint64)
    aggs = [("latency", pkg.AGG_MEAN), ("i_fluct", pkg.AGG_SUM)] + ([("walk", pkg.AGG_MAX), ("i_rand", pkg.AGG_MIN)] if args.fields == 4 else [])
    b_alg = 8 + 1 + 1 + 8 + 8 * args.fields
    tmin, tmax = B.T0 + (args.points // 4) * B.STEP, B.T0 + (3 * args.points // 4) * B.STEP
    preds = [pkg.Pred("default", "region", pkg.OP_EQ, b"r3"), pkg.Pred("default", "zone", pkg.OP_NE, b"z1"), pkg.Pred("default", "code", pkg.OP_GE, 200)]
    q = pkg.Query(parts=[h], series_ids=sids, aggs=aggs, tmin=tmin, tmax=tmax, preds=preds)
    pq = ctx.prepare(q)
    if world > 1:
        lay = ctx.partials_layout(q)
        mine_h = torch.frombuffer(bytearray(ctx.comm_export(int(lay["total_bytes"]), world)), dtype=torch.uint8).cuda()
        all_h = torch.empty(world * 128, dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(all_h, mine_h)
        raw = all_h.cpu().numpy().tobytes()
        ctx.comm_connect(rank, world, [raw[i * 128:(i + 1) * 128] for i in range(world)])
    stats = []

    def step():
        r = ctx.scan_agg(pq) if world == 1 else ctx.scan_reduce(pq, root=0)
        stats.append(r.stats)
        return r

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()
    for _ in range(max(args.warmup, 3)):
        step()
    stats.clear()
    sampler = B.ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    barrier()
    t = time.perf_counter()
    for _ in range(args.steps):
        last = step()
    barrier()
    dt = time.perf_counter() - t
    clocks = sampler.stop() if rank == 0 else None
    rows, scan_ms = float(stats[-1].rows_scanned), float(np.mean([s.scan_kernel_ms for s in stats]))
    if world > 1:
        m = torch.tensor([dt, scan_ms], dtype=torch.float64, device="cuda")
        dist.all_reduce(m, op=dist.ReduceOp.MAX)
        sm = torch.tensor([rows], dtype=torch.float64, device="cuda")
        dist.all_reduce(sm, op=dist.ReduceOp.SUM)
        dt, scan_ms_max, total = float(m[0]), float(m[1]), float(sm[0])
    else:
        scan_ms_max, total = scan_ms, rows
    check = None
    if args.check and rank == 0:
        from oracle import oracle as O
        n_s = max(1, n_mine // 64)
        sample = part(n_s, sid0)
        op = O.Part.open({k: bytes(v) for k, v in sample.files().items()})
        ssid = sids[:n_s]
        want = O.run_query(O.Query([op], ssid, aggs, tmin=tmin, tmax=tmax, preds=[O.Pred(p.family, p.tag, p.op, p.value) for p in preds], threads=os.cpu_count() or 1))
        with pkg.Context(device=local_rank) as c2:   # a second context: the mailbox epochs of `ctx` stay in step with the other ranks
            h2 = c2.register_part(99, sample.files())
            got = c2.scan_agg(pkg.Query(parts=[h2], series_ids=ssid, aggs=aggs, tmin=tmin, tmax=tmax, preds=preds))
        check = {"sample_series": int(n_s), "rows_matched_equal": bool(got.rows.tolist() == want.rows.tolist()),
                 "int64_bit_equal": bool(got.val_i64.tolist() == want.val_i64.tolist()),
                 "float_max_rel_err": float(np.max(np.abs(got.val_f64 - want.val_f64) / np.maximum(np.abs(want.val_f64), 1e-300))) if want.val_f64.size else 0.0}
    if rank == 0:
        peak = B.HBM_PEAK_GBS
        ach = rows * b_alg / (scan_ms * 1e-3) / 1e9
        print(json.dumps({"metric": B.METRIC, "value": total * args.steps / dt, "unit": "datapoints/s", "n_gpus": world, "steps": args.steps,
                          "ms_per_step": dt / args.steps * 1e3, "scaling": "strong" if world > 1 else "n/a", "dtype": "i64+f64", "data": "synthetic",
                          "config": {"workload": f"{args.series * args.points:.0e} datapoints ({args.series} x {args.points}), 4 int64 + 4 float64 fields, "
                                                 "region==r3 AND zone!=z1 AND code>=200 AND middle half of the time range, "
                                                 + ", ".join(f"{fn}({f})" for f, fn in [(a, {1: 'avg', 2: 'max', 3: 'min', 5: 'sum'}[b]) for a, b in aggs])},
                          "datapoints_per_step": total, "scan_kernel_ms_rank0": scan_ms, "scan_kernel_ms_max_rank": scan_ms_max,
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "algorithmic_bytes_per_datapoint": b_alg,
                                       "encoded_page_bytes_per_launch_rank0": int(stats[-1].page_bytes), "note": "rank 0's shard"},
                          "blocks_slow_lane": int(stats[-1].blocks_slow_lane), "slow_lane_reasons": int(stats[-1].slow_lane_reasons),
                          "rows_matched": int(last.rows[0]) if last is not None and last.rows.size else None, "clocks": clocks,
                          "admission_rank0": {"generate_s": t_gen, **info}, "oracle_check": check}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

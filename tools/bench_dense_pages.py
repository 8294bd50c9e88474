#!/usr/bin/env python
"""bench_dense_pages.py -- the express lane over dense pages against the same lane over the reference's varint pages.

    python tools/bench_dense_pages.py [--rounds 3] [--steps 20]

One process on one GPU: bench.py's 1e9-datapoint part is generated once and registered in two contexts, dense pages on (the
default) and off (Context(dense_pages=False)); both copies stay resident (~49 GB together).  Every round runs, alternated
between the two, bench.py's C3 query as
  plain   bydb_scan_agg calls: scan_kernel_ms and device_ms from the library's CUDA events, and page bytes (the
          query's reference page bytes on both contexts: the counter does not depend on the form read);
  graph   the prepared query replayed as one CUDA graph: wall ms per call (host clock around calls that end in a synchronise).
It prints per (round, context) those numbers and the scan's rate over those page bytes (for the dense context that is not the
rate of the bytes it read; DESIGN.md 7 gives those), the read roof (bench_express_fetch.roof: the
fastest read-only torch reduction over a buffer of the varint step's page bytes), register_ms, hbm_bytes and the dense pages,
whether both contexts' outputs (plain and graph) are bit-identical, and the card's name, power limit, SM clock and throttle
reasons (nvidia-smi, read-only queries) before and after.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench as B  # noqa: E402
from bench_express_fetch import card_state, roof  # noqa: E402


def sig(r):
    return (r.group_id.tobytes(), r.rows.tobytes(), r.val_i64.tobytes(), r.val_f64.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--services", type=int, default=1000)
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    print("card:", card_state(), flush=True)
    pkg = B.load_pkg()
    img = B.make_part(pkg, args.series, args.points, 1)
    files = img.files()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    arms = {}
    for name, dense in (("varint", False), ("dense", True)):
        ctx = pkg.Context(device=0, dense_pages=dense)
        t0 = time.perf_counter()
        h = ctx.register_part(1, files)
        reg_ms = (time.perf_counter() - t0) * 1e3
        pq = ctx.prepare(B.c3_query(pkg, [h], sids, args.services))
        gq = ctx.prepare_graph(B.c3_query(pkg, [h], sids, args.services))
        info = ctx.part_info(h)
        print(f"{name:7s} register_ms {reg_ms:.0f}  hbm_bytes {info['hbm_bytes']}  dense_pages {info['dense_pages']}  "
              f"dense_bytes {info['dense_bytes']}", flush=True)
        for _ in range(args.warmup):
            ctx.scan_agg(pq)
            gq.run()
        arms[name] = (ctx, h, pq, gq)
    rows, sigs, roof_ms, varint_bytes = {}, {}, [], None
    for rnd in range(args.rounds):
        for name, (ctx, h, pq, gq) in arms.items():
            stats = []
            for _ in range(args.steps):
                r = ctx.scan_agg(pq)
                stats.append(r.stats)
            t0 = time.perf_counter()
            for _ in range(args.steps):
                g = gq.run()
            wall = (time.perf_counter() - t0) / args.steps * 1e3
            scan = float(np.mean([s.scan_kernel_ms for s in stats]))
            dev = float(np.mean([s.device_ms for s in stats]))
            pb = int(stats[-1].page_bytes)
            if name == "varint":
                varint_bytes = pb
            sigs.setdefault(name, set()).update({sig(r), sig(g)})
            rows.setdefault(name, []).append((scan, dev, wall))
            print(f"round {rnd} {name:7s} scan_kernel_ms {scan:.4f}  device_ms {dev:.4f}  graph wall ms/call {wall:.4f}  "
                  f"page bytes {pb}  {pb / scan / 1e6:.0f} GB/s of page bytes  blocks_express_lane {stats[-1].blocks_express_lane}  "
                  f"blocks_slow_lane {stats[-1].blocks_slow_lane}  rows_scanned {stats[-1].rows_scanned}", flush=True)
        rf = roof(torch, varint_bytes, 20)
        roof_ms.append(min(rf.values()))
        print(f"round {rnd} roof    {min(rf.values()):.4f} ms over {varint_bytes} B = {varint_bytes / min(rf.values()) / 1e6:.0f} GB/s", flush=True)
    gbps = varint_bytes / float(np.mean(roof_ms)) / 1e6
    print(f"summary (mean [min, max] over rounds; read roof {gbps:.0f} GB/s):")
    for name, v in rows.items():
        a = np.array(v)
        print(f"  {name:7s} scan {a[:, 0].mean():.4f} [{a[:, 0].min():.4f}, {a[:, 0].max():.4f}] ms  "
              f"device {a[:, 1].mean():.4f} ms  graph wall {a[:, 2].mean():.4f} [{a[:, 2].min():.4f}, {a[:, 2].max():.4f}] ms")
    same = len(sigs["varint"]) == 1 and sigs["varint"] == sigs["dense"]
    print("outputs bit-identical (plain and graph, dense vs varint):", same, flush=True)
    for ctx, h, pq, gq in arms.values():
        gq.close()
        ctx.release_part(h)
        ctx.close()
    print("card:", card_state(), flush=True)


if __name__ == "__main__":
    main()

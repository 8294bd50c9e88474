#!/usr/bin/env python
"""time_variants.py -- times several builds of libbydbgpu.so (kernel experiments, `make variant` in skywalking-banyandb_b200/) in ONE
process on one GPU: the synthetic part is generated once, every variant registers it, runs two queries of the bench
shape and must return bit-identical results to the first library given.

    python tools/time_variants.py libbydbgpu.so variants/dual.so variants/allrows.so [--steps 30]

Queries: Q1 = bench.py's (time range AND region=="r3", mean(latency)+max(walk): masked rows), Q2 = sum(latency)+
count(latency) over every row of the part (no predicate, full range: the all-rows-active shape of BASELINE config 3).
Prints one line per (variant, query): wall ms/step, device ms/step, scan kernel ms (CUDA events inside the library).
"""
from __future__ import annotations

import argparse
import importlib
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402


def fresh_package(lib_path):
    """Re-imports the package bound to another shared library (each library keeps its own context and kernels)."""
    os.environ["BYDB_GPU_LIB"] = lib_path
    import __graft_entry__ as ge
    for name in [m for m in sys.modules if m == ge.PKG_NAME or m.startswith(ge.PKG_NAME + ".")]:
        del sys.modules[name]
    return ge.load_package()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="paths relative to skywalking-banyandb_b200/")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--series", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100_000)
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    pkg0 = B.load_pkg()
    img = B.make_part(pkg0, args.series, args.points, 1)
    files = img.files()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    reference = {}
    for lib in args.libs:
        path = os.path.join(ROOT, "skywalking-banyandb_b200", lib)
        if not os.path.exists(path):
            print(lib, "MISSING")
            continue
        pkg = fresh_package(path)
        ctx = pkg.Context(device=0)
        h = ctx.register_part(1, files)
        q1 = B.c2_query(pkg, [h], sids, args.points)
        q2 = pkg.Query(parts=[h], series_ids=sids, aggs=[("latency", pkg.AGG_SUM), ("latency", pkg.AGG_COUNT)])
        for qname, q in (("masked", q1), ("allrows", q2)):
            pq = ctx.prepare(q)
            for _ in range(3):
                r = ctx.scan_agg(pq)
            torch.cuda.synchronize()
            t = time.perf_counter()
            stats = []
            for _ in range(args.steps):
                r = ctx.scan_agg(pq)
                stats.append(r.stats)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t) / args.steps * 1e3
            sig = (r.val_i64.tobytes(), r.val_f64.tobytes(), r.rows.tobytes())
            same = reference.setdefault(qname, sig) == sig
            print(f"{lib:28s} {qname:8s} wall {wall:.4f} ms  device {np.mean([s.device_ms for s in stats]):.4f} ms  "
                  f"scan {np.mean([s.scan_kernel_ms for s in stats]):.4f} ms  slow-lane blocks {stats[-1].blocks_slow_lane}  "
                  f"{'result identical' if same else 'RESULT DIFFERS FROM ' + args.libs[0]}", flush=True)
        ctx.release_part(h)
        ctx.close()
    os.environ.pop("BYDB_GPU_LIB", None)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_express_fetch.py -- how close the express lane (scan_sum_express_kernel) comes to the page stream's read roof.

    python tools/bench_express_fetch.py [--make] [--rounds 2] [--steps 20] [NAME=LIB ...]

One process on one GPU: bench.py's 1e9-datapoint part is generated once, then every round runs, alternated,
  roof      read-only torch reductions over a device buffer of the step's page bytes (float32 / float16 .sum(), float32
            .amax(), and float32 .sum() over rows of 4 KB); the fastest of them is the read bandwidth this card is shown to
            reach in this session.  The skeleton can beat it: it is a reachable rate, not a bound;
  skeleton  the express lane built with -DBYDB_EXPRESS_DECODE=0 (ring, batches and bookkeeping kept, the decode skipped:
            its sums are WRONG on purpose; it is only ever timed, never a result);
  the libraries given (default: the shipped build).
Each library registers the part and runs bench.py's C3 query (plain calls, CUDA events inside the library); the script prints
scan_kernel_ms, page bytes, GB/s and the fraction of the roof per (round, variant), blocks_express_lane and whether the result
arrays are bit-identical to the first decoding library's.  The card's name, power limit, SM clock and throttle reasons
(nvidia-smi, read-only queries) are printed before and after.

--make builds the skeleton with `make variant` into skywalking-banyandb_b200/variants/skeleton.so (git-ignored) and times it
with the shipped build; other kernel variants (make variant OUT=variants/x.so EXTRA=...) are given as NAME=LIB, paths relative
to skywalking-banyandb_b200/.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "skywalking-banyandb_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench as B  # noqa: E402
from time_variants import fresh_package  # noqa: E402

SKELETON_FLAGS = "-DBYDB_EXPRESS_DECODE=0"


def card_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active,temperature.gpu"
    try:
        return subprocess.check_output(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], text=True).strip()
    except Exception as ex:  # noqa: BLE001
        return f"nvidia-smi unavailable ({ex})"


def roof(torch, nbytes, reps):
    """ms of read-only reductions over nbytes (CUDA events, median of reps after a warm-up)."""
    x32 = torch.ones(nbytes // 4, dtype=torch.float32, device="cuda")
    x16 = x32.view(torch.float16)
    rows = x32[: x32.numel() // 1024 * 1024].view(-1, 1024)  # 4 KB rows
    ops = {"float32.sum": x32.sum, "float16.sum": x16.sum, "float32.amax": x32.amax, "float32.sum(rows of 4 KB)": lambda: rows.sum(1)}
    out = {}
    for name, op in ops.items():
        for _ in range(3):
            op()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            op()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = float(np.median(ts))
    del x32, x16, rows
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", help="NAME=LIB (relative to skywalking-banyandb_b200/)")
    ap.add_argument("--make", action="store_true", help="build variants/skeleton.so with make variant first")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--services", type=int, default=1000)
    args = ap.parse_args()
    if args.make:
        subprocess.check_call(["make", "-s", "-C", PKG_DIR, "variant", "OUT=variants/skeleton.so", f"EXTRA={SKELETON_FLAGS}"])
    libs = [tuple(s.split("=", 1)) for s in args.libs]
    if not libs:
        libs = [("shipped", "libbydbgpu.so")]
        if args.make:
            libs = [("skeleton", "variants/skeleton.so")] + libs
    import torch
    torch.cuda.set_device(0)
    print("card:", card_state(), flush=True)
    pkg0 = B.load_pkg()
    img = B.make_part(pkg0, args.series, args.points, 1)
    files = img.files()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    reference, rows = None, {}
    for rnd in range(args.rounds):
        page_bytes = None
        for name, lib in libs:
            path = os.path.join(PKG_DIR, lib)
            if not os.path.exists(path):
                print(f"round {rnd} {name:10s} MISSING {path}", flush=True)
                continue
            pkg = fresh_package(path)
            ctx = pkg.Context(device=0)
            h = ctx.register_part(1, files)
            pq = ctx.prepare(B.c3_query(pkg, [h], sids, args.services))
            for _ in range(args.warmup):
                r = ctx.scan_agg(pq)
            stats = []
            for _ in range(args.steps):
                r = ctx.scan_agg(pq)
                stats.append(r.stats)
            ms = float(np.mean([s.scan_kernel_ms for s in stats]))
            page_bytes = int(stats[-1].page_bytes)
            sig = (r.group_id.tobytes(), r.rows.tobytes(), r.val_i64.tobytes(), r.val_f64.tobytes())
            if "skeleton" in name:
                same = "skeleton: result not checked"
            else:
                reference = reference or sig
                same = "result identical" if sig == reference else "RESULT DIFFERS"
            rows.setdefault(name, []).append(ms)
            print(f"round {rnd} {name:10s} scan_kernel_ms {ms:.4f} (min {min(s.scan_kernel_ms for s in stats):.4f})  "
                  f"page bytes {page_bytes}  {page_bytes / ms / 1e6:.0f} GB/s  blocks_express_lane {stats[-1].blocks_express_lane}  "
                  f"blocks_slow_lane {stats[-1].blocks_slow_lane}  {same}", flush=True)
            ctx.release_part(h)
            ctx.close()
            os.environ.pop("BYDB_GPU_LIB", None)
        if page_bytes:
            rf = roof(torch, page_bytes, 20)
            best = min(rf.values())
            rows.setdefault("roof", []).append(best)
            print(f"round {rnd} roof       " + "  ".join(f"{k} {v:.4f} ms {page_bytes / v / 1e6:.0f} GB/s" for k, v in rf.items()),
                  flush=True)
    if "roof" in rows:
        r = float(np.mean(rows["roof"]))
        print(f"summary (mean over rounds; fraction of the roof = roof ms / variant ms, roof {r:.4f} ms "
              f"= {page_bytes / r / 1e6:.0f} GB/s):")
        for name, v in rows.items():
            m = float(np.mean(v))
            print(f"  {name:10s} {m:.4f} ms  [{min(v):.4f}, {max(v):.4f}]  {page_bytes / m / 1e6:.0f} GB/s  {r / m:.3f} of the roof")
    print("card:", card_state(), flush=True)


if __name__ == "__main__":
    main()

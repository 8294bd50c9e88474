#!/usr/bin/env python
"""bench_step_stages.py -- where one replayed prepared step (bydb_scan_agg_prepared) spends its time beside its scan.

    python tools/bench_step_stages.py [--lib NAME=LIB ...] [--rounds 2] [--replays 2000] [--out DIR] [--dump-outputs DIR]

One process on one GPU (it fails without one: nothing here has a CPU form).  bench.py's part and C3 query are built once;
every library given (default: the shipped build; paths relative to skywalking-banyandb_b200/, e.g. a build of another
commit kept under variants/) registers the part in a context of its own, and the rounds then alternate the libraries
A/B/A/B.  Per (round, library), after a warm-up of every shape:
  plain      mean scan_kernel_ms and device_ms of bydb_scan_agg (CUDA events inside the library), as bench.py reports them
  wall       --replays replays through GraphQuery.run(), timed with a host clock in blocks of --block calls (each call ends in
             the library's synchronise): min / median / p90 of the per-block ms per step
  device     stats.device_ms of every one of those replays (events around the graph launch): min / median
  host       wall median - device median: launch, synchronise, result parsing, Python
  bare       the same replays through a bare ctypes loop (bydb_scan_agg_prepared + bydb_result_free, no numpy arrays): wall
             median per block; wall - bare is the Python wrapper's share
The summary gives, per library, the median over rounds and the round-to-round spread of each line: a difference between
two libraries means something only when it is larger than that spread.  Afterwards one torch.profiler pass per library
(CUDA activities, a run of its own: tracing slows the host) lists the kernel, memcpy and memset rows of one replay with the
gaps between them; the traces go to --out (a temporary directory when not given).  The card's name, power limit, SM clock
and throttle reasons (nvidia-smi, read-only queries) are printed before and after.  --dump-outputs DIR writes each library's last replayed result as DIR/NAME/*.npy.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "skywalking-banyandb_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench as B  # noqa: E402
from bench_express_fetch import card_state  # noqa: E402
from time_variants import fresh_package  # noqa: E402


def blocks_ms(call, replays, block):
    """-> ms per step of each block of `block` calls (host clock; every call returns synchronised)."""
    out = []
    for _ in range(replays // block):
        t = time.perf_counter()
        for _ in range(block):
            call()
        out.append((time.perf_counter() - t) / block * 1e3)
    return np.asarray(out)


def one_round(lib, args):
    ctx, gq, pq, capi = lib["ctx"], lib["gq"], lib["pq"], lib["capi"]
    for _ in range(3):
        ctx.scan_agg(pq)
    plain = [ctx.scan_agg(pq).stats for _ in range(args.plain_steps)]
    for _ in range(args.block):
        gq.run()
    dev = []

    def wrapped():
        lib["last"] = gq.run()
        dev.append(lib["last"].stats.device_ms)
    wall = blocks_ms(wrapped, args.replays, args.block)
    L, r = ctx._L, capi._Result()
    run, free, ch, qh, ref = L.bydb_scan_agg_prepared, L.bydb_result_free, ctx._h, gq._h, C.byref(r)

    def bare():
        if run(ch, qh, ref) != 0:
            raise RuntimeError(L.bydb_last_error())
        free(ch, ref)
    bare_ms = blocks_ms(bare, args.replays, args.block)
    return {"plain_scan_ms": float(np.mean([s.scan_kernel_ms for s in plain])), "plain_device_ms": float(np.mean([s.device_ms for s in plain])),
            "wall_min": float(wall.min()), "wall_median": float(np.median(wall)), "wall_p90": float(np.percentile(wall, 90)),
            "device_min": float(np.min(dev)), "device_median": float(np.median(dev)),
            "host_share": float(np.median(wall) - np.median(dev)), "bare_median": float(np.median(bare_ms)),
            "wrapper_share": float(np.median(wall) - np.median(bare_ms))}


def profile_replay(torch, lib, out_dir, n=5):
    """One traced pass of n replays: the device rows (kernel / memcpy / memset) of the last one, with the gap before each."""
    from torch.profiler import ProfilerActivity, profile
    gq = lib["gq"]
    for _ in range(3):
        gq.run()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            gq.run()
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"replay_{lib['name']}.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    ev.sort(key=lambda e: e["ts"])
    print(f"per-node trace of {lib['name']}: {len(ev)} device rows in {n} replays -> {path}")
    if not ev or len(ev) % n:
        print("  the rows do not divide into equal replays; see the trace")
        return
    one = ev[-(len(ev) // n):]
    t0, end = one[0]["ts"], None
    for e in one:
        gap = 0.0 if end is None else e["ts"] - end
        print(f"  +{e['ts'] - t0:9.2f} us  gap {gap:7.2f} us  dur {e['dur']:9.2f} us  {e['cat']:10s} {e['name'][:70]}")
        end = e["ts"] + e["dur"]
    print(f"  {len(one)} rows; first start to last end {end - t0:.2f} us; busy {sum(e['dur'] for e in one):.2f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=LIB", help="a build of libbydbgpu.so, relative to skywalking-banyandb_b200/; repeat to alternate builds")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--replays", type=int, default=2000)
    ap.add_argument("--block", type=int, default=100)
    ap.add_argument("--plain-steps", type=int, default=20)
    ap.add_argument("--series", type=int, default=10_000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--services", type=int, default=1000)
    ap.add_argument("--out", help="directory of the profiler traces (default: a fresh temporary directory, printed with the trace)")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write each library's last replayed result as DIR/NAME/<array>.npy (float64)")
    args = ap.parse_args()
    if args.replays < args.block or args.block < 1:
        ap.error("--replays must hold at least one --block")
    named = [tuple(s.split("=", 1)) if "=" in s else (os.path.splitext(os.path.basename(s))[0], s) for s in args.lib] or [("shipped", "libbydbgpu.so")]
    for name, rel in named:
        if not os.path.exists(os.path.join(PKG_DIR, rel)):
            sys.exit(f"{name}: {os.path.join(PKG_DIR, rel)} is missing")
    pkg0 = B.load_pkg()
    img = B.make_part(pkg0, args.series, args.points, 1)
    files = img.files()
    sids = np.arange(1, args.series + 1, dtype=np.uint64)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_step_stages.py times a CUDA graph replay on the GPU and has no CPU form: no CUDA device found")
    torch.cuda.set_device(0)
    print("card:", card_state(), flush=True)
    libs = []
    for name, rel in named:
        pkg = fresh_package(os.path.join(PKG_DIR, rel))
        ctx = pkg.Context(device=0)
        h = ctx.register_part(1, files)
        q = B.c3_query(pkg, [h], sids, args.services)
        libs.append({"name": name, "pkg": pkg, "capi": sys.modules[pkg.__name__ + ".capi"], "ctx": ctx, "h": h, "pq": ctx.prepare(q), "gq": ctx.prepare_graph(q),
                     "rounds": []})
    os.environ.pop("BYDB_GPU_LIB", None)
    for rnd in range(args.rounds):
        for lib in libs:
            m = one_round(lib, args)
            lib["rounds"].append(m)
            print(f"round {rnd} {lib['name']:10s} plain scan {m['plain_scan_ms']:.4f} device {m['plain_device_ms']:.4f} | replay wall min {m['wall_min']:.4f} "
                  f"median {m['wall_median']:.4f} p90 {m['wall_p90']:.4f} | device min {m['device_min']:.4f} median {m['device_median']:.4f} | "
                  f"host share {m['host_share']:.4f} | bare ctypes median {m['bare_median']:.4f} (wrapper share {m['wrapper_share']:.4f})  ms/step", flush=True)
    print(f"summary: median over {args.rounds} rounds [round-to-round spread = max - min], ms per step, {args.replays} replays in blocks of {args.block}")
    keys = ("plain_scan_ms", "plain_device_ms", "wall_median", "device_median", "host_share", "bare_median", "wrapper_share")
    for lib in libs:
        cells = []
        for k in keys:
            v = [m[k] for m in lib["rounds"]]
            cells.append(f"{k} {np.median(v):.4f} [{max(v) - min(v):.4f}]")
        print(f"  {lib['name']:10s} " + "  ".join(cells))
    first = libs[0]
    sig = lambda r: (r.group_id.tobytes(), r.rows.tobytes(), r.is_float.tobytes(), r.val_i64.tobytes(), r.val_f64.tobytes())  # noqa: E731
    for lib in libs[1:]:
        d = {k: float(np.median([m[k] for m in lib["rounds"]]) - np.median([m[k] for m in first["rounds"]])) for k in ("wall_median", "device_median", "bare_median")}
        wins = sum(b["wall_median"] < a["wall_median"] for a, b in zip(first["rounds"], lib["rounds"]))
        print(f"  {lib['name']} - {first['name']}: wall {d['wall_median']:+.4f}  device {d['device_median']:+.4f}  bare {d['bare_median']:+.4f} ms/step; "
              f"wall median lower in {wins} of {args.rounds} alternated pairs; result {'identical' if sig(lib['last']) == sig(first['last']) else 'DIFFERS'}")
    if args.dump_outputs:
        for lib in libs:
            B.dump_outputs(os.path.join(args.dump_outputs, lib["name"]), lib["last"])
    if not args.no_profile:
        out_dir = args.out or tempfile.mkdtemp(prefix="bydb_step_stages_")
        for lib in libs:
            profile_replay(torch, lib, out_dir)
    print("card:", card_state(), flush=True)
    for lib in libs:
        lib["gq"].close()
        lib["ctx"].release_part(lib["h"])
        lib["ctx"].close()


if __name__ == "__main__":
    main()

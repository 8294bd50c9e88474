"""Prepared map-phase answers (bydb_scan_partials_prepared / bydb_scan_partials_keyed_prepared, DESIGN.md 4.5 / 4.6).

A data node in a cluster answers the liaison's pushed-down aggregation with partial rows.  The prepared forms run the unprepared
sequence on their first execution, capture it as one CUDA graph on the second and replay it afterwards; the graph's last kernel
writes the zero pages, the control word and exactly the present rows into the handle's page-locked staging.  Every handle here
runs at least five times, and every execution must give what the unprepared form gives on the same context at that moment:
  - plain: bydb_scan_partials (with stats) into a table of the test's own, then bydb_partials_rows over it;
  - keyed: bydb_scan_partials_keyed;
rows, key values, Partial words bit for bit, the counters, the refusals.  Those unprepared answers are themselves pinned against
the oracle through the liaison's Combine (test_gpu_partials.py / test_gpu_keyed_partials.py), so every replay is too.  Replays
must also keep the stats contract of bydb_gpu.h: h2d_bytes 0, d2h_bytes = 256 V + 8 + 8 F + n_rows (8 + 16 A), and the stated
kernel_launches.
"""
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, build_part, grid, to_gpu_query
from tests.test_gpu_keyed import FAM, KT, build_keyed, limit_series, mk
from tests.test_gpu_keyed_partials import GID, node_parts
from tests.test_gpu_keyed_prepared import COUNTERS, refusal
from tests.test_gpu_masks import I64_MAX, I64_MIN
from tests.test_gpu_partials import B_AGGS, BOUNDARY, boundary_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUM, COUNT, MIN, MAX, MEAN = O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN
I, F = O.VT_INT64, O.VT_FLOAT64
FNS = (SUM, COUNT, MIN, MAX, MEAN)
RUNS = 5
ARRAYS = ("group_id", "is_float", "val_i64", "cnt_i64")
_pid = [12_400_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


def n_fields(q):
    return len(dict.fromkeys(f for f, _ in q.aggs))


def assert_same_rows(got, want, what, keyed=False):
    """partial rows against the unprepared answer: arrays exactly, floats as bit patterns, keys, the counters"""
    for k in ARRAYS:
        assert np.asarray(got[k]).tolist() == np.asarray(want[k]).tolist(), (what, k)
    for k in ("val_f64", "cnt_f64"):
        assert got[k].view(np.uint64).tolist() == want[k].view(np.uint64).tolist(), (what, k)
    if keyed:
        assert got["key"] == want["key"] and got["n_keys"] == want["n_keys"] and got["key_table"] == want["key_table"], what
    assert {k: getattr(got["stats"], k) for k in COUNTERS} == {k: getattr(want["stats"], k) for k in COUNTERS}, what


def replay_d2h(q, n_rows, V=1):
    return 256 * V + 8 + 8 * n_fields(q) + n_rows * (8 + 16 * len(q.aggs))


class Tables:
    """the unprepared plain form on a table the test owns (torch), on the current stream"""

    def __init__(self, ctx):
        import torch
        self.ctx, self.torch = ctx, torch
        self.stream = torch.cuda.current_stream().cuda_stream

    def rows(self, q):
        nb = self.ctx.partials_layout(q)["total_bytes"]
        t = self.torch.zeros(nb // 8, dtype=self.torch.int64, device="cuda")
        st = self.ctx.scan_partials(q, t.data_ptr(), nb, self.stream)
        out = dict(self.ctx.partials_rows(q, t.data_ptr(), nb, self.stream))
        out["stats"] = st
        return out


def run_plain(bydb, ctx, q, what, runs=RUNS, captured=True):
    """a plain handle `runs` times against the unprepared form; the first execution and the replays against the stats contract"""
    want = Tables(ctx).rows(q)
    g = ctx.prepare_graph(q)
    try:
        outs = [g.run_partials() for _ in range(runs)]
    finally:
        g.close()
    n = len(want["group_id"])
    for i, got in enumerate(outs):
        assert_same_rows(got, want, (what, i))
        s, w = got["stats"], want["stats"]
        if i == 0 or not captured:  # the unprepared path: bydb_scan_partials' stats, plus the three row kernels and their read-back
            assert s.kernel_launches == w.kernel_launches + 3 and s.h2d_bytes == w.h2d_bytes, (what, i, s)
            assert s.d2h_bytes == w.d2h_bytes + replay_d2h(q, n) - 256, (what, i, s.d2h_bytes)
        else:
            assert s.h2d_bytes == 0 and s.scan_kernel_ms == 0 and s.device_ms > 0, (what, i, s)
            assert s.kernel_launches == w.kernel_launches + 4, (what, i, s.kernel_launches, w.kernel_launches)
            assert s.d2h_bytes == replay_d2h(q, n), (what, i, s.d2h_bytes, replay_d2h(q, n))
    return want


def run_keyed(bydb, ctx, q, key, max_values, value_type, what, runs=RUNS):
    """a keyed handle `runs` times against bydb_scan_partials_keyed; replays against the stats contract"""
    want = ctx.scan_partials_keyed(q, FAM, key, max_values, value_type)
    g = ctx.prepare_keyed(q, FAM, key, max_values, value_type)
    try:
        outs = [g.run_partials() for _ in range(runs)]
    finally:
        g.release()
    for i, got in enumerate(outs):
        assert_same_rows(got, want, (what, i), keyed=True)
        s, w = got["stats"], want["stats"]
        if i == 0:
            assert (s.kernel_launches, s.h2d_bytes, s.d2h_bytes) == (w.kernel_launches, w.h2d_bytes, w.d2h_bytes), (what, s)
        elif want["n_keys"] > 0:
            assert s.h2d_bytes == 0 and s.scan_kernel_ms == 0 and s.device_ms > 0, (what, i, s)
            assert s.kernel_launches == w.kernel_launches, (what, i, s.kernel_launches, w.kernel_launches)
            d2h = replay_d2h(q, len(got["key"]), want["n_keys"])
            assert s.d2h_bytes == d2h, (what, i, s.d2h_bytes, d2h)
    return want


# ------------------------------------------------------------------ plain form: group counts and which groups appear
N_WIDE = 100_000


@pytest.fixture(scope="module")
def wide(bydb, gpu_ctx):
    """100 000 series of two rows each: series k can stand for group k, so every pattern of present groups is reachable"""
    rng = np.random.default_rng(17)
    sids, ts, ver = grid(N_WIDE, 2)
    part = build_part(sids, ts, ver, [("i", I, rng.integers(-(1 << 40), 1 << 40, sids.size), None),
                                      ("f", F, np.round(rng.normal(10, 4, sids.size), 3), None)])
    h = gpu_ctx.register_part(_next_pid(), part.files())
    yield h, np.unique(sids)
    gpu_ctx.release_part(h)


def patterns(G, usid):
    """(name, series ids, their groups): no group, the first, the last, all, every other"""
    one = usid[:1]
    half = (G + 1) // 2
    return [("none", np.array([10 ** 9], np.uint64), [0]), ("first", one, [0]), ("last", one, [G - 1]),
            ("all", usid[:G], np.arange(G)), ("every other", usid[:half], np.arange(half) * 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 32, 33, 1023, 1024, 1025, 8192, 8193, 100_000])
def test_plain_group_counts(bydb, gpu_ctx, wide, G):
    h, usid = wide
    for name, sids, groups in patterns(G, usid):
        q = bydb.Query([h], sids, [("i", SUM), ("f", MEAN)], series_group=np.asarray(groups, np.int32), n_groups=G)
        want = run_plain(bydb, gpu_ctx, q, (G, name))
        present = sorted(set(np.asarray(groups).tolist())) if name != "none" else []
        assert want["group_id"].tolist() == present, (G, name)


@pytest.mark.gpu
def test_plain_aggregation_widths(bydb, gpu_ctx, wide):
    """A = 1 and A = 32 (validate_query's limit), several fields, ROW_PATH_TYPES, Top-N ignored"""
    h, usid = wide
    sids = usid[:3000]
    grp = (np.arange(sids.size) % 700).astype(np.int32)
    a32 = [(("i", "f")[k % 2], FNS[k % 5]) for k in range(32)]
    for what, aggs, kw in (("A=1", [("f", COUNT)], {}), ("A=32", a32, {}), ("row path", [("f", COUNT), ("i", MEAN)], {"flags": 2}),
                           ("top ignored", [("i", MAX), ("f", MIN)], {"top_n": 5, "top_agg": 0, "top_desc": 1})):
        run_plain(bydb, gpu_ctx, bydb.Query([h], sids, aggs, series_group=grp, n_groups=700, **kw), what)


# ------------------------------------------------------------------ plain form: the edges of the encoding
# sums that wrap (int64) or overflow to +-Inf (float64) inside one part
WRAP = {16: [(0, [I64_MAX, I64_MAX, 3], [1e308, 1e308, -0.0])], 17: [(1, [I64_MIN, -1], [-1e308, -1e308])]}


@pytest.mark.gpu
def test_plain_boundaries(bydb, gpu_ctx):
    """test_gpu_partials' boundary groups one part at a time (INT64_MIN / MAX, sums that wrap, groups that met only nulls or
    never met the column, NaN / +-Inf / -0.0), int64 and float64 fields with MEAN counts; then all three parts together, which
    overlap in time: the unprepared path, answered alike"""
    with boundary_shards(bydb, gpu_ctx, cases={**BOUNDARY, **WRAP}) as sh:
        for r in range(len(sh.parts)):
            run_plain(bydb, gpu_ctx, sh.q(r, B_AGGS), f"rank {r}")
        run_plain(bydb, gpu_ctx, sh.q_whole(B_AGGS), "overlapping parts", captured=False)


def without_block(err):
    """(code, text) of a device error without the block it names: the first block to see the mix wins, which varies from one
    unprepared call to the next (the number is required to be there)"""
    head, sep, tail = str(err).rpartition(" (block/series #")
    assert sep and tail.endswith(")") and tail[:-1].isdigit(), str(err)
    return err.code, head


@pytest.mark.gpu
def test_plain_device_error_on_replay(bydb, gpu_ctx):
    """v is int64 in one part and float64 in a later, time-disjoint one: every execution (the replays too) fails with the
    unprepared call's code and text; the context answers a plain query afterwards"""
    s1, t1, v1 = grid(4, 50)
    s2, t2, v2 = grid(4, 50, sid0=5, t0=T0 + 10_000 * STEP)
    pa = build_part(s1, t1, v1, [("v", I, np.arange(s1.size, dtype=np.int64), None)])
    pb = build_part(s2, t2, v2, [("v", F, np.arange(s2.size) * 0.5, None)])
    ha, hb = gpu_ctx.register_part(_next_pid(), pa.files()), gpu_ctx.register_part(_next_pid(), pb.files())
    try:
        usid = np.arange(1, 9, dtype=np.uint64)
        q = bydb.Query([ha, hb], usid, [("v", SUM), ("v", MAX)], series_group=(np.arange(8) % 3).astype(np.int32), n_groups=3)
        with pytest.raises(bydb.BydbError) as pe:
            Tables(gpu_ctx).rows(q)
        g = gpu_ctx.prepare_graph(q)
        try:
            for run in range(RUNS):
                with pytest.raises(bydb.BydbError) as e:
                    g.run_partials()
                assert without_block(e.value) == without_block(pe.value), run
        finally:
            g.close()
        run_plain(bydb, gpu_ctx, bydb.Query([ha], usid[:4], [("v", SUM)]), "after the error")
    finally:
        gpu_ctx.release_part(ha)
        gpu_ctx.release_part(hb)


# ------------------------------------------------------------------ keyed form
@pytest.mark.gpu
@pytest.mark.parametrize("int64", [False, True], ids=["string", "int64"])
def test_keyed_node(bydb, gpu_ctx, int64):
    """test_gpu_keyed_partials' node (two time-disjoint parts, nil keys, null cells, a group that never met `i`), string and
    int64 keys, every aggregation of both fields; a cut, one group per series, and a query that selects no block (V = 0)"""
    parts = node_parts(int64)
    vt = bydb.VT_INT64 if int64 else 0
    handles = [gpu_ctx.register_part(_next_pid() + i, p.files()) for i, (p, _) in enumerate(parts)]
    try:
        aggs = [(f, fn) for f in ("i", "f") for fn in FNS]
        for what, gid, kw in (("all rows", GID, {}), ("cut", GID, {"tmin": T0 + 100 * STEP, "tmax": T0 + 20010 * STEP}),
                              ("one group per series", {1: 0, 2: 1, 3: 2, 4: 3}, {})):
            sids = np.array(sorted(gid), dtype=np.uint64)
            oq = O.Query([p for p, _ in parts], sids, aggs, groups=np.array([gid[int(s)] for s in sids], np.int32),
                         n_groups=max(gid.values()) + 1, **kw)
            want = run_keyed(bydb, gpu_ctx, to_gpu_query(bydb, handles, oq), KT, 256, vt, what)
            assert want["n_keys"] > 0 and len(want["key"]) > 0, what
        q0 = bydb.Query(handles, np.array([999], np.uint64), aggs)
        want = run_keyed(bydb, gpu_ctx, q0, KT, 256, vt, "V = 0")
        assert want["n_keys"] == 0 and len(want["key"]) == 0
    finally:
        for h in handles:
            gpu_ctx.release_part(h)


@pytest.mark.gpu
def test_keyed_one_and_256_values_over_many_groups(bydb, gpu_ctx):
    """V = 1; V = 256 over G = 5000 series groups (G x V above 2^20 composite groups, of which a few are present)"""
    ss = [mk(1, [b"k000"] * 50), mk(2, [b"k%03d" % (r % 256) for r in range(600)]), mk(3, [b"k%03d" % (r * 7 % 256) for r in range(300)])]
    h = gpu_ctx.register_part(_next_pid(), build_keyed(ss).files())
    try:
        aggs = [("i", SUM), ("f", MEAN), ("i", MAX)]
        want = run_keyed(bydb, gpu_ctx, bydb.Query([h], np.array([1], np.uint64), aggs), KT, 1, 0, "V = 1")
        assert want["n_keys"] == 1
        q = bydb.Query([h], np.array([1, 2, 3], np.uint64), aggs, series_group=np.array([4999, 7, 4999], np.int32), n_groups=5000)
        want = run_keyed(bydb, gpu_ctx, q, KT, 256, 0, "V = 256")
        assert want["n_keys"] == 256 and 256 * 5000 > 1 << 20
    finally:
        gpu_ctx.release_part(h)


@pytest.mark.gpu
def test_keyed_refusals(bydb, gpu_ctx):
    """bydb_scan_partials_keyed's refusals (the cap, max_values 257, a plain key page, 8 predicates, overlapping parts): the
    prepared form refuses alike at prepare or on every execution, and a plain answer follows each"""
    ss = limit_series()
    P, E = O.Pred, bydb.capi
    seven = [P(FAM, "c", O.OP_GE, -5), P(FAM, "c", O.OP_LE, 5), P(FAM, "c", O.OP_NE, 9), P(FAM, "c", O.OP_GT, -9),
             P(FAM, "c", O.OP_LT, 9), P(FAM, "c", O.OP_EQ, 1), P(FAM, "nope", O.OP_NE, b"x")]
    over = [mk(40, [b"a00", b"late"] * 20, row0=30)]
    over[0].tags["c"] = (np.ones(40, np.int64), np.zeros(40, bool))
    ha, hb = gpu_ctx.register_part(_next_pid(), build_keyed(ss).files()), gpu_ctx.register_part(_next_pid(), build_keyed(over, 2).files())
    try:
        def q(sids, preds=(), handles=(ha,)):
            return bydb.Query(list(handles), np.array(sids, np.uint64), [("i", SUM), ("f", MAX)],
                              preds=[bydb.Pred(p.family, p.tag, p.op, p.value) for p in preds])
        cases = [(E.ENOMEM, q([40, 41]), 0), (E.ENOMEM, q([41, 42]), 1), (E.EINVAL, q([40]), 257), (E.ENOTSUP, q([46]), 256),
                 (E.ENOTSUP, q([40], seven + [P(FAM, "c", O.OP_GE, 0)]), 256), (E.ENOTSUP, q([40], handles=(ha, hb)), 256)]
        for code, qq, mv in cases:
            with pytest.raises(bydb.BydbError) as pe:
                gpu_ctx.scan_partials_keyed(qq, FAM, KT, mv)
            assert pe.value.code == code, (code, pe.value)
            try:
                g = gpu_ctx.prepare_keyed(qq, FAM, KT, mv)
            except bydb.BydbError as e:
                assert refusal(e) == refusal(pe.value)
            else:
                try:
                    for run in range(RUNS):
                        with pytest.raises(bydb.BydbError) as e:
                            g.run_partials()
                        assert refusal(e.value) == refusal(pe.value), (code, run)
                finally:
                    g.release()
            run_keyed(bydb, gpu_ctx, q([40, 45]), KT, 256, 0, ("plain answer after", code))
    finally:
        gpu_ctx.release_part(ha)
        gpu_ctx.release_part(hb)


# ------------------------------------------------------------------ parts, forms and threads
@pytest.mark.gpu
def test_parts_change_between_executions(bydb, gpu_ctx):
    """another part coming and going leaves the step standing; the handle's own part released gives ENOENT on every execution,
    for both forms; the part id registered again is answered alike by new handles"""
    ss = [mk(1, [b"a", b"b"] * 30), mk(2, [b"b", None] * 30)]
    part = build_keyed(ss)
    pid = _next_pid()
    h = gpu_ctx.register_part(pid, part.files())
    usid, grp = np.array([1, 2], np.uint64), np.array([0, 1], np.int32)
    aggs = [("i", SUM), ("f", MEAN)]
    q = bydb.Query([h], usid, aggs, series_group=grp, n_groups=2)
    want, kwant = Tables(gpu_ctx).rows(q), gpu_ctx.scan_partials_keyed(q, FAM, KT, 16)
    g, k = gpu_ctx.prepare_graph(q), gpu_ctx.prepare_keyed(q, FAM, KT, 16)
    try:
        for run in range(3):
            assert_same_rows(g.run_partials(), want, run)
            assert_same_rows(k.run_partials(), kwant, run, keyed=True)
        h2 = gpu_ctx.register_part(_next_pid(), part.files())
        assert_same_rows(g.run_partials(), want, "after a registration")
        gpu_ctx.release_part(h2)
        assert_same_rows(k.run_partials(), kwant, "after a release of another part", keyed=True)
        gpu_ctx.release_part(h)
        for call in (g.run_partials, k.run_partials):
            for _ in range(2):
                with pytest.raises(bydb.BydbError) as e:
                    call()
                assert e.value.code == bydb.capi.ENOENT
    finally:
        g.close()
        k.release()
    h = gpu_ctx.register_part(pid, part.files())
    try:
        q = bydb.Query([h], usid, aggs, series_group=grp, n_groups=2)
        got = run_plain(bydb, gpu_ctx, q, "registered again")
        assert_same_rows(got, want, "registered again: the same answer")
        run_keyed(bydb, gpu_ctx, q, KT, 16, 0, "registered again")
    finally:
        gpu_ctx.release_part(h)


@pytest.mark.gpu
def test_forms_alternate_and_handles_run_concurrently(bydb, gpu_ctx):
    """finalised and partial executions alternating on one handle (each drops the other's step and captures its own), then
    several handles replayed from threads at once"""
    ss = [mk(1, [b"a", b"b", None] * 40), mk(2, [b"c", b"a"] * 50), mk(3, [b"b"] * 70)]
    h = gpu_ctx.register_part(_next_pid(), build_keyed(ss).files())
    try:
        usid, grp = np.array([1, 2, 3], np.uint64), np.array([0, 1, 0], np.int32)
        qa = bydb.Query([h], usid, [("i", SUM), ("f", MAX), ("i", MEAN)], series_group=grp, n_groups=2)
        qb = bydb.Query([h], usid[1:], [("f", SUM), ("i", COUNT)])
        wa, wfa = Tables(gpu_ctx).rows(qa), gpu_ctx.scan_agg(qa)
        ka, kfa = gpu_ctx.scan_partials_keyed(qa, FAM, KT, 64), gpu_ctx.scan_agg_keyed(qa, FAM, KT, 64)
        wb, kb = Tables(gpu_ctx).rows(qb), gpu_ctx.scan_partials_keyed(qb, FAM, KT, 64)
        ga, gk = gpu_ctx.prepare_graph(qa), gpu_ctx.prepare_keyed(qa, FAM, KT, 64)
        gb, gkb = gpu_ctx.prepare_graph(qb), gpu_ctx.prepare_keyed(qb, FAM, KT, 64)
        try:
            for rnd in range(6):
                assert_same_rows(ga.run_partials(), wa, ("plain partial", rnd))
                fin = ga.run()
                assert fin.group_id.tolist() == wfa.group_id.tolist() and fin.val_i64.tolist() == wfa.val_i64.tolist(), rnd
                assert fin.val_f64.view(np.uint64).tolist() == wfa.val_f64.view(np.uint64).tolist(), rnd
                assert_same_rows(gk.run_partials(), ka, ("keyed partial", rnd), keyed=True)
                kf = gk.run()
                assert kf.key == kfa.key and kf.val_i64.tolist() == kfa.val_i64.tolist(), rnd
                assert kf.val_f64.view(np.uint64).tolist() == kfa.val_f64.view(np.uint64).tolist(), rnd
            errors = []

            def worker(call, want, keyed, name):
                try:
                    for i in range(8):
                        assert_same_rows(call(), want, (name, i), keyed=keyed)
                except Exception as e:   # noqa: BLE001 -- reported by the main thread
                    errors.append(e)
            jobs = ((ga.run_partials, wa, False, "a"), (gb.run_partials, wb, False, "b"), (gk.run_partials, ka, True, "ka"),
                    (gkb.run_partials, kb, True, "kb"))
            ths = [threading.Thread(target=worker, args=j) for j in jobs]
            for t in ths:
                t.start()
            for _ in range(4):
                Tables(gpu_ctx).rows(qa)
            for t in ths:
                t.join()
            assert not errors, errors
        finally:
            for g in (ga, gb):
                g.close()
            for g in (gk, gkb):
                g.release()
    finally:
        gpu_ctx.release_part(h)


# ------------------------------------------------------------------ the cgo shim's way, from plain C
def _caller(tmp_path, bydb):
    cuda_lib = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "lib64")
    if shutil.which("gcc") is None or not os.path.exists(os.path.join(cuda_lib, "libcudart.so")):
        pytest.skip("no gcc / libcudart")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "partials_prepared_caller"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "partials_prepared_caller.c"), "-L", lib_dir, "-lbydbgpu",
                           "-L", cuda_lib, "-lcudart", "-Wl,-rpath," + lib_dir + ":" + cuda_lib])
    return exe


def test_c_caller_builds_against_the_header(tmp_path, bydb):
    out = subprocess.run([str(_caller(tmp_path, bydb))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr


@pytest.mark.gpu
def test_c_caller_on_the_device(tmp_path, bydb, gpu_ctx):
    out = subprocess.run([str(_caller(tmp_path, bydb))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
    assert "init refused" not in out.stdout and "plain run 5" in out.stdout and "keyed run 5" in out.stdout, out.stdout

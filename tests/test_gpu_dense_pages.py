"""Dense pages (DESIGN.md 3.3): a resident part's narrow delta field pages get a bit-plane form at registration, and the express
lane sums the planes instead of the varints.  Every answer must be the one the reference pages give, bit for bit: two contexts,
dense pages on and off, run the same queries on the same parts, and both are held against the oracle.  Pages that must keep their
varints sit in the same blocks as converted ones: a range of 2^32 or more, a 4-byte varint, values at the end of int64 whose
deltas wrap, and a random walk whose planes would not be smaller."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query

gpu = pytest.mark.gpu
FAM = "default"
FIELDS = ["lat", "ints", "range33", "wide4", "wrap", "walk"]


def _opposite(d):
    """the first two deltas of opposite signs keep the writer on the delta encoding"""
    d = d.copy()
    if d.size >= 2:
        d[0], d[1] = abs(d[0]) + 1, -(abs(d[1]) + 1)
    return d


def _series_values(rng, n):
    lat = np.round(25 + rng.normal(0, 5, n), 2)
    ints = rng.integers(0, 1000, n).astype(np.int64)
    # climbs over more than 2^32 in 3-byte steps
    range33 = np.concatenate([[0], np.cumsum(_opposite(950_000 + rng.integers(-5000, 5000, n - 1)))]).astype(np.int64)
    wide4 = rng.integers(0, 50, n).astype(np.int64)
    wide4[n // 2:] += 1 << 24                                  # one 4-byte varint in the middle
    top = np.iinfo(np.int64).max
    with np.errstate(over="ignore"):   # a prefix that wraps past INT64_MAX
        wrap = np.concatenate([[top - 30], top - 30 + np.cumsum(_opposite(rng.integers(1, 6, n - 1)))]).astype(np.int64)
    walk = np.concatenate([[0], np.cumsum(_opposite(rng.integers(-8000, 8001, n - 1)))]).astype(np.int64)
    return dict(lat=lat, ints=ints, range33=range33, wide4=wide4, wrap=wrap, walk=walk)


def make_part(seed, n_series=24, sid0=1, t0=T0):
    rng = np.random.default_rng(seed)
    lens = [9000 if s % 3 else 17000 for s in range(n_series)]
    lens[1] = 1                                                # a 1-row block
    sids = np.concatenate([np.full(L, sid0 + s, np.uint64) for s, L in enumerate(lens)])
    ts = np.concatenate([t0 + np.arange(L, dtype=np.int64) * STEP for L in lens])
    vals = [_series_values(rng, L) for L in lens]
    fields = []
    for f in FIELDS:
        v = np.concatenate([x[f] for x in vals])
        fields.append((f, O.VT_FLOAT64 if f == "lat" else O.VT_INT64, v, None))
    svc = [b"svc-%d" % (s % 4) for s, L in enumerate(lens) for _ in range(L)]
    part = build_part(sids, ts, np.ones(sids.size, np.int64), fields, [(FAM, [("svc", O.VT_STR, svc, None)])])
    return part, np.unique(sids)


@pytest.fixture(scope="module")
def pair(bydb):
    on, off = bydb.Context(device=0), bydb.Context(device=0, dense_pages=False)
    yield on, off
    on.close()
    off.close()


@pytest.fixture(scope="module")
def parts():
    # the second part follows the first in time (the express lane takes both), the third overlaps it (version dedup)
    return [make_part(5), make_part(6, n_series=10, sid0=100, t0=T0 + 20000 * STEP), make_part(7, n_series=6, sid0=3, t0=T0 + 3 * STEP)]


def same_result(a, b, ctx):
    assert a.group_id.tolist() == b.group_id.tolist(), ctx
    assert a.rows.tolist() == b.rows.tolist(), ctx
    assert a.val_i64.tolist() == b.val_i64.tolist(), ctx
    assert a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist(), ctx


def same_rows(a, b, ctx):
    for k, y in b.items():
        if k == "stats":
            continue
        x = a[k]
        if isinstance(y, np.ndarray):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), (ctx, k)
        else:
            assert x == y, (ctx, k)


def register(ctx, ps, pid0):
    return [ctx.register_part(pid0 + i, p.files()) for i, (p, _) in enumerate(ps)]


SUMS = [(f, fn) for f in FIELDS for fn in (O.AGG_SUM, O.AGG_COUNT, O.AGG_MEAN)]


@gpu
def test_dense_pages_admission_and_budget(bydb, pair, parts):
    on, off = pair
    p, _ = parts[0]
    h_on, h_off = on.register_part(1, p.files()), off.register_part(1, p.files())
    i_on, i_off = on.part_info(h_on), off.part_info(h_off)
    # lat and ints of every block of more than one row; nothing else qualifies
    assert i_on["dense_pages"] > 0 and i_off["dense_pages"] == 0 and i_off["dense_bytes"] == 0, (i_on, i_off)
    assert i_on["hbm_bytes"] == i_off["hbm_bytes"] + i_on["dense_bytes"], (i_on, i_off)
    on.release_part(h_on)
    off.release_part(h_off)
    with bydb.Context(device=0, hbm_budget_bytes=i_on["hbm_bytes"] - 1) as tight:
        with pytest.raises(bydb.BydbError) as ei:
            tight.register_part(1, p.files())
        assert ei.value.code == bydb.capi.ENOMEM
    with bydb.Context(device=0, hbm_budget_bytes=i_off["hbm_bytes"], dense_pages=False) as tight:
        tight.release_part(tight.register_part(1, p.files()))


@gpu
@pytest.mark.parametrize("shape", ["all", "groups", "top", "two_parts", "overlapping_parts", "cut_minmax"])
def test_dense_pages_answer_like_the_reference_pages(bydb, pair, parts, shape):
    on, off = pair
    ps = {"two_parts": parts[:2], "overlapping_parts": parts[::2]}.get(shape, parts[:1])
    sids = np.unique(np.concatenate([s for _, s in ps]))
    aggs, kw = SUMS, {}
    if shape in ("groups", "two_parts", "overlapping_parts"):
        kw = dict(groups=(np.arange(sids.size) % 5).astype(np.int32), n_groups=5)
    if shape == "top":
        kw = dict(groups=np.arange(sids.size, dtype=np.int32), n_groups=sids.size, top_n=7, top_agg=0, top_desc=True)
    if shape == "cut_minmax":
        aggs = [(f, fn) for f in FIELDS for fn in (O.AGG_SUM, O.AGG_MIN, O.AGG_MAX)]
        kw = dict(tmin=T0 + 100 * STEP, tmax=T0 + 12000 * STEP)
    oq = O.Query([p for p, _ in ps], sids, aggs, **kw)
    h_on, h_off = register(on, ps, 10), register(off, ps, 10)
    try:
        r_on, r_off = on.scan_agg(to_gpu_query(bydb, h_on, oq)), off.scan_agg(to_gpu_query(bydb, h_off, oq))
    finally:
        for h in h_on:
            on.release_part(h)
        for h in h_off:
            off.release_part(h)
    same_result(r_on, r_off, shape)
    assert_parity(r_on, O.run_query(oq), aggs, shape)
    s_on, s_off = r_on.stats, r_off.stats
    assert s_on.rows_scanned == s_off.rows_scanned and s_on.blocks_express_lane == s_off.blocks_express_lane, shape
    if shape not in ("cut_minmax", "overlapping_parts"):
        assert s_on.blocks_express_lane > 0 and s_on.page_bytes == s_off.page_bytes, (s_on, s_off)


@gpu
def test_dense_pages_prepared_graph_and_partials(bydb, pair, parts):
    on, off = pair
    p, sids = parts[0]
    oq = O.Query([p], sids, SUMS, groups=(np.arange(sids.size) % 3).astype(np.int32), n_groups=3)
    want = O.run_query(oq)
    for rnd in range(2):   # the second round registers the part again after its release
        h_on, h_off = on.register_part(20, p.files()), off.register_part(20, p.files())
        q_on, q_off = to_gpu_query(bydb, [h_on], oq), to_gpu_query(bydb, [h_off], oq)
        g_on, g_off = on.prepare_graph(q_on), off.prepare_graph(q_off)
        for _ in range(4):   # graph replay from the third run on
            r_on, r_off = g_on.run(), g_off.run()
            same_result(r_on, r_off, f"graph round {rnd}")
            assert_parity(r_on, want, SUMS, f"graph round {rnd}")
        same_rows(g_on.run_partials(), g_off.run_partials(), "partials")
        same_rows(on.scan_partials_keyed(q_on, FAM, "svc"), off.scan_partials_keyed(q_off, FAM, "svc"), "keyed partials")
        same_result(on.scan_agg_keyed(q_on, FAM, "svc"), off.scan_agg_keyed(q_off, FAM, "svc"), "keyed")
        g_on.close()
        g_off.close()
        on.release_part(h_on)
        off.release_part(h_off)

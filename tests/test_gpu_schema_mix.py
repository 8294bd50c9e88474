"""Queries over parts whose blocks carry different schemas (tests/schema_mix.py), on the device.

A part holds the series of several measures; neighbouring blocks differ in tag families, tags, fields, column count and
sometimes in the value type of one field name.  The block index decoders (index_walk_kernel on the device, part_dir.cc on the
host) resolve names through a positional cache that once matched a tag by position and bytes only: `storage-only/entity_id`
after a block of `default/entity_id` took the latter's id, so predicates and group keys on it saw the wrong column or none.

Every query is checked
  - against the oracle on the mixed part (assert_parity; rows_matched);
  - through scan_agg on a default context and on a host_index context, a prepared graph (capture and replays), and
    scan_agg_host over pageable (gathered: plan_gather rewrites each block's column list) and pinned images;
  - when its series belong to one measure: against the device over that measure's own single-schema part, built from the
    same rows.  Those are the same blocks in the same order, so everything is bit-identical, float SUM / MEAN included, and
    rows_scanned / blocks_scanned equal.
Directories are compared between the two contexts for every part: DevBlock equal, DevCol offsets, sizes and value types
equal, name ids and file ids equal up to one consistent relabelling, and one id per (family, name).
"""
import dataclasses
import itertools

import numpy as np
import pytest

from oracle import oracle as O
from tests import schema_mix as M
from tests.helpers import assert_parity, to_gpu_query
from tests.test_gpu_masks import host_images

gpu = pytest.mark.gpu

SUM, COUNT, MIN, MAX, MEAN = O.AGG_SUM, O.AGG_COUNT, O.AGG_MIN, O.AGG_MAX, O.AGG_MEAN
EINVAL, ENOTSUP = -22, -95
_pid = [900_000]


def _next_pid():
    _pid[0] += 100
    return _pid[0]


@pytest.fixture(scope="module")
def ctxs(bydb):
    """a default context (block index walked on the device) and a host_index one (part_dir.cc); their own name tables"""
    dev, host = bydb.Context(device=0), bydb.Context(device=0, host_index=True)
    yield {"device": dev, "host_index": host}
    dev.close()
    host.close()


def same_bits(a, b, what, stats=True):
    assert a.group_id.tolist() == b.group_id.tolist() and a.rows.tolist() == b.rows.tolist(), f"{what}: groups / rows"
    assert a.is_float.tolist() == b.is_float.tolist(), f"{what}: output types"
    assert a.val_i64.tolist() == b.val_i64.tolist(), f"{what}: int64 values"
    assert a.val_f64.view(np.uint64).tolist() == b.val_f64.view(np.uint64).tolist(), f"{what}: float64 values, bit for bit"
    assert (a.key or []) == (b.key or []), f"{what}: keys"
    if stats:
        for s in ("rows_scanned", "rows_matched", "blocks_scanned"):
            assert getattr(a.stats, s) == getattr(b.stats, s), f"{what}: {s} {getattr(a.stats, s)} vs {getattr(b.stats, s)}"


def directories_match(bydb, ctxs, hd, hh, files, ctx):
    """device index vs host index of one part (see the module docstring); returns the device directory's columns"""
    bd, cd = ctxs["device"].part_directory(hd)
    bh, ch = ctxs["host_index"].part_directory(hh)
    assert bd.shape == bh.shape and (bd == bh).all(), f"{ctx}: DevBlock[] differs"
    assert cd.shape == ch.shape, f"{ctx}: column count"
    dcol = np.dtype([("off", "<u8"), ("size", "<u4"), ("name", "<u2"), ("vt", "u1"), ("file", "u1")])
    d, h = cd.view(dcol).ravel(), ch.view(dcol).ravel()
    for f in ("off", "size", "vt"):
        assert (d[f] == h[f]).all(), f"{ctx}: DevCol.{f} differs"
    for f in ("name", "file"):
        pairs = set(zip(d[f].tolist(), h[f].tolist()))
        assert len(pairs) == len({p[0] for p in pairs}) == len({p[1] for p in pairs}), f"{ctx}: {f} ids are not one relabelling"
    # one id per (family, name), different pairs never share one: the assertion the family-blind cache failed
    keys = [k for b in M.block_schemas(files) for k, _ in b["cols"]]
    assert len(keys) == d.size
    for label, col in (("device", d), ("host_index", h)):
        by_key = {}
        for k, i in zip(keys, col["name"].tolist()):
            by_key.setdefault(k, set()).add(i)
        assert all(len(v) == 1 for v in by_key.values()), f"{ctx}/{label}: a name under several ids"
        ids = [next(iter(v)) for v in by_key.values()]
        assert len(set(ids)) == len(ids), f"{ctx}/{label}: two names share an id"


class Mix:
    """a mixed part registered on both contexts, and each measure's own part on the default one"""

    def __init__(self, bydb, ctxs, measures, ctx):
        self.bydb, self.ctxs, self.ms = bydb, ctxs, measures
        self.part = M.mixed(measures)
        self.files = self.part.files()
        pid = _next_pid()
        self.h = {name: c.register_part(pid, self.files) for name, c in ctxs.items()}
        self.own = {}
        for k, m in enumerate(measures):
            p = m.own_part()
            self.own[m.label] = (p, ctxs["device"].register_part(pid + 1 + k, p.files()))
        directories_match(bydb, ctxs, self.h["device"], self.h["host_index"], self.files, ctx)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for name, c in self.ctxs.items():
            c.release_part(self.h[name])
        for _, h in self.own.values():
            self.ctxs["device"].release_part(h)

    def measure(self, label):
        return next(m for m in self.ms if m.label == label)

    def oquery(self, sids, aggs, preds=(), top=None, groups=None):
        sids = np.asarray(sorted(int(s) for s in sids), np.uint64)
        groups = (sids % 3).astype(np.int32) if groups is None else np.asarray(groups, np.int32)
        tn, ta, td = top or (0, 0, True)
        return O.Query([self.part], sids, list(aggs), groups=groups, n_groups=int(groups.max()) + 1, preds=list(preds),
                       top_n=tn, top_agg=ta, top_desc=td)

    def check(self, sids, aggs, preds=(), top=None, groups=None, own=None, ctx=""):
        """one query through every entry point; own: the label of the measure that holds all of `sids`"""
        oq = self.oquery(sids, aggs, preds, top, groups)
        want = O.run_query(oq)
        ctx = f"{ctx}/{[(f, fn) for f, fn in aggs]}/{[(p.family, p.tag, p.op, p.value) for p in preds]}/top{top}"
        got = {name: c.scan_agg(to_gpu_query(self.bydb, [self.h[name]], oq)) for name, c in self.ctxs.items()}
        g = self.ctxs["device"].prepare_graph(to_gpu_query(self.bydb, [self.h["device"]], oq))
        try:
            for run in range(3):
                got[f"graph{run}"] = g.run()
        finally:
            g.close()
        for pinned in (False, True):
            q = to_gpu_query(self.bydb, [], oq)
            q.flags = self.bydb.capi.Q_HOST_ZERO_COPY if pinned else 0
            got["pinned" if pinned else "pageable"] = self.ctxs["device"].scan_agg_host(host_images([self.part], pinned), q)
        for name, r in got.items():
            assert_parity(r, want, aggs, f"{ctx}/{name}")
            assert r.stats.rows_matched == want.rows_matched, f"{ctx}/{name}: rows_matched {r.stats.rows_matched} vs {want.rows_matched}"
        for name in ("host_index", "graph0", "graph1", "graph2"):
            same_bits(got[name], got["device"], f"{ctx}/{name} vs device", stats=not name.startswith("graph"))
        if own is not None:
            ref = self.ctxs["device"].scan_agg(to_gpu_query(self.bydb, [self.own[own][1]], oq))
            same_bits(got["device"], ref, f"{ctx}: mixed part vs {own}'s own part")
        return got["device"]

    def keyed(self, sids, aggs, family, tag, preds=(), own=None, ctx=""):
        """GROUP BY a stored string tag: the oracle's group_key, both contexts, and the own part"""
        oq = self.oquery(sids, aggs, preds)
        want = O.run_query(dataclasses.replace(oq, group_key=(family, tag)))
        ctx = f"{ctx}/key {family}/{tag}"
        got = {}
        for name, c in self.ctxs.items():
            got[name] = c.scan_agg_keyed(to_gpu_query(self.bydb, [self.h[name]], oq), family, tag, 0)
            assert_parity(got[name], want, aggs, f"{ctx}/{name}")
            assert got[name].key == want.key, f"{ctx}/{name}: keys {got[name].key[:6]} vs {want.key[:6]}"
        same_bits(got["host_index"], got["device"], f"{ctx}: host_index vs device")
        if own is not None:
            ref = self.ctxs["device"].scan_agg_keyed(to_gpu_query(self.bydb, [self.own[own][1]], oq), family, tag, 0)
            same_bits(got["device"], ref, f"{ctx}: mixed part vs {own}'s own part")
        return got["device"], want

    def keyed64(self, sids, aggs, family, tag, own=None, ctx=""):
        """GROUP BY a stored int64 tag: per key value v the rows and values of the oracle under the predicate tag == v"""
        oq = self.oquery(sids, aggs)
        vt = self.bydb.capi.VT_INT64
        got = {name: c.scan_agg_keyed(to_gpu_query(self.bydb, [self.h[name]], oq), family, tag, 0, vt) for name, c in self.ctxs.items()}
        same_bits(got["host_index"], got["device"], f"{ctx}: int64 key, host_index vs device")
        r = got["device"]
        for v in sorted({int.from_bytes(k, "little", signed=True) for k in r.key} - {0}):
            want = O.run_query(dataclasses.replace(oq, preds=[O.Pred(family, tag, O.OP_EQ, v)]))
            mine = {int(r.group_id[i]): (int(r.rows[i]), r.val_i64[i].tolist()) for i, k in enumerate(r.key)
                    if int.from_bytes(k, "little", signed=True) == v}
            theirs = {int(g): (int(n), want.val_i64[j].tolist()) for j, (g, n) in enumerate(zip(want.group_id, want.rows))}
            assert mine == theirs, f"{ctx}: key {v}: {mine} vs the oracle under {tag} == {v}: {theirs}"
        if own is not None:
            ref = self.ctxs["device"].scan_agg_keyed(to_gpu_query(self.bydb, [self.own[own][1]], oq), family, tag, 0, vt)
            same_bits(r, ref, f"{ctx}: int64 key, mixed part vs {own}'s own part")


def str_tags(m):
    return [(fam, t) for fam, tags in m.families for t, vt in tags if vt == M.S]


AGGS_I = [("i", SUM), ("i", COUNT), ("i", MIN), ("i", MAX), ("i", MEAN)]


@gpu
@pytest.mark.parametrize("name", ["fam_ab", "fam_ba", "moved", "frames"])
def test_same_tag_name_in_other_families_and_positions(bydb, ctxs, name):
    """a predicate and a GROUP BY on each family's tag, over its own measure and over series of every measure"""
    ms = M.collision_cases()[name]
    everyone = [s for m in ms for s in m.sids.tolist()]
    aggs = AGGS_I + ([("f", SUM), ("f", MAX)] if name != "frames" else [])
    with Mix(bydb, ctxs, ms, name) as x:
        for m in ms:
            mine = m.sids.tolist() if name != "frames" else m.sids.tolist()[:300]
            for fam, tag in str_tags(m):
                lit = f"{m.label}-1".encode()
                for op in (O.OP_EQ, O.OP_NE):
                    pred = [O.Pred(fam, tag, op, lit)]
                    x.check(mine, AGGS_I, pred, own=m.label, ctx=f"{name}/{m.label}")
                    x.check(everyone, aggs, pred, ctx=f"{name}/all")
                x.keyed(mine, AGGS_I, fam, tag, own=m.label, ctx=f"{name}/{m.label}")
                x.keyed(everyone, [("i", SUM), ("i", COUNT)], fam, tag, ctx=f"{name}/all")
        x.check(everyone, aggs, ctx=f"{name}/all, no predicate")


@gpu
def test_blocks_with_and_without_a_family(bydb, ctxs):
    """families [a, b], [b], [] and [a]: a predicate on a family some selected blocks lack (nil: EQ fails, NE passes)"""
    ms = M.family_cases()
    everyone = [s for m in ms for s in m.sids.tolist()]
    with Mix(bydb, ctxs, ms, "families") as x:
        for op in (O.OP_EQ, O.OP_NE, O.OP_GE):
            x.check(everyone, AGGS_I, [O.Pred("a", "x", op, b"ab-1")], ctx="families/a.x")
            x.check(everyone, AGGS_I, [O.Pred("b", "y", op, 0)], ctx="families/b.y")
        x.check(everyone, AGGS_I, [O.Pred("a", "x", O.OP_NE, b"a-0"), O.Pred("b", "y", O.OP_LT, 500)], ctx="families/a.x and b.y")
        for m in ms:
            x.check(m.sids, AGGS_I, [O.Pred("a", "x", O.OP_NE, b"zz")], own=m.label, ctx=f"families/{m.label}")
        x.keyed(everyone, [("i", SUM), ("i", COUNT)], "a", "x", ctx="families/all")
        x.keyed64(everyone, [("i", SUM), ("i", COUNT)], "b", "y", ctx="families/all")
        x.keyed64(x.measure("b").sids, [("i", SUM), ("i", COUNT)], "b", "y", own="b", ctx="families/b")


@gpu
def test_sixteen_families_in_a_block_and_seventeen_refused(bydb, ctxs):
    ms = M.many_families(16)
    everyone = [s for m in ms for s in m.sids.tolist()]
    with Mix(bydb, ctxs, ms, "16 families") as x:
        for k in (0, 7, 15):
            x.check(everyone, AGGS_I, [O.Pred(f"fam{k:02d}", "t", O.OP_EQ, b"wide-2")], ctx=f"16 families/fam{k:02d}")
        x.keyed(everyone, [("i", COUNT)], "fam15", "t", ctx="16 families")
        files17 = M.mixed(M.many_families(17)).files()
        for name, c in ctxs.items():
            with pytest.raises(bydb.BydbError) as e:
                c.register_part(_next_pid(), files17)
            assert e.value.code == ENOTSUP, f"{name}: 17 families in a block: {e.value.code} {e.value.msg}"
        with pytest.raises(bydb.BydbError) as e:
            ctxs["device"].scan_agg_host([files17], bydb.Query([], x.measure("wide").sids, [("i", SUM)]))
        assert e.value.code == ENOTSUP
        # the contexts still answer after the refusals
        x.check(everyone, AGGS_I, [O.Pred("fam00", "t", O.OP_NE, b"one-0")], ctx="16 families, after the refusal")


@gpu
def test_fields_per_block_and_the_met_column_rule(bydb, ctxs):
    """i in f1 only, j in f2 and f3, f in f1 and f2: groups of series that never met a column keep MIN / MAX at zero and are
    null to Top-N (DESIGN 4.3)"""
    ms = M.field_cases()
    everyone = np.asarray(sorted(s for m in ms for s in m.sids.tolist()), np.uint64)
    per_series = np.arange(everyone.size, dtype=np.int32)
    aggs = [("i", MIN), ("i", MAX), ("i", COUNT), ("j", SUM), ("j", MIN), ("f", MIN), ("f", MAX), ("f", SUM)]
    with Mix(bydb, ctxs, ms, "fields") as x:
        x.check(everyone, aggs, groups=per_series, ctx="fields/per series")
        x.check(everyone, aggs, ctx="fields/mod 3")
        x.check(everyone, aggs, [O.Pred("default", "region", O.OP_NE, b"f2-0")], ctx="fields/pred")
        for top in ((3, 1, True), (3, 1, False), (5, 4, True), (4, 6, False)):
            x.check(everyone, aggs, groups=per_series, top=top, ctx="fields/top")
        for m in ms:
            x.check(m.sids, [(f, fn) for f, _ in m.fields for fn in (SUM, MIN, MAX)], own=m.label, ctx=f"fields/{m.label}")


@gpu
def test_one_field_name_int64_in_one_measure_float64_in_another(bydb, ctxs):
    ms = M.type_mix_cases()
    with Mix(bydb, ctxs, ms, "type mix") as x:
        for m in ms:
            r = x.check(m.sids, [("v", SUM), ("v", COUNT)], groups=np.zeros(m.sids.size), own=m.label, ctx=f"type mix/{m.label}")
            if m.label == "vi":
                assert r.stats.blocks_express_lane > 0, "an all-rows int64 SUM takes the express lane"
            x.check(m.sids, [("v", MIN), ("v", MAX), ("v", MEAN)], own=m.label, ctx=f"type mix/{m.label}")
        everyone = [s for m in ms for s in m.sids.tolist()]
        for name, c in ctxs.items():
            for aggs in ([("v", SUM), ("v", COUNT)], [("v", MAX)]):
                with pytest.raises(bydb.BydbError) as e:
                    c.scan_agg(to_gpu_query(bydb, [x.h[name]], x.oquery(everyone, aggs, groups=np.zeros(len(everyone)))))
                assert e.value.code == EINVAL, f"{name}: {e.value.code} {e.value.msg}"


@gpu
def test_wide_blocks(bydb, ctxs):
    """65 columns: field q and tag w/k at column positions 0, 31, 32, 33, 63 and 64 (find_col's 32-column windows, the express
    lane's serial column walk); tag names past the positional cache change from block to block"""
    ms = M.wide_cases()
    everyone = [s for m in ms for s in m.sids.tolist()]
    aggs = [("q", SUM), ("q", COUNT), ("q", MIN), ("q", MAX)]
    with Mix(bydb, ctxs, ms, "wide") as x:
        x.check(everyone, aggs, ctx="wide/all")
        x.check(everyone, aggs, [O.Pred("w", "k", O.OP_NE, b"w0-1")], ctx="wide/all")
        x.keyed(everyone, [("q", SUM), ("q", COUNT)], "w", "k", ctx="wide/all")
        for m, (pf, pt) in zip(ms, M.WIDE_POS):
            if pf is not None:
                x.check(m.sids, [("q", SUM), ("q", COUNT)], groups=np.zeros(m.sids.size), own=m.label, ctx=f"wide/{m.label} express")
            if pt is not None and pf is not None:
                x.check(m.sids, aggs, [O.Pred("w", "k", O.OP_EQ, f"{m.label}-2".encode())], own=m.label, ctx=f"wide/{m.label}")
                x.keyed(m.sids, aggs, "w", "k", own=m.label, ctx=f"wide/{m.label}")
            last = [t for t, _ in dict(m.families).get("w", [])][-1:]
            for t in last:   # a tag far past the 24-slot cache, named after its measure
                x.check(everyone, aggs, [O.Pred("w", t, O.OP_EQ, f"{m.label}-0".encode())], ctx=f"wide/{m.label}/{t}")


@gpu
def test_long_column_names(bydb, ctxs):
    """names of 1, 60, 61 and 127 bytes: past 60 the device walker's table cannot hold them and the part's directory comes
    from the host parser, transparently"""
    ms = M.long_name_cases()
    everyone = [s for m in ms for s in m.sids.tolist()]
    with Mix(bydb, ctxs, ms, "long names") as x:
        for n, m in zip(M.NAME_LENS, ms):
            f, k = "f" * n, "k" * n
            x.check(m.sids, [(f, SUM), (f, MAX), ("i", COUNT)], [O.Pred("default", k, O.OP_NE, f"{m.label}-0".encode())], own=m.label,
                    ctx=f"names/{n}")
            x.check(everyone, [(f, SUM), (f, MIN), ("i", SUM)], [O.Pred("default", k, O.OP_EQ, f"{m.label}-1".encode())], ctx=f"names/{n}/all")
            x.keyed(everyone, [("i", SUM), ("i", COUNT)], "default", k, ctx=f"names/{n}/all")


@gpu
@pytest.mark.parametrize("total", [1024, 1025])
def test_distinct_names_at_the_device_table_size(bydb, ctxs, total):
    """1024 distinct names fill the device walker's table; the 1025th sends the part to the host parser"""
    ms = M.many_names(total)
    assert len(M.distinct_names(ms)) == total
    everyone = [s for m in ms for s in m.sids.tolist()]
    with Mix(bydb, ctxs, ms, f"{total} names") as x:
        x.check(everyone, AGGS_I, [O.Pred("default", "k", O.OP_NE, b"x0-0")], ctx=f"{total} names")
        last = ms[-1]
        f = last.fields[-1][0]
        x.check(last.sids, [(f, SUM), (f, MAX)], own=last.label, ctx=f"{total} names/{f}")
        x.keyed(everyone, [("i", COUNT)], "default", "k", ctx=f"{total} names")

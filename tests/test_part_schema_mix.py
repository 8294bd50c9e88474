"""The block index of parts whose blocks carry different schemas, parsed on the host (part_dir.cc), without a GPU.

A part holds the series of several measures, and each block carries its own measure's tag families and fields
(tests/schema_mix.py).  Both index decoders resolve a column's name through a positional cache before interning it; a cache
hit that ignored the family gave a block of family `storage-only` the id of `default`'s tag at the same position.  Here the
directory of tests/native/part_dir_dump.cc (compiled with g++ against the product's part_dir.cc) is checked column by column
against what each block's metadata records.  What the GPU suite (test_gpu_schema_mix.py) rests on is checked here too: which
blocks carry which families and fields, that the collision pattern crosses primary frames (walkers), and that each measure's
rows in the mixed part are those of its own single-schema part.
"""
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests import schema_mix as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "skywalking-banyandb_b200", "csrc")
ENOTSUP = -95


@functools.lru_cache(maxsize=None)
def cases():
    out = dict(M.collision_cases())
    out.update(families=M.family_cases(), fam16=M.many_families(16), fields=M.field_cases(), type_mix=M.type_mix_cases(),
               wide=M.wide_cases(), long_names=M.long_name_cases(), names1024=M.many_names(1024), names1025=M.many_names(1025))
    return out


@functools.lru_cache(maxsize=None)
def part_of(name):
    return M.mixed(cases()[name])


CASES = ["fam_ab", "fam_ba", "moved", "frames", "families", "fam16", "fields", "type_mix", "wide", "long_names", "names1024", "names1025"]


@pytest.fixture(scope="module")
def dump_exe(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = tmp_path_factory.mktemp("dump") / "part_dir_dump"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", str(exe), os.path.join(ROOT, "tests", "native", "part_dir_dump.cc"),
                           os.path.join(CSRC, "part_dir.cc"), "-ldl", "-lpthread"])
    return str(exe)


def host_dump(exe, tmp_path, files, keys):
    d = tmp_path / "part"
    d.mkdir()
    for k, v in files.items():
        (d / k).write_bytes(v)
    out = subprocess.run([exe, str(d)], input="".join(k + "\n" for k in keys), capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    res = dict(rc=None, files=[], blocks=[], find={}, sliced=None)
    for line in out.stdout.splitlines():
        tag, _, rest = line.partition(" ")
        if tag == "RC":
            res["rc"] = int(rest.split(" ", 1)[0])
        elif tag == "FILES":
            res["files"] = rest.split()
        elif tag == "B":
            sid, count, _ = map(int, rest.split())
            res["blocks"].append(dict(sid=sid, count=count, cols=[]))
        elif tag == "C":
            res["blocks"][-1]["cols"].append(tuple(map(int, rest.split())))
        elif tag == "K":
            i, _, key = rest.partition(" ")
            res["find"][key] = int(i)
        elif tag == "SLICED":
            res["sliced"] = int(rest)
    return res


def owner(measures):
    return {int(s): m for m in measures for s in m.sids.tolist()}


@pytest.mark.parametrize("name", CASES)
def test_blocks_carry_their_measures_schema(name):
    """each block's metadata lists its own measure's fields and families, blocks in series order, .tf / .tfm shared by name"""
    ms, files = cases()[name], part_of(name).files()
    own = owner(ms)
    blocks = M.block_schemas(files)
    assert [b["sid"] for b in blocks] == sorted(own), f"{name}: one block per series, in series order"
    for b in blocks:
        m = own[b["sid"]]
        assert b["cols"] == m.expected_cols(), f"{name}: series {b['sid']} of {m.label}"
        assert b["count"] == m.sid.size // m.sids.size
    fams = {f for m in ms for f, _ in m.families}
    assert set(files) == {"meta.bin", "primary.bin", "timestamps.bin", "fv.bin"} | {f + ext for f in fams for ext in (".tf", ".tfm")}
    schemas = {tuple(b["cols"]) for b in blocks}
    assert len(schemas) == len(ms), f"{name}: every measure's schema appears"
    if name in ("fam_ab", "fam_ba"):
        first = [k for k, _ in blocks[0]["cols"] if k.startswith("t:")][0]
        assert first ==("t:default/entity_id" if name == "fam_ab" else "t:storage-only/entity_id")


def test_collision_pattern_crosses_primary_frames():
    files = part_of("frames").files()
    frames = M.primary_frames(files)
    assert len(frames) >= 2, "several primary frames: the index walkers each start with an empty cache"
    blocks = M.block_schemas(files)
    for f in range(len(frames)):
        fams = {c[0].split("/")[0] for b in blocks if b["frame"] == f for c in b["cols"] if c[0].startswith("t:")}
        assert fams == {"t:default", "t:storage-only"}, f"frame {f}: both families alternate inside the frame"
    assert [s for s, *_ in frames] == sorted(s for s, *_ in frames)


@pytest.mark.parametrize("name", ["fam_ab", "fam_ba", "moved", "families", "fields", "type_mix", "wide", "long_names"])
def test_each_measures_rows_equal_its_own_part(name):
    """through the oracle's reader: a measure's rows in the mixed part are the rows of its own single-schema part"""
    mixed = part_of(name)
    for m in cases()[name]:
        own = m.own_part()
        for fname, _ in m.fields:
            q = lambda p: O.Query([p], m.sids, [(fname, O.AGG_SUM)])   # noqa: E731
            a, b = O.scan_rows(q(mixed)), O.scan_rows(q(own))
            assert a["sid"].tolist() == b["sid"].tolist() and a["ts"].tolist() == b["ts"].tolist(), f"{name}/{m.label}/{fname}"
            (_, fa, va, na), (_, fb, vb, nb) = a["fields"][0], b["fields"][0]
            assert fa == fb and na.tolist() == nb.tolist() and va.view(np.uint64).tolist() == vb.view(np.uint64).tolist(), f"{name}/{m.label}/{fname}"
        if m.fields:
            r_mixed = O.run_query(O.Query([mixed], m.sids, [(m.fields[0][0], O.AGG_COUNT)]))
            assert r_mixed.rows.tolist() == [m.sid.size]


def test_one_builder_is_the_single_schema_part_and_shared_series_are_refused():
    m = cases()["fam_ab"][0]
    assert O.build_mixed_part([m.rows()]).files() == m.own_part().files(), "one builder: byte-identical to PartBuilder.finish"
    b = cases()["fam_ab"][1]
    clash = M.Measure("c", [int(b.sids[2])], 3, *M.A, seed=99)
    with pytest.raises(ValueError, match="more than one builder"):
        M.mixed([cases()["fam_ab"][0], b, clash])


@pytest.mark.parametrize("name", CASES)
def test_host_parser_resolves_each_column_to_its_own_name(dump_exe, tmp_path, name):
    """every column's name id is the id of the name its block records: field, or family and tag.  The positional cache used
    to hand `storage-only/entity_id` the id of `default/entity_id` whenever a block of the other family preceded it."""
    ms, files = cases()[name], part_of(name).files()
    expect = M.block_schemas(files)
    keys = sorted(M.distinct_names(ms))
    got = host_dump(dump_exe, tmp_path, files, keys)
    assert got["rc"] == 0
    missing = [k for k in keys if got["find"][k] == 0]
    assert not missing, f"{name}: names never interned: {missing[:4]}"
    assert len(set(got["find"].values())) == len(keys)
    assert len(got["blocks"]) == len(expect)
    for b, e in zip(got["blocks"], expect):
        assert b["sid"] == e["sid"] and b["count"] == e["count"] and len(b["cols"]) == len(e["cols"])
        for c, (col, (key, vt)) in enumerate(zip(b["cols"], e["cols"])):
            name_id, value_type, _, _, file_id = col
            assert name_id == got["find"][key], f"{name}: series {b['sid']} column {c} is {key}, resolved as id {name_id}"
            assert value_type == vt
            want_file = "fv.bin" if key.startswith("f:") else key[2:].split("/")[0] + ".tf"
            assert got["files"][file_id] == want_file
    assert got["sliced"] == 1, f"{name}: parsed in slices and merged, the directory differs"


def test_more_than_16_families_in_a_block_is_not_supported(dump_exe, tmp_path):
    got = host_dump(dump_exe, tmp_path, M.mixed(M.many_families(17)).files(), [])
    assert got["rc"] == ENOTSUP

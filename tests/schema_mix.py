"""Parts whose blocks carry different schemas, shared by test_part_schema_mix.py (host parser, no GPU) and
test_gpu_schema_mix.py.

A part holds every series of its group and shard, so the series of several measures share one part, and each block carries
the tag families and fields of its own series (banyand/measure/block.go:88-123 processTagFamilies / processTags): neighbouring
blocks differ in families, tags, fields, column count and sometimes in the value type of one field name.  oracle.build_mixed_part
writes such parts; `block_schemas` reads back, with a decoder of its own, what each block's metadata records.
"""
from __future__ import annotations

import struct

import numpy as np

from oracle import oracle as O
from tests.helpers import STEP, T0, build_part

S, I, F = O.VT_STR, O.VT_INT64, O.VT_FLOAT64


class Measure:
    """n_pts rows per series; fields [(name, vt)], families [(family, [(tag, vt)])].  Values are random per measure: string
    tags take 3 values prefixed with the measure's label, so that rows of different measures never share a key."""

    def __init__(self, label, sids, n_pts, fields, families, seed=0):
        self.label = label
        self.sids = np.asarray(sids, np.uint64)
        self.fields, self.families = list(fields), list(families)
        n = self.sids.size * n_pts
        self.sid = np.repeat(self.sids, n_pts)
        self.ts = np.tile(T0 + np.arange(n_pts, dtype=np.int64) * STEP, self.sids.size)
        self.ver = np.ones(n, np.int64)
        rng = np.random.default_rng(seed)

        def vals(vt):
            if vt == I:
                return rng.integers(-1000, 1000, n)
            if vt == F:
                return np.round(rng.uniform(-50.0, 150.0, n), 2)
            return [b"%s-%d" % (label.encode(), x) for x in rng.integers(0, 3, n)]
        self.field_data = [(name, vt, vals(vt), None) for name, vt in self.fields]
        self.fam_data = [(fam, [(t, vt, vals(vt), None) for t, vt in tags]) for fam, tags in self.families]

    def rows(self):
        return self.sid, self.ts, self.ver, self.field_data, self.fam_data

    def own_part(self):
        """the measure alone, in a single-schema part: the same blocks the mixed part holds for it"""
        return build_part(*self.rows())

    def expected_cols(self):
        """the columns of each of this measure's blocks, as the index decoders list them: fields in order, then families
        sorted by name (block_metadata.go:119-124), each with its tags in order"""
        cols = [("f:" + name, vt) for name, vt in self.fields]
        for fam, tags in sorted(self.families):
            cols += [(f"t:{fam}/{t}", vt) for t, vt in tags]
        return cols


def mixed(measures):
    return O.build_mixed_part([m.rows() for m in measures])


def interleave(n, k):
    """series ids 1..n*k dealt round-robin to k measures: consecutive series, and so consecutive blocks, alternate"""
    return [list(range(1 + j, n * k + 1, k)) for j in range(k)]


# ------------------------------------------------------------------ the block index, read back
def _varu(b, p):
    x = s = 0
    while True:
        c = b[p]
        p += 1
        x |= (c & 0x7F) << s
        s += 7
        if c < 0x80:
            return x, p


def _name(b, p):
    n, p = _varu(b, p)
    return bytes(b[p:p + n]).decode(), p + n


def _cfm(b, p):
    """columnFamilyMetadata (column_metadata.go:108-122) -> [(name, value_type)]"""
    n, p = _varu(b, p)
    out = []
    for _ in range(n):
        name, p = _name(b, p)
        vt = b[p]
        _, p = _varu(b, p + 1)
        _, p = _varu(b, p)
        out.append((name, vt))
    return out, p


def primary_frames(files):
    """meta.bin: one 40-byte primaryBlockMetadata per zstd frame of primary.bin (primary_metadata.go:60-83)"""
    meta = O.zstd_decompress(files["meta.bin"])
    return [struct.unpack(">QqqQQ", meta[i:i + 40]) for i in range(0, len(meta), 40)]


def block_schemas(files):
    """-> [dict(sid, count, frame, cols=[(key, value_type)])] for every block, keys "f:<field>" / "t:<family>/<tag>", read from
    meta.bin / primary.bin / <family>.tfm (block_metadata.go:133-168)"""
    out = []
    for frame, (_, _, _, off, size) in enumerate(primary_frames(files)):
        raw = O.zstd_decompress(files["primary.bin"][off:off + size])
        p = 0
        while p < len(raw):
            sid = struct.unpack(">Q", raw[p:p + 8])[0]
            _, p = _varu(raw, p + 8)           # uncompressedSizeBytes
            count, p = _varu(raw, p)
            _, p = _varu(raw, p)               # timestamps offset, size
            _, p = _varu(raw, p)
            _, p = _varu(raw, p + 17)          # min, max, encode type; version offset
            nfam, p = _varu(raw, p + 9)        # first version, its encode type
            fams = []
            for _ in range(nfam):
                name, p = _name(raw, p)
                o, p = _varu(raw, p)
                s, p = _varu(raw, p)
                fams.append((name, o, s))
            fields, p = _cfm(raw, p)
            cols = [("f:" + n, vt) for n, vt in fields]
            for name, o, s in fams:
                tags, _ = _cfm(files[name + ".tfm"][o:o + s], 0)
                cols += [(f"t:{name}/{t}", vt) for t, vt in tags]
            out.append(dict(sid=sid, count=count, frame=frame, cols=cols))
    return out


# ------------------------------------------------------------------ the cases
A = ([("i", I), ("f", F)], [("default", [("entity_id", S), ("region", S)])])
B = ([("i", I)], [("storage-only", [("entity_id", S)])])


def collision_cases():
    """-> {name: [Measure]}: one tag name in different families or at different positions, series alternating in the part"""
    ab, ba = interleave(6, 2), interleave(6, 2)
    # the same family with other tag lists: region moves from position 1 to 0, entity_id from 0 to 1 and 2
    moved = ([("i", I), ("g", I)], [("default", [("region", S), ("entity_id", S)])])
    longer = ([("i", I)], [("default", [("entity_id", S), ("zone", S), ("region", S)])])
    m3 = interleave(5, 3)
    many = interleave(1500, 2)   # 3000 blocks: primary.bin holds several frames, so the pattern crosses walkers
    return {
        "fam_ab": [Measure("a", ab[0], 5, *A, seed=1), Measure("b", ab[1], 5, *B, seed=2)],
        "fam_ba": [Measure("b", ba[0], 5, *B, seed=3), Measure("a", ba[1], 5, *A, seed=4)],
        "moved": [Measure("a", m3[0], 4, *A, seed=5), Measure("m", m3[1], 4, *moved, seed=6), Measure("l", m3[2], 4, *longer, seed=7)],
        "frames": [Measure("a", many[0], 2, *A, seed=8), Measure("b", many[1], 2, *B, seed=9)],
    }


def family_cases():
    """blocks with families [a, b], [b], [] and [a]"""
    ids = interleave(4, 4)
    return [Measure("ab", ids[0], 6, [("i", I)], [("a", [("x", S)]), ("b", [("y", I)])], seed=11),
            Measure("b", ids[1], 6, [("i", I)], [("b", [("y", I)])], seed=12),
            Measure("none", ids[2], 6, [("i", I)], [], seed=13),
            Measure("a", ids[3], 6, [("i", I)], [("a", [("x", S)])], seed=14)]


def many_families(n_fam):
    """one measure with n_fam families of one tag each, next to a measure with one family"""
    ids = interleave(3, 2)
    fams = [(f"fam{k:02d}", [("t", S)]) for k in range(n_fam)]
    return [Measure("wide", ids[0], 4, [("i", I)], fams, seed=15), Measure("one", ids[1], 4, [("i", I)], [("fam00", [("t", S)])], seed=16)]


def field_cases():
    """different field sets per block: i in F1 only, j in F2 and F3, f in F1 and F2"""
    ids = interleave(4, 3)
    fam = [("default", [("region", S)])]
    return [Measure("f1", ids[0], 6, [("i", I), ("f", F)], fam, seed=21),
            Measure("f2", ids[1], 6, [("f", F), ("j", I)], fam, seed=22),
            Measure("f3", ids[2], 6, [("j", I)], fam, seed=23)]


def type_mix_cases():
    """one field name, v, int64 in one measure and float64 in the other"""
    ids = interleave(4, 2)
    return [Measure("vi", ids[0], 50, [("v", I)], [("default", [("region", S)])], seed=31),
            Measure("vf", ids[1], 50, [("v", F)], [("default", [("region", S)])], seed=32)]


WIDE_POS = [(0, 64), (31, 32), (32, 33), (33, 63), (63, 64), (64, None), (None, 0)]


def wide_cases():
    """blocks of 65 columns: field q and tag w/k at the column positions WIDE_POS (None: absent).  Filler names belong to
    their measure, so the tag names at positions past the 24-slot positional cache change from block to block."""
    ids = interleave(3, len(WIDE_POS))
    out = []
    for m, (pf, pt) in enumerate(WIDE_POS):
        nf = 65 if pt is None else pt if pf is None else pf + 1
        fields = [(f"m{m}f{c}", I) for c in range(nf)]
        if pf is not None:
            fields[pf] = ("q", I)
        tags = [(f"m{m}t{c}", S) for c in range(nf, 65)]
        if pt is not None:
            tags[pt - nf] = ("k", S)
        out.append(Measure(f"w{m}", ids[m], 5, fields, [("w", tags)] if tags else [], seed=40 + m))
    return out


NAME_LENS = (1, 60, 61, 127)


def long_name_cases():
    """field and tag names of 1, 60, 61 and 127 bytes (the device index holds up to 60)"""
    ids = interleave(3, len(NAME_LENS))
    return [Measure(f"n{n}", ids[m], 4, [("i", I), ("f" * n, I)], [("default", [("k" * n, S)])], seed=50 + m)
            for m, n in enumerate(NAME_LENS)]


def many_names(total):
    """`total` distinct (kind, family, name) column names in one part: field i and family default/k in every measure, the
    rest fields of one measure each"""
    per = 62
    rest = total - 2
    n_meas = (rest + per - 1) // per
    ids = interleave(2, n_meas)
    out = []
    for m in range(n_meas):
        k = min(per, rest - m * per)
        out.append(Measure(f"x{m}", ids[m], 3, [("i", I)] + [(f"x{m}_{c}", I) for c in range(k)], [("default", [("k", S)])], seed=60 + m))
    return out


def distinct_names(measures):
    return {key for m in measures for key, _ in m.expected_cols()}

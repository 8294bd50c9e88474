"""ctypes binding of the CPU ORACLE (oracle/liboracle.so).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and the cpu_baseline /
``--impl reference`` legs of bench.py.  The product package never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

ENC_CONST, ENC_DELTA_CONST, ENC_DELTA, ENC_DELTA_OF_DELTA = 1, 2, 3, 4
ENC_PLAIN, ENC_DICTIONARY = 9, 10
VT_STR, VT_INT64, VT_FLOAT64, VT_BINARY = 1, 2, 3, 4
AGG_MEAN, AGG_MAX, AGG_MIN, AGG_COUNT, AGG_SUM = 1, 2, 3, 4, 5
OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE = 1, 2, 3, 4, 5, 6


def build(force: bool = False) -> str:
    """Compile oracle/liboracle.so with the committed Makefile (gcc only)."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs):
        subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    return _LIB_PATH


class _Buf(C.Structure):
    _fields_ = [("p", C.POINTER(C.c_uint8)), ("len", C.c_size_t), ("cap", C.c_size_t)]

    def bytes(self) -> bytes:
        return C.string_at(self.p, self.len) if self.len else b""


class _Bytes(C.Structure):
    _fields_ = [("p", C.c_void_p), ("len", C.c_int64)]


class _Column(C.Structure):
    _fields_ = [("name", C.c_char_p), ("value_type", C.c_int), ("i64", C.c_void_p), ("f64", C.c_void_p),
                ("bytes", C.POINTER(_Bytes)), ("nulls", C.c_void_p)]


class _Family(C.Structure):
    _fields_ = [("name", C.c_char_p), ("n_cols", C.c_int), ("cols", C.POINTER(_Column))]


class _Pred(C.Structure):
    _fields_ = [("family", C.c_char_p), ("tag", C.c_char_p), ("op", C.c_int), ("value_type", C.c_int),
                ("str", _Bytes), ("i64", C.c_int64)]


class _Agg(C.Structure):
    _fields_ = [("field", C.c_char_p), ("func", C.c_int)]


class _GroupKey(C.Structure):
    _fields_ = [("family", C.c_char_p), ("tag", C.c_char_p), ("value_type", C.c_int)]


class _Query(C.Structure):
    _fields_ = [("n_parts", C.c_int), ("parts", C.POINTER(C.c_void_p)), ("n_series", C.c_size_t),
                ("sids", C.c_void_p), ("groups", C.c_void_p), ("n_groups", C.c_int32),
                ("tmin", C.c_int64), ("tmax", C.c_int64), ("n_preds", C.c_int), ("preds", C.POINTER(_Pred)),
                ("n_aggs", C.c_int), ("aggs", C.POINTER(_Agg)), ("top_n", C.c_int), ("top_agg", C.c_int),
                ("top_desc", C.c_int), ("threads", C.c_int), ("per_thread_partials", C.c_int),
                ("n_keys", C.c_int), ("keys", C.POINTER(_GroupKey))]


class _Result(C.Structure):
    _fields_ = [("n_rows", C.c_int32), ("n_aggs", C.c_int32), ("group_id", C.POINTER(C.c_int32)),
                ("rows", C.POINTER(C.c_int64)), ("is_float", C.POINTER(C.c_uint8)),
                ("val_i64", C.POINTER(C.c_int64)), ("val_f64", C.POINTER(C.c_double)),
                ("rows_scanned", C.c_uint64), ("rows_matched", C.c_uint64), ("blocks_scanned", C.c_uint64),
                ("n_keys", C.c_int32), ("key", C.POINTER(_Bytes))]


class _Rows(C.Structure):
    _fields_ = [("n", C.c_size_t), ("sid", C.POINTER(C.c_uint64)), ("ts", C.POINTER(C.c_int64)),
                ("version", C.POINTER(C.c_int64)), ("n_fields", C.c_int), ("is_float", C.POINTER(C.c_uint8)),
                ("i64", C.POINTER(C.POINTER(C.c_int64))), ("f64", C.POINTER(C.POINTER(C.c_double))),
                ("null", C.POINTER(C.POINTER(C.c_uint8)))]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build()
    L = C.CDLL(_LIB_PATH)
    L.ob_last_error.restype = C.c_char_p
    L.ob_buf_free.argtypes = [C.POINTER(_Buf)]
    L.ob_varint64_append.argtypes = [C.POINTER(_Buf), C.c_int64]
    L.ob_varuint64_append.argtypes = [C.POINTER(_Buf), C.c_uint64]
    L.ob_varint64_list_read.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.ob_varint64_list_read.restype = C.c_size_t
    L.ob_int64_list_encode.argtypes = [C.POINTER(_Buf), C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
    L.ob_int64_list_decode.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_int64, C.c_size_t]
    L.ob_conv_int64_to_bytes.argtypes = [C.c_int64, C.c_char_p]
    L.ob_conv_bytes_to_int64.argtypes = [C.c_char_p]
    L.ob_conv_bytes_to_int64.restype = C.c_int64
    L.ob_float64_to_decimal_list.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int16)]
    L.ob_decimal_list_to_float64.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int16]
    L.ob_pow10.argtypes = [C.c_int]
    L.ob_pow10.restype = C.c_double
    L.ob_bytes_block_encode.argtypes = [C.POINTER(_Buf), C.POINTER(_Bytes), C.c_size_t]
    L.ob_bytes_block_decode.argtypes = [C.POINTER(_Bytes), C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(_Buf), C.c_int]
    L.ob_bytes_block_decode.restype = C.c_int64
    L.ob_dictionary_encode.argtypes = [C.POINTER(_Buf), C.POINTER(_Bytes), C.c_size_t]
    L.ob_dictionary_decode.argtypes = [C.POINTER(_Bytes), C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(_Buf)]
    L.ob_bitpack_encode.argtypes = [C.POINTER(_Buf), C.c_void_p, C.c_size_t]
    L.ob_zstd_compress.argtypes = [C.POINTER(_Buf), C.c_char_p, C.c_size_t, C.c_int]
    L.ob_zstd_decompress.argtypes = [C.POINTER(_Buf), C.c_char_p, C.c_size_t]
    L.ob_column_encode.argtypes = [C.POINTER(_Buf), C.c_int, C.POINTER(_Bytes), C.c_size_t]
    L.ob_column_decode.argtypes = [C.POINTER(_Bytes), C.c_size_t, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(_Buf)]
    L.ob_builder_new.restype = C.c_void_p
    L.ob_builder_free.argtypes = [C.c_void_p]
    L.ob_builder_append.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.POINTER(_Column), C.c_int, C.POINTER(_Family)]
    L.ob_builder_finish.argtypes = [C.c_void_p]
    L.ob_builder_finish.restype = C.c_void_p
    L.ob_builder_finish_many.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    L.ob_builder_finish_many.restype = C.c_void_p
    L.ob_part_open.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t)]
    L.ob_part_open.restype = C.c_void_p
    L.ob_part_free.argtypes = [C.c_void_p]
    L.ob_part_n_files.argtypes = [C.c_void_p]
    L.ob_part_file_name.argtypes = [C.c_void_p, C.c_int]
    L.ob_part_file_name.restype = C.c_char_p
    L.ob_part_file_data.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t)]
    L.ob_part_file_data.restype = C.POINTER(C.c_uint8)
    L.ob_part_meta.argtypes = [C.c_void_p] + [C.c_void_p] * 6
    L.ob_query_run.argtypes = [C.POINTER(_Query), C.POINTER(_Result)]
    L.ob_result_free.argtypes = [C.POINTER(_Result)]
    L.ob_scan_rows.argtypes = [C.POINTER(_Query), C.POINTER(_Rows)]
    L.ob_rows_free.argtypes = [C.POINTER(_Rows)]
    # bit writer
    L.ob_bitw_init.argtypes = [C.c_void_p, C.POINTER(_Buf)]
    L.ob_bitw_bool.argtypes = [C.c_void_p, C.c_int]
    L.ob_bitw_bits.argtypes = [C.c_void_p, C.c_uint64, C.c_int]
    L.ob_bitw_byte.argtypes = [C.c_void_p, C.c_uint8]
    L.ob_bitw_flush.argtypes = [C.c_void_p]
    _lib = L
    return L


def _err() -> str:
    return (lib().ob_last_error() or b"").decode()


# ------------------------------------------------------------------ codec helpers (golden tests)
def varint_encode(vals: Sequence[int]) -> bytes:
    b = _Buf()
    for v in vals:
        lib().ob_varint64_append(C.byref(b), int(v))
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def varuint_encode(v: int) -> bytes:
    b = _Buf()
    lib().ob_varuint64_append(C.byref(b), int(v))
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def int64_list_encode(a: Sequence[int]) -> Tuple[bytes, int, int]:
    arr = np.asarray(a, dtype=np.int64)
    b = _Buf()
    first = C.c_int64(0)
    enc = lib().ob_int64_list_encode(C.byref(b), arr.ctypes.data, arr.size, C.byref(first))
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out, enc, first.value


def int64_list_decode(src: bytes, enc: int, first: int, count: int) -> np.ndarray:
    dst = np.zeros(count, dtype=np.int64)
    rc = lib().ob_int64_list_decode(dst.ctypes.data, src, len(src), enc, first, count)
    if rc != 0:
        raise ValueError("int64 list decode failed")
    return dst


def conv_int64_to_bytes(v: int) -> bytes:
    out = C.create_string_buffer(8)
    lib().ob_conv_int64_to_bytes(int(v), out)
    return out.raw


def conv_bytes_to_int64(b: bytes) -> int:
    return lib().ob_conv_bytes_to_int64(b)


def float64_to_decimal_list(vals: Sequence[float]) -> Tuple[np.ndarray, int]:
    src = np.asarray(vals, dtype=np.float64)
    dst = np.zeros(max(src.size, 1), dtype=np.int64)
    e = C.c_int16(0)
    rc = lib().ob_float64_to_decimal_list(dst.ctypes.data, src.ctypes.data, src.size, C.byref(e))
    if rc != 0:
        raise ValueError("cannot encode float64 losslessly as decimal int")
    return dst[:src.size], e.value


def decimal_list_to_float64(ints: Sequence[int], exp: int) -> np.ndarray:
    src = np.asarray(ints, dtype=np.int64)
    dst = np.zeros(max(src.size, 1), dtype=np.float64)
    lib().ob_decimal_list_to_float64(dst.ctypes.data, src.ctypes.data, src.size, exp)
    return dst[:src.size]


def force_slow_float(on: bool) -> None:
    """Tests: disable the fast shortest-decimal path so both searches can be compared."""
    C.c_int.in_dll(lib(), "ob_force_slow_float").value = int(on)


def pow10(n: int) -> float:
    return lib().ob_pow10(n)


def _mk_bytes_array(items: Sequence[Optional[bytes]]):
    n = len(items)
    arr = (_Bytes * max(n, 1))()
    keep = []
    for i, it in enumerate(items):
        if it is None:
            arr[i].p = None
            arr[i].len = -1
        else:
            buf = C.create_string_buffer(bytes(it), max(len(it), 1))
            keep.append(buf)
            arr[i].p = C.cast(buf, C.c_void_p)
            arr[i].len = len(it)
    return arr, keep


def _read_bytes_array(arr, n) -> List[Optional[bytes]]:
    out: List[Optional[bytes]] = []
    for i in range(n):
        if arr[i].len < 0:
            out.append(None)
        else:
            out.append(C.string_at(arr[i].p, arr[i].len) if arr[i].len else b"")
    return out


def bytes_block_encode(items: Sequence[Optional[bytes]]) -> bytes:
    arr, _keep = _mk_bytes_array(items)
    b = _Buf()
    lib().ob_bytes_block_encode(C.byref(b), arr, len(items))
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def bytes_block_decode(src: bytes, n: int) -> List[Optional[bytes]]:
    arr = (_Bytes * max(n, 1))()
    arena = _Buf()
    rc = lib().ob_bytes_block_decode(arr, n, src, len(src), C.byref(arena), 0)
    if rc < 0:
        lib().ob_buf_free(C.byref(arena))
        raise ValueError("bytes block decode failed")
    out = _read_bytes_array(arr, n)
    lib().ob_buf_free(C.byref(arena))
    return out


def dictionary_encode(items: Sequence[Optional[bytes]]) -> Optional[bytes]:
    arr, _keep = _mk_bytes_array(items)
    b = _Buf()
    ok = lib().ob_dictionary_encode(C.byref(b), arr, len(items))
    out = b.bytes() if ok else None
    lib().ob_buf_free(C.byref(b))
    return out


def dictionary_decode(src: bytes, n: int) -> List[Optional[bytes]]:
    arr = (_Bytes * max(n, 1))()
    arena = _Buf()
    rc = lib().ob_dictionary_decode(arr, n, src, len(src), C.byref(arena))
    if rc != 0:
        lib().ob_buf_free(C.byref(arena))
        raise ValueError("dictionary decode failed")
    out = _read_bytes_array(arr, n)
    lib().ob_buf_free(C.byref(arena))
    return out


def bitpack_encode(vals: Sequence[int]) -> bytes:
    a = np.asarray(vals, dtype=np.uint32)
    b = _Buf()
    lib().ob_bitpack_encode(C.byref(b), a.ctypes.data, a.size)
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


class BitWriter:
    """pkg/encoding/writer.go Writer."""

    class _W(C.Structure):
        _fields_ = [("out", C.POINTER(_Buf)), ("cache", C.c_uint8), ("available", C.c_uint8)]

    def __init__(self):
        self._buf = _Buf()
        self._w = BitWriter._W()
        lib().ob_bitw_init(C.byref(self._w), C.byref(self._buf))

    def write_bool(self, b: bool):
        lib().ob_bitw_bool(C.byref(self._w), int(b))

    def write_bits(self, u: int, n: int):
        lib().ob_bitw_bits(C.byref(self._w), u, n)

    def write_byte(self, b: int):
        lib().ob_bitw_byte(C.byref(self._w), b)

    def flush(self):
        lib().ob_bitw_flush(C.byref(self._w))

    def bytes(self) -> bytes:
        return self._buf.bytes()


def bit_reader_script(data: bytes, ops: Sequence[int]) -> List[int]:
    """pkg/encoding/reader.go Reader over `data`: ops 0 = ReadBool, -1 = ReadByte, n > 0 = ReadBits(n)."""
    arr = (C.c_int * len(ops))(*ops)
    out = (C.c_uint64 * len(ops))()
    L = lib()
    L.ob_bit_reader_script.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int), C.c_size_t, C.POINTER(C.c_uint64)]
    if L.ob_bit_reader_script(data, len(data), arr, len(ops), out) != 0:
        raise RuntimeError("bit reader ran out of data")
    return list(out)


def zstd_compress(data: bytes, level: int = 1) -> bytes:
    b = _Buf()
    if lib().ob_zstd_compress(C.byref(b), data, len(data), level) != 0:
        raise RuntimeError("zstd compress failed")
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def zstd_decompress(data: bytes) -> bytes:
    b = _Buf()
    if lib().ob_zstd_decompress(C.byref(b), data, len(data)) != 0:
        raise RuntimeError("zstd decompress failed")
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def column_encode(value_type: int, cells: Sequence[Optional[bytes]]) -> bytes:
    arr, _keep = _mk_bytes_array(cells)
    b = _Buf()
    lib().ob_column_encode(C.byref(b), value_type, arr, len(cells))
    out = b.bytes()
    lib().ob_buf_free(C.byref(b))
    return out


def column_decode(value_type: int, src: bytes, n: int) -> List[Optional[bytes]]:
    arr = (_Bytes * max(n, 1))()
    arena = _Buf()
    rc = lib().ob_column_decode(arr, n, value_type, src, len(src), C.byref(arena))
    if rc != 0:
        lib().ob_buf_free(C.byref(arena))
        raise ValueError("column decode failed")
    out = _read_bytes_array(arr, n)
    lib().ob_buf_free(C.byref(arena))
    return out


# ------------------------------------------------------------------ parts
class Part:
    def __init__(self, handle):
        self._h = handle

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ob_part_free(self._h)
            self._h = None

    def files(self) -> Dict[str, bytes]:
        out = {}
        n = lib().ob_part_n_files(self._h)
        for i in range(n):
            ln = C.c_size_t(0)
            p = lib().ob_part_file_data(self._h, i, C.byref(ln))
            out[lib().ob_part_file_name(self._h, i).decode()] = C.string_at(p, ln.value) if ln.value else b""
        return out

    def meta(self) -> Dict[str, int]:
        tc, bc, unc, comp = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        mn, mx = C.c_int64(), C.c_int64()
        lib().ob_part_meta(self._h, C.byref(tc), C.byref(bc), C.byref(mn), C.byref(mx), C.byref(unc), C.byref(comp))
        return dict(total_count=tc.value, blocks_count=bc.value, min_ts=mn.value, max_ts=mx.value,
                    uncompressed=unc.value, compressed=comp.value)

    @staticmethod
    def open(files: Dict[str, bytes]) -> "Part":
        n = len(files)
        names = (C.c_char_p * n)(*[k.encode() for k in files])
        datas = (C.c_char_p * n)(*[bytes(v) for v in files.values()])
        lens = (C.c_size_t * n)(*[len(v) for v in files.values()])
        h = lib().ob_part_open(n, names, datas, lens)
        if not h:
            raise ValueError("ob_part_open: " + _err())
        return Part(h)


FieldSpec = Tuple[str, int, object, Optional[np.ndarray]]  # (name, value_type, values, nulls)


class PartBuilder:
    """Row batches -> measure part (memPart.mustInitFromDataPoints)."""

    def __init__(self):
        self._h = lib().ob_builder_new()

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ob_builder_free(self._h)
            self._h = None

    @staticmethod
    def _column(name: str, vt: int, values, nulls, keep: list) -> _Column:
        col = _Column()
        nb = name.encode()
        keep.append(nb)
        col.name = nb
        col.value_type = vt
        if vt == VT_INT64:
            a = np.ascontiguousarray(values, dtype=np.int64)
            keep.append(a)
            col.i64 = a.ctypes.data
        elif vt == VT_FLOAT64:
            a = np.ascontiguousarray(values, dtype=np.float64)
            keep.append(a)
            col.f64 = a.ctypes.data
        else:
            arr, k2 = _mk_bytes_array(values)
            keep.extend([arr, k2])
            col.bytes = arr
        if nulls is not None:
            nn = np.ascontiguousarray(nulls, dtype=np.uint8)
            keep.append(nn)
            col.nulls = nn.ctypes.data
        return col

    def append(self, sids, ts, versions, fields: Sequence[FieldSpec] = (),
               families: Sequence[Tuple[str, Sequence[FieldSpec]]] = ()):
        sids = np.ascontiguousarray(sids, dtype=np.uint64)
        ts = np.ascontiguousarray(ts, dtype=np.int64)
        versions = np.ascontiguousarray(versions, dtype=np.int64)
        n = sids.size
        keep: list = []
        fcols = (_Column * max(len(fields), 1))()
        for i, (name, vt, vals, nulls) in enumerate(fields):
            fcols[i] = self._column(name, vt, vals, nulls, keep)
        fams = (_Family * max(len(families), 1))()
        for i, (fname, cols) in enumerate(families):
            carr = (_Column * max(len(cols), 1))()
            for j, (name, vt, vals, nulls) in enumerate(cols):
                carr[j] = self._column(name, vt, vals, nulls, keep)
            fb = fname.encode()
            keep.extend([fb, carr])
            fams[i].name = fb
            fams[i].n_cols = len(cols)
            fams[i].cols = carr
        rc = lib().ob_builder_append(self._h, n, sids.ctypes.data, ts.ctypes.data, versions.ctypes.data,
                                     len(fields), fcols, len(families), fams)
        if rc != 0:
            raise ValueError("ob_builder_append: " + _err())

    def finish(self) -> Part:
        h = lib().ob_builder_finish(self._h)
        if not h:
            raise ValueError("ob_builder_finish: " + _err())
        return Part(h)


MeasureRows = Tuple[object, object, object, Sequence[FieldSpec], Sequence[Tuple[str, Sequence[FieldSpec]]]]


def build_mixed_part(measures: Sequence[MeasureRows]) -> Part:
    """One part holding several measures' series, as a part of one group and shard does.

    measures: (sids, ts, versions, fields, families) per measure, each with its own schema; no series may appear in
    two measures.  Each measure's rows are cut into blocks exactly as PartBuilder.finish cuts them, and the blocks of
    all measures are written in series order, so consecutive blocks carry different tag families and fields."""
    builders = []
    for sids, ts, versions, fields, families in measures:
        b = PartBuilder()
        b.append(sids, ts, versions, fields, families)
        builders.append(b)
    hs = (C.c_void_p * max(len(builders), 1))(*[b._h for b in builders])
    h = lib().ob_builder_finish_many(hs, len(builders))
    if not h:
        raise ValueError("ob_builder_finish_many: " + _err())
    return Part(h)


# ------------------------------------------------------------------ query
@dataclass
class Pred:
    family: str
    tag: str
    op: int
    value: object  # bytes/str for string tags, int for int64 tags


@dataclass
class Query:
    parts: Sequence[Part]
    sids: Sequence[int]
    aggs: Sequence[Tuple[str, int]]  # (field, func)
    groups: Optional[Sequence[int]] = None
    n_groups: int = 1
    tmin: int = -(1 << 63)
    tmax: int = (1 << 63) - 1
    preds: Sequence[Pred] = field(default_factory=list)
    top_n: int = 0
    top_agg: int = 0
    top_desc: bool = True
    threads: int = 1
    per_thread_partials: bool = False
    group_key: Optional[Tuple[str, str]] = None  # (family, tag): shorthand for group_keys=[(family, tag, VT_STR)]
    # per-row group key: 1..4 stored tags (family, tag, VT_STR / VT_BINARY / VT_INT64) in GroupBy order
    group_keys: Optional[Sequence[Tuple[str, str, int]]] = None


@dataclass
class Result:
    group_id: np.ndarray
    rows: np.ndarray
    is_float: np.ndarray
    val_i64: np.ndarray  # [n_rows, n_aggs]
    val_f64: np.ndarray
    rows_scanned: int
    rows_matched: int
    blocks_scanned: int
    # [n_rows] key of each row (queries with a group key): with one component its bytes, with K >= 2 a tuple of K components;
    # a string component is its bytes, an int64 one its 8 little-endian bytes
    key: Optional[List[object]] = None

    def value(self, row: int, agg: int):
        return float(self.val_f64[row, agg]) if self.is_float[agg] else int(self.val_i64[row, agg])


def _mk_query(q: Query):
    keep: list = []
    cq = _Query()
    parts = (C.c_void_p * max(len(q.parts), 1))(*[p._h for p in q.parts])
    keep.append(parts)
    cq.n_parts = len(q.parts)
    cq.parts = parts
    sids = np.ascontiguousarray(q.sids, dtype=np.uint64)
    keep.append(sids)
    cq.n_series = sids.size
    cq.sids = sids.ctypes.data
    if q.groups is not None:
        g = np.ascontiguousarray(q.groups, dtype=np.int32)
        keep.append(g)
        cq.groups = g.ctypes.data
        cq.n_groups = q.n_groups
    else:
        cq.groups = None
        cq.n_groups = 1
    cq.tmin, cq.tmax = q.tmin, q.tmax
    preds = (_Pred * max(len(q.preds), 1))()
    for i, p in enumerate(q.preds):
        fb, tb = p.family.encode(), p.tag.encode()
        keep.extend([fb, tb])
        preds[i].family, preds[i].tag, preds[i].op = fb, tb, p.op
        if isinstance(p.value, (int, np.integer)):
            preds[i].value_type = VT_INT64
            preds[i].i64 = int(p.value)
            preds[i].str.p, preds[i].str.len = None, -1
        else:
            vb = p.value.encode() if isinstance(p.value, str) else bytes(p.value)
            buf = C.create_string_buffer(vb, max(len(vb), 1))
            keep.append(buf)
            preds[i].value_type = VT_STR
            preds[i].str.p = C.cast(buf, C.c_void_p)
            preds[i].str.len = len(vb)
    keep.append(preds)
    cq.n_preds, cq.preds = len(q.preds), preds
    aggs = (_Agg * max(len(q.aggs), 1))()
    for i, (fname, func) in enumerate(q.aggs):
        nb = fname.encode()
        keep.append(nb)
        aggs[i].field, aggs[i].func = nb, func
    keep.append(aggs)
    cq.n_aggs, cq.aggs = len(q.aggs), aggs
    cq.top_n, cq.top_agg, cq.top_desc = q.top_n, q.top_agg, int(q.top_desc)
    cq.threads, cq.per_thread_partials = q.threads, int(q.per_thread_partials)
    gks = _group_keys(q)
    keys = (_GroupKey * max(len(gks), 1))()
    for i, (fam, tag, vt) in enumerate(gks):
        fb, tb = fam.encode(), tag.encode()
        keep.extend([fb, tb])
        keys[i].family, keys[i].tag, keys[i].value_type = fb, tb, vt
    keep.append(keys)
    cq.n_keys, cq.keys = len(gks), keys
    return cq, keep


def _group_keys(q: Query) -> List[Tuple[str, str, int]]:
    if q.group_keys is not None:
        if q.group_key is not None:
            raise ValueError("group_key and group_keys both set")
        return list(q.group_keys)
    return [] if q.group_key is None else [(q.group_key[0], q.group_key[1], VT_STR)]


def run_query(q: Query) -> Result:
    cq, _keep = _mk_query(q)
    r = _Result()
    if lib().ob_query_run(C.byref(cq), C.byref(r)) != 0:
        raise RuntimeError("ob_query_run: " + _err())
    n, a = r.n_rows, r.n_aggs
    res = Result(
        group_id=np.ctypeslib.as_array(r.group_id, (max(n, 1),))[:n].copy(),
        rows=np.ctypeslib.as_array(r.rows, (max(n, 1),))[:n].copy(),
        is_float=np.ctypeslib.as_array(r.is_float, (max(a, 1),))[:a].copy().astype(bool),
        val_i64=np.ctypeslib.as_array(r.val_i64, (max(n, 1) * max(a, 1),))[:n * a].copy().reshape(n, a),
        val_f64=np.ctypeslib.as_array(r.val_f64, (max(n, 1) * max(a, 1),))[:n * a].copy().reshape(n, a),
        rows_scanned=r.rows_scanned, rows_matched=r.rows_matched, blocks_scanned=r.blocks_scanned)
    K = r.n_keys
    if K:
        parts = [C.string_at(r.key[j].p, r.key[j].len) if r.key[j].len > 0 else b"" for j in range(n * K)]
        res.key = parts if K == 1 else [tuple(parts[i * K:(i + 1) * K]) for i in range(n)]
    lib().ob_result_free(C.byref(r))
    return res


def scan_rows(q: Query) -> Dict[str, object]:
    """Every selected row after merge + version dedup + predicates (test helper)."""
    cq, _keep = _mk_query(q)
    r = _Rows()
    if lib().ob_scan_rows(C.byref(cq), C.byref(r)) != 0:
        raise RuntimeError("ob_scan_rows: " + _err())
    n = r.n
    out: Dict[str, object] = {
        "sid": np.ctypeslib.as_array(r.sid, (max(n, 1),))[:n].copy() if n else np.zeros(0, np.uint64),
        "ts": np.ctypeslib.as_array(r.ts, (max(n, 1),))[:n].copy() if n else np.zeros(0, np.int64),
        "version": np.ctypeslib.as_array(r.version, (max(n, 1),))[:n].copy() if n else np.zeros(0, np.int64),
        "fields": []}
    seen: List[str] = []
    for fname, _ in q.aggs:
        if fname not in seen:
            seen.append(fname)
    for f in range(r.n_fields):
        isf = bool(r.is_float[f])
        if n:
            vals = np.ctypeslib.as_array(r.f64[f] if isf else r.i64[f], (n,)).copy()
            nulls = np.ctypeslib.as_array(r.null[f], (n,)).copy().astype(bool)
        else:
            vals = np.zeros(0, np.float64 if isf else np.int64)
            nulls = np.zeros(0, bool)
        out["fields"].append((seen[f], isf, vals, nulls))
    lib().ob_rows_free(C.byref(r))
    return out

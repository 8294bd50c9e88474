"""GPUScanAgg: the vectorized.PullOperator that replaces Scan -> GroupByAgg (-> Top) of the reference's
vec plan tree (pkg/query/vectorized/measure/plan/{dispatch.go:97-277,executor.go:45-80}) with one call
into libbydbgpu.so.  Names and contracts follow the reference:

  AggFunc / AggSpec                 pkg/query/vectorized/measure/aggregation.go:44-66
  ColumnRole / ColumnType / ColumnDef / BatchSchema   pkg/query/vectorized/schema.go
  RecordBatch (Columns, Len, Selection=None)          pkg/query/vectorized/batch.go:33
  PullOperator {Init, OutputSchema, NextBatch, Close} pkg/query/vectorized/operator.go:34-52
  output schema = buildAggOutputSchema               aggregation.go:402-418
  Top semantics                                       pkg/query/vectorized/measure/top.go:145-214

A GroupBy key column with per-series values (ScanSpec.series_tags: entity / indexed tags) is densified per series.  A key column
that is a stored tag (a tag column absent from series_tags) makes the operator call bydb_scan_agg_keyed(_wide), which adds the row's
value of that tag to the group.  With max_key_values above 256, two to four stored key columns go to bydb_scan_agg_keys_wide as a
tuple, in GroupBy order; at 256 or below only one may be a stored tag (include/bydb_operator.hpp follows the same rules).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from enum import IntEnum
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import capi


class AggFunc(IntEnum):  # aggregation.go:47-55
    AggSum = 0
    AggCount = 1
    AggMin = 2
    AggMax = 3
    AggMean = 4


AggSum, AggCount, AggMin, AggMax, AggMean = AggFunc.AggSum, AggFunc.AggCount, AggFunc.AggMin, AggFunc.AggMax, AggFunc.AggMean

_TO_MODEL = {AggSum: capi.AGG_SUM, AggCount: capi.AGG_COUNT, AggMin: capi.AGG_MIN, AggMax: capi.AGG_MAX,
             AggMean: capi.AGG_MEAN}  # toModelAggFunc, aggregation.go:377-392


class ColumnRole(IntEnum):  # schema.go
    RoleTimestamp = 0
    RoleVersion = 1
    RoleSeriesID = 2
    RoleShardID = 3
    RoleTag = 4
    RoleField = 5


class ColumnType(IntEnum):
    ColumnTypeInt64 = 0
    ColumnTypeFloat64 = 1
    ColumnTypeString = 2
    ColumnTypeBytes = 3


@dataclass(frozen=True)
class ColumnDef:
    Name: str
    Role: ColumnRole
    Type: ColumnType
    TagFamily: str = ""


@dataclass
class BatchSchema:
    Columns: List[ColumnDef]

    def field_index(self, name: str) -> int:
        for i, c in enumerate(self.Columns):
            if c.Role == ColumnRole.RoleField and c.Name == name:
                return i
        raise KeyError(name)


@dataclass
class RecordBatch:
    """Columnar batch: Columns[i] is a python list (tags) or numpy array (fields); Selection is always None."""
    Schema: BatchSchema
    Columns: List[object]
    Len: int
    Selection: Optional[np.ndarray] = None


@dataclass
class AggSpec:
    Output: str
    Func: AggFunc
    InputCol: int  # index into the input schema; must be an int64 or float64 field column


@dataclass
class TopSpec:
    N: int
    AggIndex: int = 0       # which AggSpec orders the rows
    Desc: bool = True       # modelv1.Sort_SORT_DESC


@dataclass
class LimitSpec:
    """BatchLimit (pkg/query/vectorized/measure/limit.go:27-73): the rows [Offset, Offset+Limit) of the output stream."""
    Offset: int = 0
    Limit: int = 100   # the planner's default when the request sets none (pkg/query/logical/measure/measure_analyzer.go:31)


@dataclass
class ScanSpec:
    """What measure.Query resolved before the scan (banyand/measure/query.go:88-312)."""
    parts: Sequence[int]                       # part handles (snapshot.getParts, query.go:216)
    series_ids: Sequence[int]                  # searchSeriesList result, in index order
    series_tags: Dict[Tuple[str, str], Sequence[object]] = field(default_factory=dict)
    # ^ entity / indexed tag values per series (storedIndexValue, block.go:509-530): (family, tag) -> [value per series]
    tmin: int = -(1 << 63)
    tmax: int = (1 << 63) - 1
    preds: Sequence[capi.Pred] = field(default_factory=list)
    order_desc: bool = False
    # ^ orderBy sort of the request: the scan visits the series list backwards, so groups are numbered (and non-key
    #   projected tags take their first-seen value) from the far end -- aggregation.go:211-213 on a reversed stream
    max_key_values: int = 0
    # ^ distinct values a stored-tag GroupBy key may take over the query (bydb_group_key.max_values; 0 = the library's 64):
    #   up to 256 the per-value passes of scan_agg_keyed answer, up to 65,536 the one pass of scan_agg_keyed_wide; with two to
    #   four stored keys (above 256 only) the distinct key tuples (bydb_group_keys.max_values) of scan_agg_keys_wide


_MAX_STORED_KEYS = 4   # the tags of a bydb_group_keys tuple


def _key_cell(t: ColumnType, k: bytes):
    """a row's stored-tag key bytes (groupby.go:226-254) as a cell of the key column; a nil cell came back as 0 / \"\" """
    if t == ColumnType.ColumnTypeInt64:
        return int.from_bytes(k, "little", signed=True)
    if t == ColumnType.ColumnTypeString:
        return k.decode("utf-8", "surrogateescape")
    return k


class GPUScanAgg:
    """PullOperator: (batch) / None at EOF / raises BydbError (sticky) -- operator.go:41-48."""

    def __init__(self, ctx: capi.Context, input_schema: BatchSchema, key_indices: Sequence[int], aggs: Sequence[AggSpec],
                 scan: ScanSpec, batch_size: int = 1024, top: Optional[TopSpec] = None, limit: Optional[LimitSpec] = None):
        self._ctx = ctx
        self._in = input_schema
        self._keys = list(key_indices)
        self._aggs = list(aggs)
        self._scan = scan
        self._batch = max(1, int(batch_size))
        self._top = top
        self._limit = limit
        self._row_end = 0
        self._tag_idx = [i for i, c in enumerate(input_schema.Columns) if c.Role == ColumnRole.RoleTag] or list(self._keys)
        for a in self._aggs:
            col = input_schema.Columns[a.InputCol]
            if col.Role != ColumnRole.RoleField or col.Type not in (ColumnType.ColumnTypeInt64, ColumnType.ColumnTypeFloat64):
                raise ValueError(f"AggSpec {a.Output}: input column must be an int64/float64 field")
        defs = [input_schema.Columns[i] for i in self._tag_idx]
        for a in self._aggs:  # aggOutputType, aggregation.go:425-430
            t = ColumnType.ColumnTypeInt64 if a.Func == AggCount else input_schema.Columns[a.InputCol].Type
            defs.append(ColumnDef(a.Output, ColumnRole.RoleField, t))
        self._out = BatchSchema(defs)
        self._result: Optional[capi.Result] = None
        self._group_first_series: List[int] = []
        self._stored_keys: List[int] = []   # input columns of the stored-tag GroupBy keys, in GroupBy order
        self._cursor = 0
        self._closed = False
        self._err: Optional[Exception] = None
        self._inited = False
        self.stats: Optional[capi.Stats] = None

    # ---- BatchOperator
    def Init(self, ctx=None) -> None:
        self._inited = True

    def OutputSchema(self) -> BatchSchema:
        return self._out

    def Close(self) -> None:  # idempotent
        self._closed = True
        self._result = None

    # ---- PullOperator
    def NextBatch(self, ctx=None) -> Optional[RecordBatch]:
        if self._err is not None:
            raise self._err
        if self._closed:
            return None
        if self._result is None:
            try:
                self._run()
            except Exception as e:  # sticky error contract (model/batch.go:41-46)
                self._err = e
                raise
        r = self._result
        if self._cursor >= self._row_end:
            return None
        lo, hi = self._cursor, min(self._cursor + self._batch, self._row_end)
        self._cursor = hi
        cols: List[object] = []
        for ti in self._tag_idx:
            cdef = self._in.Columns[ti]
            if ti in self._stored_keys:
                t = self._stored_keys.index(ti)
                tuple_key = len(self._stored_keys) > 1   # a row's key is then the tuple of its tags' key bytes
                cols.append([_key_cell(cdef.Type, k[t] if tuple_key else k) for k in r.key[lo:hi]])
                continue
            vals = self._scan.series_tags.get((cdef.TagFamily, cdef.Name))
            cols.append([None if vals is None else vals[self._group_first_series[g]] for g in r.group_id[lo:hi]])
        for ai, _ in enumerate(self._aggs):
            cols.append(r.val_f64[lo:hi, ai].copy() if r.is_float[ai] else r.val_i64[lo:hi, ai].copy())
        return RecordBatch(self._out, cols, hi - lo)

    def _run(self) -> None:
        sc = self._scan
        sids = np.asarray(sc.series_ids, dtype=np.uint64)
        # group key per series = tuple of key-column values; dense ids in first-appearance order
        # (aggregation.go:211-213; series-major scan order for group-by-entity).  A tag key column without per-series values
        # is a stored tag: its value changes from row to row, and bydb_scan_agg_keyed adds it to the series group (above 256
        # values bydb_scan_agg_keys_wide adds the tuple of two to four of them).  Any other key column (a field) still needs
        # per-series values.
        keyvals = []
        self._stored_keys = []
        for ki in self._keys:
            cdef = self._in.Columns[ki]
            vals = sc.series_tags.get((cdef.TagFamily, cdef.Name))
            if vals is None and cdef.Role == ColumnRole.RoleTag:
                if self._stored_keys and sc.max_key_values <= 256:
                    raise capi.BydbError(capi.ENOTSUP, f"GroupBy key {cdef.TagFamily}/{cdef.Name}: at most one stored-tag key per query")
                if len(self._stored_keys) == _MAX_STORED_KEYS:
                    raise capi.BydbError(capi.ENOTSUP, f"GroupBy key {cdef.TagFamily}/{cdef.Name}: at most four stored-tag keys per query")
                self._stored_keys.append(ki)
                continue
            if vals is None or len(vals) != len(sids):
                raise ValueError(f"GroupBy key {cdef.TagFamily}/{cdef.Name} needs one value per series (entity / indexed tag)")
            keyvals.append(vals)
        if self._stored_keys and sc.order_desc:
            raise capi.BydbError(capi.ENOTSUP, "a stored-tag GroupBy key takes the ascending series order only (order_desc)")
        group_of: Dict[tuple, int] = {}
        gids = np.zeros(len(sids), dtype=np.int32)
        self._group_first_series = []
        for i in (range(len(sids) - 1, -1, -1) if sc.order_desc else range(len(sids))):
            k = tuple(kv[i] for kv in keyvals)
            g = group_of.get(k)
            if g is None:
                g = len(group_of)
                group_of[k] = g
                self._group_first_series.append(i)
            gids[i] = g
        order = np.argsort(sids, kind="stable")  # the C ABI wants ascending series ids (query.go:601)
        q = capi.Query(parts=list(sc.parts), series_ids=sids[order], series_group=gids[order] if self._keys else None,
                       n_groups=max(len(group_of), 1),
                       aggs=[(self._in.Columns[a.InputCol].Name, _TO_MODEL[a.Func]) for a in self._aggs],
                       tmin=sc.tmin, tmax=sc.tmax, preds=list(sc.preds),
                       top_n=self._top.N if self._top else 0, top_agg=self._top.AggIndex if self._top else 0,
                       top_desc=self._top.Desc if self._top else True)
        if not self._keys:
            self._group_first_series = ([len(sids) - 1] if sc.order_desc else [0]) if len(sids) else []
        ckeys = []
        for ki in self._stored_keys:
            cdef = self._in.Columns[ki]
            ckeys.append((cdef.TagFamily, cdef.Name, capi.VT_INT64 if cdef.Type == ColumnType.ColumnTypeInt64 else 0))
        if not ckeys:
            self._result = self._ctx.scan_agg(q)
        elif len(ckeys) == 1:
            family, tag, vt = ckeys[0]
            # above the per-value passes' 256 values, the one-pass form (which answers the same rows)
            keyed = self._ctx.scan_agg_keyed_wide if sc.max_key_values > 256 else self._ctx.scan_agg_keyed
            self._result = keyed(q, family, tag, sc.max_key_values, vt)
        else:   # max_key_values counts the distinct tuples
            self._result = self._ctx.scan_agg_keys_wide(q, ckeys, sc.max_key_values)
        self.stats = self._result.stats
        # offset / limit window over the (Top-ordered) output rows, limit.go:56-73
        n = len(self._result.group_id)
        if self._limit is None:
            self._cursor, self._row_end = 0, n
        else:
            self._cursor = min(max(int(self._limit.Offset), 0), n)
            self._row_end = min(self._cursor + max(int(self._limit.Limit), 0), n)

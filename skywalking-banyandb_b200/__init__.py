"""bydb_b200 -- host-side mirror of BanyanDB's measure-query operator surface over libbydbgpu.so.

The reference's host code is Go; there is no Go toolchain in this image, so the layer above the C ABI
(include/bydb_gpu.h) is mirrored here for tests and the bench: same names, argument meaning and error
behaviour as the reference's vectorized operator API

  * ``AggFunc`` / ``AggSpec``         pkg/query/vectorized/measure/aggregation.go:44-66
  * ``ColumnDef`` / ``BatchSchema``   pkg/query/vectorized/schema.go:32-66
  * ``RecordBatch``                   pkg/query/vectorized/batch.go:33
  * ``GPUScanAgg`` (a PullOperator: Init / OutputSchema / NextBatch / Close with the
    (batch, None) / (None, None) EOF / raise-on-error, sticky-error, idempotent-Close contract of
    pkg/query/vectorized/operator.go:34-52) -- the operator INTEGRATION.md installs as ``scan.Source``
    in plan.Dispatch, collapsing Scan -> GroupByAgg (-> Top).

Everything that touches data goes through the C ABI; there is no CPU fallback in this package.
The directory name contains a hyphen, so the package is registered under the import name
``bydb_b200`` by ``__graft_entry__`` / ``tests/conftest.py`` (importlib).
"""
from .capi import (  # noqa: F401
    AGG_COUNT, AGG_MAX, AGG_MEAN, AGG_MIN, AGG_SUM, OP_EQ, OP_GE, OP_GT, OP_LE, OP_LT, OP_NE,
    VT_BINARY, VT_FLOAT64, VT_INT64, VT_STR, BydbError, Context, Pred, PreparedQuery, Query, Result, Stats,
    keyed_reduce_slot_bytes, keyed_wide_reduce_slot_bytes, keys_wide_reduce_slot_bytes, library_path, load_library,
)
from .scan_operator import (  # noqa: F401
    AggCount, AggFunc, AggMax, AggMean, AggMin, AggSpec, AggSum, BatchSchema, ColumnDef, ColumnType,
    ColumnRole, GPUScanAgg, LimitSpec, RecordBatch, ScanSpec, TopSpec,
)

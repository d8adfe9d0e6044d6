"""Async surface mirroring the reference's `AsyncTable.query().nearest_to(...).to_arrow()` for the vector-query hot
path (python/python/lancedb/query.py:3307-3405 `AsyncQuery.nearest_to`, :3551-3723
`AsyncVectorQueryBase`, :2867-2960 `to_batches / to_arrow / to_list / to_pandas`; SURVEY.md 8b "Surface that must stay
unchanged").

In the reference the coroutine hands the request to tokio workers (python/src/runtime.rs:113-151) and each query vector
becomes its own plan; here the coroutine runs the synchronous builder (query.py, same request semantics) in a worker
thread -- the ctypes call releases the GIL, the library is re-entrant (per-call stream + workspace), and concurrent
single-vector callers are what `lgpu_search_coalesced` batches -- so `asyncio.gather` over many queries overlaps them
on the GPU exactly as tokio would.  Setter names, defaults (limit 10, nprobes 20) and error types are the reference's.
Plain scans (`query()` without `nearest_to`) are served from the host table: they are not on the GPU path.
"""
from __future__ import annotations

import asyncio
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Union

import numpy as np
import pyarrow as pa

from . import filter as _filter
from .table import DBConnection, Table


@dataclass
class IvfPq:
    """Index.IvfPq parameters (python/python/lancedb/index.py:670-800, rust/lancedb/src/index/vector.rs:246-319)."""
    distance_type: str = "l2"
    num_partitions: Optional[int] = None
    num_sub_vectors: Optional[int] = None
    num_bits: int = 8
    max_iterations: int = 50
    sample_rate: int = 256


@dataclass
class IvfRq:
    """Index.IvfRq parameters (python/python/lancedb/index.py:803-856, rust/lancedb/src/index/vector.rs:321-369):
    RaBitQ with num_bits = 1 (the only width served)."""
    distance_type: str = "l2"
    num_partitions: Optional[int] = None
    num_bits: int = 1
    max_iterations: int = 50
    sample_rate: int = 256


@dataclass
class IvfFlat:
    """Index.IvfFlat parameters (rust/lancedb/src/index/vector.rs:169-209): served over binary (fixed_size_list<uint8>)
    columns with distance_type="hamming"; the default "l2", like any other metric there, is refused (ValueError), and a
    float column raises NotImplementedError."""
    distance_type: str = "l2"
    num_partitions: Optional[int] = None
    max_iterations: int = 50
    sample_rate: int = 256


class AsyncRecordBatchReader:
    """What `to_batches` resolves to: `async for batch in reader`, `await reader.read_all()`."""

    def __init__(self, table: pa.Table, max_batch_length: Optional[int]):
        self.schema = table.schema
        self._batches = table.to_batches(max_chunksize=max_batch_length or 1024)   # MaxBatchLengthStream, utils/mod.rs:395
        self._i = 0

    def __aiter__(self):
        return self

    async def __anext__(self) -> pa.RecordBatch:
        if self._i >= len(self._batches):
            raise StopAsyncIteration
        self._i += 1
        return self._batches[self._i - 1]

    async def read_all(self) -> pa.Table:
        rest, self._i = self._batches[self._i:], len(self._batches)
        return pa.Table.from_batches(rest, schema=self.schema)


class _AsyncQueryBase:
    def __init__(self, table: Table):
        self._table = table
        self._where: Optional[str] = None
        self._limit: Optional[int] = None
        self._offset = 0
        self._columns: Optional[List[str]] = None
        self._with_row_id = False
        self._postfilter = False

    def where(self, predicate: str):
        self._where = predicate if self._where is None else f"({self._where}) AND ({predicate})"
        return self

    def limit(self, limit: int):
        self._limit = limit
        return self

    def offset(self, offset: int):
        self._offset = offset
        return self

    def select(self, columns: Union[List[str], Dict[str, str]]):
        if isinstance(columns, dict):
            raise NotImplementedError("computed columns are evaluated by DataFusion in the reference; select a list")
        self._columns = list(columns)
        return self

    def with_row_id(self):
        self._with_row_id = True
        return self

    def postfilter(self):
        self._postfilter = True
        return self

    # ---- execution: the blocking part runs in a worker thread ----
    def _run(self, timeout) -> pa.Table:
        raise NotImplementedError

    async def to_arrow(self, timeout=None) -> pa.Table:
        return await asyncio.to_thread(self._run, timeout)

    async def to_list(self, timeout=None) -> List[dict]:
        return (await self.to_arrow(timeout)).to_pylist()

    async def to_pandas(self, timeout=None, **kw):
        return (await self.to_arrow(timeout)).to_pandas(**kw)

    async def to_batches(self, *, max_batch_length: Optional[int] = None, timeout=None) -> AsyncRecordBatchReader:
        return AsyncRecordBatchReader(await self.to_arrow(timeout), max_batch_length)


class AsyncQuery(_AsyncQueryBase):
    """`AsyncTable.query()`: a plain scan until `nearest_to` turns it into a vector query."""

    def nearest_to(self, query_vector) -> "AsyncVectorQuery":
        if query_vector is None:
            raise ValueError("query_vector can not be None")
        return AsyncVectorQuery(self, query_vector)

    def _run(self, timeout) -> pa.Table:
        t = self._table._data
        if self._with_row_id:
            t = t.append_column("_rowid", pa.array(np.arange(t.num_rows, dtype=np.uint64)))
        if self._where is not None:
            t = t.filter(pa.array(_filter.evaluate(self._table._data, self._where)))
        if self._columns is not None:
            t = t.select(self._columns + (["_rowid"] if self._with_row_id else []))
        t = t.slice(self._offset)
        return t if self._limit is None else t.slice(0, self._limit)


class AsyncVectorQuery(_AsyncQueryBase):
    def __init__(self, base: AsyncQuery, query_vector):
        super().__init__(base._table)
        self.__dict__.update({k: v for k, v in base.__dict__.items() if k != "_table"})
        q = query_vector
        multi = isinstance(q, (list, tuple, np.ndarray)) and len(q) > 0 and isinstance(q[0], (list, tuple, np.ndarray))
        self._vectors: List[np.ndarray] = [np.asarray(v, np.float32) for v in (q if multi else [q])]
        self._column: Optional[str] = None
        self._distance_type: Optional[str] = None
        # the request's defaults (rust/lancedb/src/query.rs:1097-1113); the setters below validate EAGERLY against the
        # current state like the Rust builder they call into (query.rs:1232-1275), so the order of calls matters
        self._minimum_nprobes: int = 20
        self._maximum_nprobes: Optional[int] = 20       # None = no limit
        self._lower: Optional[float] = None
        self._upper: Optional[float] = None
        self._refine_factor: Optional[int] = None
        self._use_index = True

    def add_query_vector(self, vector):
        self._vectors.append(np.asarray(vector, np.float32))
        return self

    def column(self, column: str):
        self._column = column
        return self

    def nprobes(self, nprobes: int):
        if nprobes <= 0:
            raise ValueError("minimum_nprobes must be greater than 0")
        self._minimum_nprobes = self._maximum_nprobes = int(nprobes)
        return self

    def minimum_nprobes(self, minimum_nprobes: int):
        if minimum_nprobes <= 0:
            raise ValueError("minimum_nprobes must be greater than 0")
        if self._maximum_nprobes is not None and minimum_nprobes > self._maximum_nprobes:
            raise ValueError("minimum_nprobes must be less than or equal to maximum_nprobes")
        self._minimum_nprobes = int(minimum_nprobes)
        return self

    def maximum_nprobes(self, maximum_nprobes: int):
        if maximum_nprobes == 0:                         # "no limit" (python/src/query.rs:949-954)
            self._maximum_nprobes = None
            return self
        if maximum_nprobes < self._minimum_nprobes:
            raise ValueError("maximum_nprobes must be greater than or equal to minimum_nprobes")
        self._maximum_nprobes = int(maximum_nprobes)
        return self

    def distance_range(self, lower_bound: Optional[float] = None, upper_bound: Optional[float] = None):
        self._lower, self._upper = lower_bound, upper_bound
        return self

    def ef(self, ef: int):                       # HNSW only: no effect on IVF_PQ (query.py:3642-3655)
        return self

    def refine_factor(self, refine_factor: int):
        self._refine_factor = refine_factor
        return self

    def distance_type(self, distance_type: str):
        self._distance_type = distance_type
        return self

    def bypass_vector_index(self):
        self._use_index = False
        return self

    def _builder(self):
        dims = {v.shape[-1] for v in self._vectors}
        if len(dims) != 1 or any(v.ndim != 1 for v in self._vectors):
            raise ValueError("query vectors must be one-dimensional and of equal length")
        q = self._vectors[0] if len(self._vectors) == 1 else np.stack(self._vectors)
        b = self._table.search(q, vector_column_name=self._column)
        if self._distance_type is not None:
            b.distance_type(self._distance_type)
        b.minimum_nprobes(self._minimum_nprobes).maximum_nprobes(self._maximum_nprobes or 0)   # validated above
        if self._lower is not None or self._upper is not None:
            b.distance_range(self._lower, self._upper)
        if self._refine_factor is not None:
            b.refine_factor(self._refine_factor)
        if self._limit is not None:
            b.limit(self._limit)
        if self._offset:
            b.offset(self._offset)
        if self._columns is not None:
            b.select(self._columns)
        if self._with_row_id:
            b.with_row_id(True)
        if not self._use_index:
            b.bypass_vector_index()
        if self._where is not None:
            b.where(self._where, prefilter=not self._postfilter)
        return b

    def _run(self, timeout) -> pa.Table:
        return self._builder().to_arrow(timeout=timeout)


class AsyncTable:
    """`AsyncTable` (python/python/lancedb/table.py:5749-5830): the hot-path part."""

    def __init__(self, table: Table):
        self._table = table
        self.name = table.name

    async def schema(self) -> pa.Schema:
        return self._table.schema

    async def count_rows(self, filter: Optional[str] = None) -> int:
        if filter is None:
            return self._table.count_rows()
        return int(_filter.evaluate(self._table._data, filter).sum())

    async def to_arrow(self) -> pa.Table:
        return self._table.to_arrow()

    async def list_indices(self):
        return self._table.list_indices()

    async def create_index(self, column: str, *, config: Optional[Union[IvfPq, IvfRq, IvfFlat]] = None,
                           replace: bool = True, accelerator: Optional[str] = "cuda"):
        cfg = config or IvfPq()
        kind = "IVF_RQ" if isinstance(cfg, IvfRq) else ("IVF_FLAT" if isinstance(cfg, IvfFlat) else "IVF_PQ")
        await asyncio.to_thread(
            self._table.create_index, metric=cfg.distance_type, num_partitions=cfg.num_partitions,
            num_sub_vectors=getattr(cfg, "num_sub_vectors", None), vector_column_name=column, replace=replace,
            accelerator=accelerator, index_type=kind, num_bits=getattr(cfg, "num_bits", 8),
            max_iterations=cfg.max_iterations, sample_rate=cfg.sample_rate)

    async def prewarm_index(self, name: str):
        return self._table.prewarm_index(name)

    def query(self) -> AsyncQuery:
        return AsyncQuery(self._table)

    def vector_search(self, query_vector) -> AsyncVectorQuery:
        return self.query().nearest_to(query_vector)


class AsyncConnection:
    def __init__(self, conn: DBConnection):
        self._conn = conn

    async def create_table(self, name: str, data=None, **kw) -> AsyncTable:
        return AsyncTable(self._conn.create_table(name, data, **kw))

    async def open_table(self, name: str) -> AsyncTable:
        return AsyncTable(self._conn.open_table(name))

    async def table_names(self) -> Iterable[str]:
        return self._conn.table_names()

    async def drop_table(self, name: str):
        self._conn.drop_table(name)


async def connect_async(uri: str = "memory://", *, device: int = 0, **_ignored) -> AsyncConnection:
    return AsyncConnection(DBConnection(uri, device))

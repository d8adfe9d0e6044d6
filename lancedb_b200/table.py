"""In-memory table + connection mirroring the part of the reference's surface that leads
into the vector-query hot path: `connect() -> create_table() -> create_index() ->
search()...to_arrow()` (python/python/lancedb/table.py:3571-3664,
2883-2937; rust/lancedb/src/table.rs:549-613 `BaseTable`).

The storage engine, catalog, write path and versioning of LanceDB are out of scope
(SURVEY.md 2b rows 9-18): a table here is a pyarrow Table held in host memory whose vector
column (and, after `create_index`, the IVF_PQ arrays) are pinned in HBM.  Row ids are the
row positions, like a single-fragment Lance dataset.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Union

import numpy as np
import pyarrow as pa

from . import _native
from .index import (RQ_MAX_DIM, IvfBinaryIndexData, IvfPqIndexData, IvfRqIndexData, IvfSqIndexData,
                    train_ivf_binary, train_ivf_pq, train_ivf_rq, train_ivf_sq)
from .query import LanceVectorQueryBuilder


def _to_arrow_table(data, schema: Optional[pa.Schema] = None) -> pa.Table:
    """`data` as an arrow table; with `schema`, built against it (a fixed_size_list<uint8> field holds packed binary
    vectors, not the float32 lists that lists of numbers become without one)."""
    if schema is not None:
        return _to_arrow_table(data).select(schema.names).cast(schema)
    if isinstance(data, pa.Table):
        return data
    if isinstance(data, dict):
        cols = {}
        for k, v in data.items():
            a = np.asarray(v)
            if a.ndim == 2:
                cols[k] = pa.FixedSizeListArray.from_arrays(pa.array(a.reshape(-1).astype(np.float32)), a.shape[1])
            else:
                cols[k] = pa.array(v)
        return pa.table(cols)
    if isinstance(data, list):
        names = list(data[0].keys())
        cols = {}
        for n in names:
            vals = [r[n] for r in data]
            if isinstance(vals[0], (list, tuple, np.ndarray)) and not isinstance(vals[0], str):
                a = np.asarray(vals, dtype=np.float32)
                cols[n] = pa.FixedSizeListArray.from_arrays(pa.array(a.reshape(-1)), a.shape[1])
            else:
                cols[n] = pa.array(vals)
        return pa.table(cols)
    try:
        import pandas as pd
        if isinstance(data, pd.DataFrame):
            return _to_arrow_table({c: list(data[c]) for c in data.columns})
    except ImportError:
        pass
    raise TypeError(f"unsupported data type {type(data)}")


def _vector_columns(schema: pa.Schema) -> List[str]:
    return [f.name for f in schema if (pa.types.is_fixed_size_list(f.type) and
            (pa.types.is_floating(f.type.value_type) or pa.types.is_uint8(f.type.value_type))) or
            _is_multivec_type(f.type)]


def _is_multivec_type(t: pa.DataType) -> bool:
    """list<fixed_size_list<f16|f32|f64, dim>> (or large_list): a multivector column, searched by late interaction
    (rust/lancedb/src/table/query.rs:180-199, the `DataType::List` branch)."""
    return ((pa.types.is_list(t) or pa.types.is_large_list(t)) and pa.types.is_fixed_size_list(t.value_type) and
            pa.types.is_floating(t.value_type.value_type))


def _is_binary_type(t: pa.DataType) -> bool:
    """fixed_size_list<uint8, nbytes>: packed binary vectors, searched by Hamming distance."""
    return pa.types.is_fixed_size_list(t) and pa.types.is_uint8(t.value_type)


class Table:
    def __init__(self, name: str, data: pa.Table, device: int = 0):
        self.name = name
        self._data = data
        self._device = device
        self._flat: Dict[str, _native.GpuFlat] = {}
        self._binary: Dict[str, _native.GpuBinary] = {}
        self._multivec: Dict[str, _native.GpuMultivec] = {}
        self._index: Dict[str, _native.GpuIvfPq] = {}
        self._index_data: Dict[str, Union[IvfPqIndexData, IvfSqIndexData, IvfRqIndexData, IvfBinaryIndexData]] = {}

    # ---- introspection ----
    @property
    def schema(self) -> pa.Schema:
        return self._data.schema

    def count_rows(self) -> int:
        return self._data.num_rows

    def __len__(self) -> int:
        return self._data.num_rows

    def to_arrow(self) -> pa.Table:
        return self._data

    def to_pandas(self):
        return self._data.to_pandas()

    def _index_type(self, column: str) -> str:
        d = self._index_data[column]
        if isinstance(d, IvfBinaryIndexData):
            return "IVF_FLAT"
        return "IVF_SQ" if isinstance(d, IvfSqIndexData) else ("IVF_RQ" if isinstance(d, IvfRqIndexData) else "IVF_PQ")

    def list_indices(self):
        return [{"name": f"{c}_idx", "index_type": self._index_type(c), "columns": [c]} for c in self._index]

    def index_stats(self, index_name: str):
        """python/python/tests/test_index.py:366-372: every row is indexed (there is no append path here)."""
        col = index_name[:-4] if index_name.endswith("_idx") else index_name
        if col not in self._index_data:
            return None
        d = self._index_data[col]
        return {"index_type": self._index_type(col), "distance_type": d.metric, "num_indexed_rows": d.nrows,
                "num_unindexed_rows": self.count_rows() - d.nrows, "num_indices": 1}

    def _vectors(self, column: str) -> np.ndarray:
        col = self._data.column(column).combine_chunks()
        dim = col.type.list_size
        return np.asarray(col.flatten().to_numpy(zero_copy_only=False), np.float32).reshape(-1, dim)

    def _dim(self, column: str) -> int:
        t = self._data.schema.field(column).type
        return t.value_type.list_size if _is_multivec_type(t) else t.list_size

    def _is_binary(self, column: str) -> bool:
        return _is_binary_type(self._data.schema.field(column).type)

    def _is_multivec(self, column: str) -> bool:
        return _is_multivec_type(self._data.schema.field(column).type)

    def _multivec_rows(self, column: str):
        """(values [T, dim] f32, offsets [N+1] u64) of a multivector column; a null row holds no vectors.  Stored
        float16 / float64 elements are upcast to f32."""
        col = self._data.column(column).combine_chunks()
        lens = col.value_lengths().fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
        inner = col.flatten()                               # skips the values behind null rows
        if inner.null_count:
            raise ValueError(f"multivector column {column!r} holds a null vector inside a row")
        dim = col.type.value_type.list_size
        vals = np.asarray(inner.flatten().to_numpy(zero_copy_only=False), np.float32).reshape(-1, dim)
        return vals, _native.multivec_offsets(lens)

    def _binary_vectors(self, column: str) -> np.ndarray:
        col = self._data.column(column).combine_chunks()
        return np.asarray(col.flatten().to_numpy(zero_copy_only=False), np.uint8).reshape(-1, col.type.list_size)

    # ---- index build (parameters of Index::IvfPq; training itself is not the hot path) ----
    def create_index(self, metric: str = "l2", num_partitions: Optional[int] = None,
                     num_sub_vectors: Optional[int] = None, vector_column_name: Optional[str] = None,
                     replace: bool = True, accelerator: Optional[str] = None, index_type: str = "IVF_PQ",
                     num_bits: int = 8, max_iterations: int = 50, sample_rate: int = 256, **_ignored):
        kind = index_type.upper()
        if kind == "IVF_FLAT":             # binary columns only: IvfFlat(distance_type="hamming")
            column = vector_column_name or self._infer_vector_column(None)
            if self._is_multivec(column):
                raise NotImplementedError("no index over multivector columns on the GPU path: they are searched flat")
            if not self._is_binary(column):
                raise NotImplementedError("IVF_FLAT is served over binary (fixed_size_list<uint8>) columns only; index "
                                          "float columns with IVF_PQ, IVF_SQ or IVF_RQ")
            if metric.lower() != "hamming":
                raise ValueError(f"IVF_FLAT over binary vectors supports the hamming distance type only, not {metric!r}")
            if column in self._index and not replace:
                raise RuntimeError(f"index {column}_idx already exists (pass replace=True)")
            dev = f"cuda:{self._device}" if accelerator in ("cuda", "gpu") else None
            self._attach_index(column, train_ivf_binary(self._binary_vectors(column), num_partitions=num_partitions,
                                                        max_iterations=max_iterations, sample_rate=sample_rate,
                                                        device=dev))
            return
        if kind not in ("IVF_PQ", "IVF_SQ", "IVF_RQ"):
            raise NotImplementedError("only IVF_PQ, IVF_SQ and IVF_RQ are on the GPU hot path")
        if kind == "IVF_RQ" and num_bits != 1:
            # RaBitQ with 1 bit per dimension only (extended RaBitQ is not served); the legacy default of 8 is refused
            # rather than quietly building a 1-bit index
            raise ValueError(f"IVF_RQ supports num_bits=1 only, got num_bits={num_bits}")
        if kind == "IVF_PQ" and num_bits not in (4, 8):
            raise ValueError(f"IVF_PQ supports num_bits 4 or 8, got num_bits={num_bits}")
        if kind == "IVF_SQ" and num_bits != 8:
            raise ValueError("only num_bits=8 is supported")
        column = vector_column_name or self._infer_vector_column(None)
        if self._is_binary(column):
            raise NotImplementedError("no index over binary vectors on the GPU path: search them flat (hamming)")
        if self._is_multivec(column):
            raise NotImplementedError("no index over multivector columns on the GPU path: they are searched flat")
        if kind in ("IVF_SQ", "IVF_RQ") and metric.lower() not in ("l2", "cosine"):
            raise ValueError(f"{kind} supports the l2 and cosine distance types, not {metric!r}")
        if kind == "IVF_RQ" and self._dim(column) > RQ_MAX_DIM:
            raise ValueError(f"IVF_RQ supports dimensions up to {RQ_MAX_DIM}, got {self._dim(column)}")
        if column in self._index and not replace:
            raise RuntimeError(f"index {column}_idx already exists (pass replace=True)")   # python/python/tests/test_index.py:357
        dev = None
        if accelerator in ("cuda", "gpu"):
            dev = f"cuda:{self._device}"
        if kind == "IVF_SQ":               # IvfSqIndexBuilder: distance_type, num_partitions, max_iterations, sample_rate
            self._attach_index(column, train_ivf_sq(self._vectors(column), num_partitions=num_partitions,
                                                    distance_type=metric, max_iterations=max_iterations,
                                                    sample_rate=sample_rate, keep_vectors=True, device=dev,
                                                    native_passes=dev is not None))
            return
        if kind == "IVF_RQ":               # IvfRqIndexBuilder: distance_type, num_partitions, num_bits, max_iterations, sample_rate
            self._attach_index(column, train_ivf_rq(self._vectors(column), num_partitions=num_partitions,
                                                    distance_type=metric, num_bits=num_bits,
                                                    max_iterations=max_iterations, sample_rate=sample_rate,
                                                    keep_vectors=True, device=dev, native_passes=dev is not None))
            return
        data = train_ivf_pq(self._vectors(column), num_partitions=num_partitions,
                            num_sub_vectors=num_sub_vectors, distance_type=metric,
                            max_iterations=max_iterations, sample_rate=sample_rate,
                            keep_vectors=True, device=dev, num_bits=num_bits,
                            native_passes=dev is not None)      # accelerator: row passes through the C ABI (build.cu)
        self._attach_index(column, data)

    def _attach_index(self, column: str,
                      data: Union[IvfPqIndexData, IvfSqIndexData, IvfRqIndexData, IvfBinaryIndexData]):
        if column in self._index:
            self._index[column].close()
        self._index_data[column] = data
        cls = (_native.GpuIvfBinary if isinstance(data, IvfBinaryIndexData) else
               _native.GpuIvfSq if isinstance(data, IvfSqIndexData) else
               _native.GpuIvfRq if isinstance(data, IvfRqIndexData) else _native.GpuIvfPq)
        self._index[column] = cls(data, device=self._device)

    # ---- on-disk Lance index (SURVEY.md 8f-3; layout [lance, recalled], see lance_index.py) ----
    def load_lance_index(self, index_dir: str, vector_column_name: Optional[str] = None) -> None:
        """Pin the IVF_PQ index stored under ``<table>.lance/_indices/<uuid>/`` in HBM.  Row ids must be row offsets
        of this table (what a freshly written Lance table has); the raw vectors for ``refine_factor`` are gathered
        from the table's own column in the index's partition order."""
        from .lance_index import read_ivf_pq_index
        data = read_ivf_pq_index(index_dir)
        column = vector_column_name or self._infer_vector_column(None)
        if self._dim(column) != data.dim:
            raise ValueError(f"index dimension {data.dim} does not match column {column} ({self._dim(column)})")
        if data.nrows and int(data.row_ids.max()) >= self._data.num_rows:
            raise ValueError("the index addresses rows this table does not have")
        data.vectors = np.ascontiguousarray(self._vectors(column)[data.row_ids.astype(np.int64)])
        self._attach_index(column, data)

    def save_lance_index(self, index_dir: str, vector_column_name: Optional[str] = None, transposed: bool = True) -> None:
        from .lance_index import write_ivf_pq_index
        column = vector_column_name or self._infer_vector_column(None)
        if self._index_type(column) != "IVF_PQ":
            raise NotImplementedError("only IVF_PQ indexes are written as Lance index files")
        if self._index_data[column].num_bits != 8:
            raise NotImplementedError("only 8-bit IVF_PQ indexes are written as Lance index files")
        write_ivf_pq_index(index_dir, self._index_data[column], transposed=transposed)

    def prewarm_index(self, name: str):           # rust/lancedb/src/table.rs:3283-3286
        return None                                # indexes are pinned in HBM at create/open time

    # ---- search ----
    def _infer_vector_column(self, query) -> str:
        cols = _vector_columns(self.schema)
        if query is not None:
            qdim = np.asarray(query).shape[-1]
            match = [c for c in cols if self._dim(c) == qdim]
            if len(match) == 1:
                return match[0]
            if not match:
                raise ValueError(f"No vector column found to match with the query vector dimension: {qdim}")
            cols = match
        if len(cols) == 1:
            return cols[0]
        if not cols:
            raise ValueError("There is no vector column in the table")
        raise ValueError(f"Table has multiple vector columns: {cols}. Please specify vector_column_name")

    def search(self, query=None, vector_column_name: Optional[str] = None, query_type: str = "auto",
               **_ignored) -> LanceVectorQueryBuilder:
        if query is None or isinstance(query, str):
            raise NotImplementedError("only vector queries are on the GPU hot path")
        column = vector_column_name or self._infer_vector_column(query)
        return LanceVectorQueryBuilder(self, query, column)

    def _vector_search(self, queries: np.ndarray, *, column, k, nprobes, refine_factor, distance_type,
                       lower, upper, use_index, allow_mask=None, max_nprobes=0, timeout_ms=0):
        allow, allow_bits = None, 0
        if allow_mask is not None:                 # prefilter: row-id allow-list as the C ABI's bitmap
            allow, allow_bits = _native.mask_bitmap(allow_mask), int(len(allow_mask))
        if self._is_binary(column):                # rust/lancedb/src/table/query.rs:229-236 (is_binary)
            if distance_type is not None and distance_type != "hamming":
                raise ValueError(f"distance type {distance_type!r} is not supported on binary column {column!r}: "
                                 "use 'hamming'")
            q = _native.binary_components(queries)   # the builder's f32 copy: integers are exact up to 2^24
            idx = self._index.get(column) if use_index else None
            if idx is not None:                    # IVF_FLAT (hamming); bypass_vector_index() searches flat below
                return idx.search(q, k=k, nprobes=nprobes, refine_factor=refine_factor or 0, lower=lower, upper=upper,
                                  allow=allow, allow_bits=allow_bits,
                                  max_nprobes=max_nprobes if allow is not None else 0, timeout_ms=timeout_ms)
            bx = self._binary.get(column)
            if bx is None:
                bx = self._binary[column] = _native.GpuBinary(self._binary_vectors(column), device=self._device)
            return bx.search(q, k=k, lower=lower, upper=upper, allow=allow, allow_bits=allow_bits, timeout_ms=timeout_ms)
        if self._is_multivec(column):              # rust/lancedb/src/table/query.rs:180-199: ONE query of nq vectors
            if distance_type is not None and distance_type != "cosine":
                raise ValueError(f"distance type {distance_type!r} is not supported on multivector column {column!r}: "
                                 "only cosine is")
            mv = self._multivec.get(column)
            if mv is None:
                vals, off = self._multivec_rows(column)
                mv = self._multivec[column] = _native.GpuMultivec(vals, off, device=self._device)
            return mv.search([np.asarray(queries, np.float32)], k=k, lower=lower, upper=upper, allow=allow,
                             allow_bits=allow_bits, timeout_ms=timeout_ms)
        if distance_type == "hamming":
            raise ValueError(f"distance type 'hamming' needs a binary (fixed_size_list<uint8>) column; {column!r} "
                             "holds floats")
        idx = self._index.get(column) if use_index else None
        if idx is not None:
            if distance_type is not None and distance_type != idx.metric:
                # the reference documents this as invalid results; be explicit instead
                raise ValueError(f"distance_type {distance_type!r} does not match the index's {idx.metric!r}")
            return idx.search(queries, k=k, nprobes=nprobes, refine_factor=refine_factor or 0,
                              lower=lower, upper=upper, allow=allow, allow_bits=allow_bits,
                              max_nprobes=max_nprobes if allow is not None else 0, timeout_ms=timeout_ms)
        fl = self._flat.get(column)
        if fl is None:
            fl = self._flat[column] = _native.GpuFlat(self._vectors(column), device=self._device)
        metric = distance_type or "l2"
        if metric not in ("l2", "cosine", "dot"):
            raise ValueError(f"unsupported distance type {metric!r}")
        return fl.search(queries, k=k, metric=metric, lower=lower, upper=upper, allow=allow, allow_bits=allow_bits,
                         timeout_ms=timeout_ms)

    def _take(self, row_ids: np.ndarray, columns: Optional[List[str]]) -> pa.Table:
        t = self._data if columns is None else self._data.select(columns)
        return t.take(pa.array(np.asarray(row_ids, np.int64)))


class DBConnection:
    """`lancedb.connect()` stand-in: an in-memory catalog of tables."""

    def __init__(self, uri: str = "memory://", device: int = 0):
        self.uri = uri
        self._device = device
        self._tables: Dict[str, Table] = {}

    def create_table(self, name: str, data=None, schema: Optional[pa.Schema] = None, mode: str = "create",
                     exist_ok: bool = False, **_ignored) -> Table:
        if name in self._tables and mode != "overwrite" and not exist_ok:
            raise ValueError(f"Table {name} already exists")
        if name in self._tables and exist_ok and mode != "overwrite":
            return self._tables[name]
        if data is None:
            if schema is None:
                raise ValueError("Either data or schema must be provided")
            data = schema.empty_table()                      # an empty table is searchable (returns no rows)
        t = Table(name, _to_arrow_table(data, schema), self._device)
        self._tables[name] = t
        return t

    def open_table(self, name: str) -> Table:
        if name not in self._tables:
            raise ValueError(f"Table {name} does not exist")
        return self._tables[name]

    def table_names(self) -> Iterable[str]:
        return sorted(self._tables)

    def drop_table(self, name: str):
        self._tables.pop(name, None)


def connect(uri: str = "memory://", *, device: int = 0, **_ignored) -> DBConnection:
    return DBConnection(uri, device)

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

import threading
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional

import numpy as np
import pyarrow as pa

from . import _native
from . import filter as _filter
from .index import IVF_KINDS
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


# create_index's refusal of a column of the other kind, by the column an index kind needs
_WRONG_COLUMN = {
    "float": "no index over binary vectors on the GPU path: search them flat (hamming)",
    "binary": "IVF_FLAT is served over binary (fixed_size_list<uint8>) columns only; index float columns with IVF_PQ, "
              "IVF_SQ or IVF_RQ",
}


@dataclass
class DeleteResult:
    """What Table.delete returns (python/python/lancedb/table.py:1672-1720)."""
    num_deleted_rows: int
    version: int


class Table:
    def __init__(self, name: str, data: pa.Table, device: int = 0):
        self.name = name
        self._data = data
        self._device = device
        # deleted rows stay in _data as tombstones, so a row's id (its position) never changes: _live is the mask of
        # the rows not deleted (None: nothing was deleted).  Every GPU handle holding a deleted row has been told so
        # (its .delete), and so leaves it out of every search.
        self._live: Optional[np.ndarray] = None
        self.version = 1                              # +1 for every add or delete that changes rows
        self._lock = threading.RLock()                # serialises add, delete and optimize
        self._flat: Dict[str, _native.GpuFlat] = {}
        self._binary: Dict[str, _native.GpuBinary] = {}
        self._multivec: Dict[str, _native.GpuMultivec] = {}
        self._index: Dict[str, _native.GpuIvfPq] = {}
        self._index_data: Dict[str, object] = {}      # the IndexData of one of IVF_KINDS
        # rows added after an indexed column's index was built: a flat handle over them (GpuFlat / GpuBinary, row ids =
        # table positions) and the position of the first
        self._tail: Dict[str, object] = {}
        self._tail_from: Dict[str, int] = {}

    # ---- introspection ----
    @property
    def schema(self) -> pa.Schema:
        return self._data.schema

    def count_rows(self) -> int:
        return self._data.num_rows if self._live is None else int(self._live.sum())

    def __len__(self) -> int:
        return self.count_rows()

    def to_arrow(self) -> pa.Table:
        return self._data if self._live is None else self._data.filter(pa.array(self._live))

    def to_pandas(self):
        return self.to_arrow().to_pandas()

    def _deleted(self) -> np.ndarray:
        """The ids (positions) of the deleted rows, u64."""
        return np.zeros(0, np.uint64) if self._live is None else np.nonzero(~self._live)[0].astype(np.uint64)

    def _live_positions(self) -> Optional[np.ndarray]:
        """The ids of the live rows, u64, or None when nothing was deleted."""
        return None if self._live is None else np.nonzero(self._live)[0].astype(np.uint64)

    def _where_mask(self, where: str) -> np.ndarray:
        """The rows (by position) that are live and satisfy the SQL predicate `where`."""
        mask = _filter.evaluate(self._data, where)
        return mask if self._live is None else mask & self._live

    def _index_type(self, column: str) -> str:
        return self._index_data[column].index_type

    def list_indices(self):
        return [{"name": f"{c}_idx", "index_type": self._index_type(c), "columns": [c]} for c in self._index]

    def index_stats(self, index_name: str):
        """python/python/tests/test_index.py:366-372: rows added after the index was built count as unindexed until
        optimize() folds them in."""
        col = index_name[:-4] if index_name.endswith("_idx") else index_name
        if col not in self._index_data:
            return None
        d = self._index_data[col]
        indexed = d.nrows if self._live is None else int(self._live[d.row_ids.astype(np.int64)].sum())
        return {"index_type": self._index_type(col), "distance_type": d.metric, "num_indexed_rows": indexed,
                "num_unindexed_rows": self.count_rows() - indexed, "num_indices": 1}

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
        """(values [T, dim], offsets [N+1] u64) of a multivector column (_multivec_rows_of)."""
        return self._multivec_rows_of(self._data, column)

    @staticmethod
    def _multivec_rows_of(table: pa.Table, column: str):
        """(values [T, dim], offsets [N+1] u64) of a multivector column of `table`; a null row holds no vectors.
        float16 elements stay float16 (GpuMultivec keeps them so, with the results of their exact f32 upcast); float64
        elements are converted to f32."""
        col = table.column(column).combine_chunks()
        lens = col.value_lengths().fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
        inner = col.flatten()                               # skips the values behind null rows
        if inner.null_count:
            raise ValueError(f"multivector column {column!r} holds a null vector inside a row")
        dim = col.type.value_type.list_size
        dt = np.float16 if pa.types.is_float16(col.type.value_type.value_type) else np.float32
        vals = np.asarray(inner.flatten().to_numpy(zero_copy_only=False), dt).reshape(-1, dim)
        return vals, _native.multivec_offsets(lens)

    def _binary_vectors(self, column: str) -> np.ndarray:
        col = self._data.column(column).combine_chunks()
        return np.asarray(col.flatten().to_numpy(zero_copy_only=False), np.uint8).reshape(-1, col.type.list_size)

    # ---- index build (parameters of Index::IvfPq; training itself is not the hot path) ----
    def create_index(self, metric: str = "l2", num_partitions: Optional[int] = None,
                     num_sub_vectors: Optional[int] = None, vector_column_name: Optional[str] = None,
                     replace: bool = True, accelerator: Optional[str] = None, index_type: str = "IVF_PQ",
                     num_bits: int = 8, max_iterations: int = 50, sample_rate: int = 256, m: int = 20,
                     ef_construction: int = 300, **_ignored):
        kind = IVF_KINDS.get(index_type.upper())
        if kind is None:
            raise NotImplementedError("only IVF_PQ, IVF_SQ, IVF_HNSW_SQ and IVF_RQ are on the GPU hot path")
        if kind.num_bits and num_bits not in kind.num_bits:
            raise ValueError(kind.num_bits_error.format(num_bits=num_bits))
        column = vector_column_name or self._infer_vector_column(None)
        if self._is_multivec(column):
            raise NotImplementedError("no index over multivector columns on the GPU path: they are searched flat")
        if self._is_binary(column) != (kind.column == "binary"):
            raise NotImplementedError(_WRONG_COLUMN[kind.column])
        if metric.lower() not in kind.metrics:
            raise ValueError(kind.metric_error.format(kind=kind.index_type, metric=metric))
        if kind.max_dim is not None and self._dim(column) > kind.max_dim:
            raise ValueError(f"{kind.index_type} supports dimensions up to {kind.max_dim}, got {self._dim(column)}")
        if column in self._index and not replace:
            raise RuntimeError(f"index {column}_idx already exists (pass replace=True)")   # python/python/tests/test_index.py:357
        dev = f"cuda:{self._device}" if accelerator in ("cuda", "gpu") else None
        args = {"num_sub_vectors": num_sub_vectors, "num_bits": num_bits, "m": m, "ef_construction": ef_construction}
        kw = {p: args[p] for p in kind.params}
        if kind.column == "binary":
            vectors = self._binary_vectors(column)
        else:       # accelerator: the row passes run through the C ABI (build.cu); keep the raw vectors for refine
            vectors = self._vectors(column)
            kw.update(keep_vectors=True, native_passes=dev is not None)
        live = self._live_positions()
        if live is not None:        # trained on the live rows, which keep their positions as row ids
            vectors = vectors[live.astype(np.int64)]
            kw.update(row_ids=live)
        self._attach_index(column, kind.train(vectors, num_partitions=num_partitions, distance_type=metric,
                                              max_iterations=max_iterations, sample_rate=sample_rate, device=dev, **kw))

    def _attach_index(self, column: str, data):
        if column in self._index:
            self._index[column].close()
        self._drop_tail(column)                 # the new index holds every row the table has
        self._index_data[column] = data
        self._index[column] = self._open_index(column)

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

    # ---- appends and index maintenance (python/python/lancedb/table.py:3393, 3970) ----
    def add(self, data, mode: str = "append", on_bad_vectors: str = "error", **_ignored) -> None:
        with self._lock:
            self._add(data, mode, on_bad_vectors)

    def _add(self, data, mode: str, on_bad_vectors: str) -> None:
        """Append rows with the table's schema.  Row ids are table positions.  An indexed column's new rows are not
        indexed: they go to its tail, which every vector search scans exactly and merges with the index's result
        (unless fast_search()), until optimize() folds them into the index.
        on_bad_vectors="error" (the reference's default, and the only policy served): a float vector holding a NaN is
        refused (python/python/lancedb/table.py:4429-4445), and so is a row the column's index could not take at
        optimize(): an infinite component, or a zero vector under a cosine index.  A multivector row holding a null vector
        is refused too.  A refused call changes nothing."""
        if mode == "overwrite":
            raise NotImplementedError("add(mode='overwrite') is not supported: only appends are")
        if mode != "append":
            raise ValueError(f"mode must be 'append' or 'overwrite', got {mode!r}")
        if on_bad_vectors != "error":
            raise NotImplementedError(f"on_bad_vectors={on_bad_vectors!r} is not supported: only 'error' is")
        new = _to_arrow_table(data)
        if sorted(new.column_names) != sorted(self.schema.names):
            raise ValueError(f"the data's columns {new.column_names} do not match the table's schema "
                             f"{self.schema.names}")
        try:
            new = new.select(self.schema.names).cast(self.schema)
        except (pa.ArrowInvalid, pa.ArrowNotImplementedError, pa.ArrowTypeError, ValueError) as e:
            raise ValueError(f"the data does not match the table's schema: {e}") from None
        n0, n = self._data.num_rows, new.num_rows          # positions, tombstones included: the new ids
        if n == 0:
            return
        rows = {c: self._rows_of(new, c) for c in _vector_columns(self.schema) if not self._is_multivec(c)}
        for c, x in rows.items():
            self._check_new_rows(c, x)
        # (values, offsets) of every multivector column: a row holding a null vector is refused here, before anything
        # changes, as a search of the column would refuse it
        mv_rows = {c: self._multivec_rows_of(new, c) for c in _vector_columns(self.schema) if self._is_multivec(c)}
        ids = np.arange(n0, n0 + n, dtype=np.uint64)
        done = []                   # the tails grow before the table does: a failure leaves the table as it was
        try:
            for column in self._index:
                if column in self._tail:
                    self._tail[column].append(rows[column], ids)
                else:
                    cls = _native.GpuBinary if self._is_binary(column) else _native.GpuFlat
                    self._tail[column] = cls(rows[column], row_ids=ids, device=self._device)
                    self._tail_from[column] = n0
                done.append(column)
        except BaseException:
            for column in done:    # back to the rows the table holds
                start = self._tail_from[column]
                self._drop_tail(column)
                if start < n0:
                    self._open_tail(column, start)
            raise
        self._data = pa.concat_tables([self._data, new]).combine_chunks()
        if self._live is not None:
            self._live = np.concatenate([self._live, np.ones(n, bool)])
        for cache in (self._flat, self._binary, self._multivec):    # full-column caches grow in place (ids = positions)
            for column in list(cache):
                new_rows = mv_rows[column] if cache is self._multivec else (rows[column],)
                try:   # (a cache opened over the live rows holds explicit ids: the new ones are passed)
                    cache[column].append(*new_rows, row_ids=None if self._live is None else ids)
                except BaseException:
                    cache.pop(column).close()             # reopened from the table on the next search
                    raise
        self.version += 1

    def _check_new_rows(self, column: str, x: np.ndarray) -> None:
        if self._is_binary(column):
            return
        bad = np.isnan(x).any(axis=1)
        if bad.any():
            raise ValueError(f"Vector column '{column}' has NaNs (row {int(np.nonzero(bad)[0][0])} of the data)")
        if column in self._index:
            bad = np.isinf(x).any(axis=1)
            if self._index_data[column].metric == "cosine":
                bad |= ~(np.square(x.astype(np.float32)).sum(axis=1) > 0)
            if bad.any():
                raise ValueError(f"row {int(np.nonzero(bad)[0][0])} of the data cannot join column '{column}''s "
                                 "index: an infinite component, or a zero vector under cosine")

    @staticmethod
    def _rows_of(table: pa.Table, column: str) -> np.ndarray:
        """The vectors of a float or binary (u8) column of `table`, as the flat handles keep them: float16 columns as
        float16 (GpuFlat keeps them so in HBM, with the results of their exact f32 upcast), other floats as f32."""
        col = table.column(column).combine_chunks()
        vt = col.type.value_type
        dt = np.uint8 if pa.types.is_uint8(vt) else (np.float16 if pa.types.is_float16(vt) else np.float32)
        return np.asarray(col.flatten().to_numpy(zero_copy_only=False), dt).reshape(-1, col.type.list_size)

    def _new_rows(self, column: str, start: int) -> np.ndarray:
        """The vectors of rows start.. of a float or binary (u8) column (_rows_of)."""
        return self._rows_of(self._data.slice(start), column)

    def _drop_tail(self, column: str) -> None:
        tail = self._tail.pop(column, None)
        if tail is not None:
            tail.close()
        self._tail_from.pop(column, None)

    def _open_tail(self, column: str, start: int) -> None:
        """The tail of `column` from the table's rows start.. (ids = positions), told of the deleted ones."""
        cls = _native.GpuBinary if self._is_binary(column) else _native.GpuFlat
        rows = self._new_rows(column, start)
        tail = cls(rows, device=self._device, row_ids=np.arange(start, start + rows.shape[0], dtype=np.uint64))
        dead = self._deleted()
        dead = dead[dead >= start]
        if dead.size:
            tail.delete(dead)
        self._tail[column], self._tail_from[column] = tail, start

    def _open_index(self, column: str):
        """The handle of `column`'s IndexData, told of the deleted rows it holds."""
        data = self._index_data[column]
        h = getattr(_native, IVF_KINDS[data.index_type].handle)(data, device=self._device)
        dead = self._deleted()
        if dead.size:
            held = np.zeros(self._data.num_rows, bool)
            held[data.row_ids.astype(np.int64)] = True
            dead = dead[held[dead.astype(np.int64)]]
            if dead.size:
                h.delete(dead)
        return h

    # ---- deletes (python/python/lancedb/table.py:1672-1720) ----
    def delete(self, where: str) -> DeleteResult:
        """Delete the rows that satisfy the SQL predicate `where`; returns DeleteResult(num_deleted_rows, version).
        The rows stay in place as tombstones, so every other row keeps its _rowid; each GPU handle holding one is told
        (lgpu_*_delete) and leaves it out of every later search, exactly as a prefilter would.  optimize() drops them
        from the handles.  A failed delete leaves the table and every handle as they were."""
        if not isinstance(where, str) or not where.strip():
            raise ValueError("delete needs a non-empty SQL predicate")
        with self._lock:
            ids = np.nonzero(self._where_mask(where))[0].astype(np.uint64)
            if ids.size == 0:
                return DeleteResult(0, self.version)
            # (handle, the ids it holds, how to open it again from the table's rows and tombstones)
            todo = []
            for column, idx in self._index.items():
                start = self._tail_from.get(column)
                held = ids if start is None else ids[ids < start]
                todo.append((idx, held, lambda c=column: self._reopen_index(c)))
            for column, tail in self._tail.items():
                start = self._tail_from[column]
                todo.append((tail, ids[ids >= start], lambda c=column, s=start: self._open_tail(c, s)))
            for cache in (self._flat, self._binary, self._multivec):
                for column, h in cache.items():
                    todo.append((h, ids, lambda c=cache, col=column: c.pop(col).close()))   # reopened lazily
            done = []
            try:
                for h, held, reopen in todo:
                    if held.size:
                        done.append(reopen)
                        h.delete(held)
            except BaseException:
                for reopen in done:
                    reopen()
                raise
            live = np.ones(self._data.num_rows, bool) if self._live is None else self._live.copy()
            live[ids.astype(np.int64)] = False
            self._live = live
            self.version += 1
            return DeleteResult(int(ids.size), self.version)

    def _reopen_index(self, column: str) -> None:
        self._index[column].close()
        self._index[column] = self._open_index(column)

    def optimize(self, *, cleanup_older_than=None, delete_unverified: bool = False, retrain: bool = False) -> None:
        """Fold every indexed column's unindexed rows into its index without retraining (IndexData.extend: the fitted
        centroids and quantiser), then reopen it.  Compaction and version cleanup have nothing to do here."""
        if retrain:
            raise NotImplementedError("optimize(retrain=True) is not supported: rows are added with the index's model")
        with self._lock:
            for column in list(self._tail):
                start = self._tail_from[column]
                rows = self._new_rows(column, start)
                if rows.dtype == np.float16:      # an index holds the f32 upcast of a float16 column
                    rows = rows.astype(np.float32)
                ids = np.arange(start, start + rows.shape[0], dtype=np.uint64)
                self._attach_index(column, self._index_data[column].extend(rows, ids, device=self._device))
            if self._live is None:
                return
            # deleted rows leave every handle (IndexData.compact: no retraining).  The host rows stay, so row ids do
            # not change: unlike a Lance compaction, which renumbers row addresses unless stable row ids are on.
            for column in list(self._index):
                data = self._index_data[column]
                keep = self._live[data.row_ids.astype(np.int64)]
                if not keep.all():
                    self._attach_index(column, data.compact(keep))
            for cache in (self._flat, self._binary, self._multivec):    # reopened over the live rows
                for h in cache.values():
                    h.close()
                cache.clear()

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
                       lower, upper, use_index, allow_mask=None, max_nprobes=0, timeout_ms=0, ef=0,
                       fast_search=False):
        allow, allow_bits = None, 0
        if allow_mask is not None:                 # prefilter: row-id allow-list as the C ABI's bitmap
            allow, allow_bits = _native.mask_bitmap(allow_mask), int(len(allow_mask))
        # deleted rows make every request prefiltered (the handles filter them out): maximum_nprobes applies
        widen = max_nprobes if (allow is not None or self._live is not None) else 0
        if self._is_binary(column):                # rust/lancedb/src/table/query.rs:229-236 (is_binary)
            if distance_type is not None and distance_type != "hamming":
                raise ValueError(f"distance type {distance_type!r} is not supported on binary column {column!r}: "
                                 "use 'hamming'")
            q = _native.binary_components(queries)   # the builder's f32 copy: integers are exact up to 2^24
            idx = self._index.get(column) if use_index else None
            if idx is not None:                    # IVF_FLAT (hamming); bypass_vector_index() searches flat below
                kw = dict(k=k, nprobes=nprobes, refine_factor=refine_factor or 0, lower=lower, upper=upper, allow=allow,
                          allow_bits=allow_bits, max_nprobes=widen, timeout_ms=timeout_ms)
                tail = None if fast_search else self._tail.get(column)
                return idx.search(q, **kw) if tail is None else idx.search_unindexed(tail, q, **kw)
            bx = self._binary.get(column)
            if bx is None:
                bx = self._binary[column] = self._open_cache(_native.GpuBinary, self._binary_vectors(column))
            return bx.search(q, k=k, lower=lower, upper=upper, allow=allow, allow_bits=allow_bits, timeout_ms=timeout_ms)
        if self._is_multivec(column):              # rust/lancedb/src/table/query.rs:180-199: ONE query of nq vectors
            if distance_type is not None and distance_type != "cosine":
                raise ValueError(f"distance type {distance_type!r} is not supported on multivector column {column!r}: "
                                 "only cosine is")
            mv = self._multivec.get(column)
            if mv is None:
                vals, off = self._multivec_rows(column)
                rid = self._live_positions()
                if rid is not None:                # the live rows' vectors, with their positions as row ids
                    lens = np.diff(off.astype(np.int64))[rid.astype(np.int64)]
                    vals = vals[np.repeat(self._live, np.diff(off.astype(np.int64)))]
                    off = _native.multivec_offsets(lens)
                mv = self._multivec[column] = _native.GpuMultivec(vals, off, row_ids=rid, device=self._device)
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
            kw = dict(k=k, nprobes=nprobes, refine_factor=refine_factor or 0, lower=lower, upper=upper, allow=allow,
                      allow_bits=allow_bits, max_nprobes=widen, timeout_ms=timeout_ms, ef=ef)
            tail = None if fast_search else self._tail.get(column)   # rows added since the index was built
            return idx.search(queries, **kw) if tail is None else idx.search_unindexed(tail, queries, **kw)
        fl = self._flat.get(column)
        if fl is None:
            fl = self._flat[column] = self._open_cache(_native.GpuFlat, self._rows_of(self._data, column))
        metric = distance_type or "l2"
        if metric not in ("l2", "cosine", "dot"):
            raise ValueError(f"unsupported distance type {metric!r}")
        return fl.search(queries, k=k, metric=metric, lower=lower, upper=upper, allow=allow, allow_bits=allow_bits,
                         timeout_ms=timeout_ms)

    def _open_cache(self, cls, x: np.ndarray):
        """A full-column cache (GpuFlat / GpuBinary) over the column's rows x: every row (ids = positions), or the live
        rows with their positions as ids."""
        rid = self._live_positions()
        if rid is None:
            return cls(x, device=self._device)
        return cls(np.ascontiguousarray(x[rid.astype(np.int64)]), row_ids=rid, device=self._device)

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

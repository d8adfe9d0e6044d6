"""Query builder mirroring the reference's vector-search surface.

Same names, argument meaning, defaults and error behaviour as
`lancedb.query.LanceVectorQueryBuilder` (python/python/lancedb/query.py:1552-1862)
and the request it lowers to, `VectorQueryRequest`
(rust/lancedb/src/query.rs:1066-1114): limit 10, nprobes 20 (min == max),
no refine, L2.  Everything below `to_arrow()` runs on the GPU through the C ABI; only the
`Take` of the non-vector columns for the k result rows (SURVEY.md 8a row a12) happens in
pyarrow on the host.  `where(...)` filters: the predicate is evaluated on the host (filter.py) and its
row-id allow-list goes to the GPU as a bitmap (prefilter, the default, `lgpu_search_filtered`) or is
applied to the k results (postfilter).  FTS and rerankers are outside the hot path and raise
NotImplementedError.
"""
from __future__ import annotations

from typing import List, Optional, Union

import numpy as np
import pyarrow as pa

from . import filter as _filter
from ._native import K_MAX

DEFAULT_TOP_K = 10          # rust/lancedb/src/query.rs:36
DEFAULT_NPROBES = 20        # rust/lancedb/src/query.rs:1097-1113


class LanceVectorQueryBuilder:
    def __init__(self, table, query, vector_column: str):
        self._table = table
        if isinstance(query, (list, tuple)) and (len(query) == 0 or (isinstance(query[0], (list, tuple)) and len(query[0]) == 0)):
            raise ValueError("Vector query must be a non-empty list")      # ensure_vector_query, query.py:332-350
        q = np.asarray(query, dtype=np.float32)      # every query vector is cast to Float32 (query.rs:1013)
        # on a multivector column a 2-D query is ONE query of several vectors, with no query_index column
        # (rust/lancedb/src/table/query.rs:180-199; python/python/lancedb/query.py:3376-3382)
        is_mv = getattr(table, "_is_multivec", None)
        self._multivector = bool(is_mv(vector_column)) if is_mv is not None else False
        if q.ndim == 1:
            q = q[None, :]
            self._multi = False
        elif q.ndim == 2:
            self._multi = q.shape[0] > 1 and not self._multivector
        else:
            raise ValueError("query must be a vector or a list of vectors")
        self._query = np.ascontiguousarray(q)
        self._vector_column = vector_column
        self._distance_type: Optional[str] = None
        self._minimum_nprobes: Optional[int] = None
        self._maximum_nprobes: Optional[int] = None
        self._lower_bound: Optional[float] = None
        self._upper_bound: Optional[float] = None
        self._refine_factor: Optional[int] = None
        self._ef: Optional[int] = None
        self._limit: Optional[int] = None
        self._offset: int = 0
        self._columns: Optional[List[str]] = None
        self._with_row_id = False
        self._use_index = True
        self._fast_search = False
        self._where: Optional[str] = None
        self._postfilter = False

    # ---- setters (same names as the reference) ----
    def metric(self, metric: str) -> "LanceVectorQueryBuilder":
        return self.distance_type(metric)

    def distance_type(self, distance_type: str) -> "LanceVectorQueryBuilder":
        self._distance_type = distance_type.lower()
        return self

    def nprobes(self, nprobes: int) -> "LanceVectorQueryBuilder":
        self._minimum_nprobes = nprobes
        self._maximum_nprobes = nprobes
        return self

    def minimum_nprobes(self, n: int) -> "LanceVectorQueryBuilder":
        self._minimum_nprobes = n
        return self

    def maximum_nprobes(self, n: int) -> "LanceVectorQueryBuilder":
        self._maximum_nprobes = n
        return self

    def distance_range(self, lower_bound: Optional[float] = None,
                       upper_bound: Optional[float] = None) -> "LanceVectorQueryBuilder":
        self._lower_bound = lower_bound
        self._upper_bound = upper_bound
        return self

    def refine_factor(self, refine_factor: int) -> "LanceVectorQueryBuilder":
        self._refine_factor = refine_factor
        return self

    def ef(self, ef: int) -> "LanceVectorQueryBuilder":
        """The HNSW search beam (python/python/lancedb/query.py:1719, rust/lancedb/src/query.rs:1290-1300): IVF_HNSW_SQ
        keeps the max(ef, limit x refine_factor) best rows seen per probed partition; unset means 1.5 x limit.  Other
        index kinds ignore it."""
        if int(ef) <= 0:
            raise ValueError("ef must be greater than 0")
        self._ef = int(ef)
        return self

    def limit(self, limit: Optional[int]) -> "LanceVectorQueryBuilder":
        if limit is None or limit <= 0:
            raise ValueError("Limit is required for ANN/KNN queries and must be greater than 0")
        self._limit = int(limit)
        return self

    def offset(self, offset: int) -> "LanceVectorQueryBuilder":
        self._offset = max(0, int(offset or 0))
        return self

    def select(self, columns: List[str]) -> "LanceVectorQueryBuilder":
        self._columns = list(columns)
        return self

    def with_row_id(self, with_row_id: bool = True) -> "LanceVectorQueryBuilder":
        self._with_row_id = with_row_id
        return self

    def bypass_vector_index(self) -> "LanceVectorQueryBuilder":
        """Exhaustive flat search even when an index exists (use_index = false)."""
        self._use_index = False
        return self

    def fast_search(self) -> "LanceVectorQueryBuilder":
        """Search the index alone: rows added since it was built (Table.add) are skipped until optimize() folds them
        in (python/python/lancedb/query.py:1950-1961).  Without an index it changes nothing."""
        self._fast_search = True
        return self

    def where(self, where: str, prefilter: Optional[bool] = None) -> "LanceVectorQueryBuilder":
        """SQL predicate over the table's columns; calling it again ANDs the filters
        (python/python/lancedb/query.py:1864-1892).  prefilter (default): rows are excluded before the
        vector search; prefilter=False: the filter is applied to the search's results, which can
        then be fewer than `limit` (rust/lancedb/src/query.rs:489-507)."""
        if not isinstance(where, str):
            raise NotImplementedError("only SQL string filters are supported (no Expr objects)")
        self._where = _filter.combine(self._where, where)
        if prefilter is not None:
            self._postfilter = not prefilter
        return self

    def postfilter(self) -> "LanceVectorQueryBuilder":
        self._postfilter = True
        return self

    def rerank(self, *a, **k):
        raise NotImplementedError("rerankers are out of scope")

    # ---- execution ----
    def _resolve(self):
        lim = self._limit if self._limit is not None else DEFAULT_TOP_K
        k = lim + self._offset                          # table/query.rs:231
        if k > K_MAX:                                   # (k x refine_factor is checked by the kinds that re-rank)
            raise ValueError(f"limit + offset = {k} is above {K_MAX} (LGPU_K_MAX), the largest k the GPU search serves")
        # The request starts at minimum_nprobes = 20, maximum_nprobes = Some(20) (query.rs:1097-1113) and the sync builder
        # is lowered onto it as python/python/lancedb/table.py:5777-5787 does: both set -> nprobes(min) then
        # maximum_nprobes(max); one set -> that setter alone, validated against the OTHER one's default of 20
        # (query.rs:1232-1275).  maximum_nprobes 0 means "no limit" (python/src/query.rs:949-954).
        mn, mx = self._minimum_nprobes, self._maximum_nprobes
        min_np = mn if mn is not None else DEFAULT_NPROBES
        max_np = mx if mx is not None else DEFAULT_NPROBES
        if min_np <= 0:
            raise ValueError("minimum_nprobes must be greater than 0")     # query.rs:1233-1236
        if mx is None and min_np > DEFAULT_NPROBES:
            raise ValueError("minimum_nprobes must be less than or equal to maximum_nprobes")   # query.rs:1238-1245
        if max_np != 0 and max_np < min_np:
            raise ValueError("maximum_nprobes must be greater than or equal to minimum_nprobes")  # query.rs:1268-1273
        # with no filter every probed partition yields rows, so min == effective probes;
        # maximum_nprobes only matters for filtered queries (query.py:1676-1692, query.rs:1250-1275):
        # 0 = "search as many partitions as needed" -> every partition
        return k, lim, min_np, (max_np if max_np != 0 else (1 << 30))

    @staticmethod
    def _timeout_ms(timeout) -> int:
        """QueryExecutionOptions.timeout (datetime.timedelta or seconds) -> ms for the C ABI; None/0 = none."""
        if timeout is None:
            return 0
        sec = timeout.total_seconds() if hasattr(timeout, "total_seconds") else float(timeout)
        if sec <= 0:
            raise ValueError("timeout must be positive")
        return max(1, int(round(sec * 1000.0)))

    def to_arrow(self, *, timeout=None) -> pa.Table:
        k, lim, nprobes, max_nprobes = self._resolve()
        timeout_ms = self._timeout_ms(timeout)
        t = self._table
        if self._query.shape[1] != t._dim(self._vector_column):
            raise ValueError(
                f"No vector column found to match with the query vector dimension: {self._query.shape[1]}")
        if t.count_rows() == 0:
            # searching an empty table returns no rows (python/python/tests/test_query.py:1990-2004), not an error
            tbl = t._take(np.zeros(0, np.int64), self._columns)
            tbl = tbl.append_column("_distance", pa.array(np.zeros(0, np.float32), pa.float32()))
            if self._with_row_id:
                tbl = tbl.append_column("_rowid", pa.array(np.zeros(0, np.uint64), pa.uint64()))
            if self._multi:
                tbl = tbl.append_column("query_index", pa.array(np.zeros(0, np.int32), pa.int32()))
            return tbl
        mask = None
        if self._where is not None:
            mask = t._where_mask(self._where)                      # row id == row position; live rows only
        ids, dist, cnt = t._vector_search(
            self._query, column=self._vector_column, k=k, nprobes=nprobes,
            refine_factor=self._refine_factor, distance_type=self._distance_type,
            lower=self._lower_bound, upper=self._upper_bound, use_index=self._use_index,
            allow_mask=None if (mask is None or self._postfilter) else mask,
            max_nprobes=max_nprobes, timeout_ms=timeout_ms, **({"ef": self._ef} if self._ef else {}),
            **({"fast_search": True} if self._fast_search else {}))
        out = []
        for qi in range(len(cnt)):                         # one result list per query (a multivector query is one)
            n = int(cnt[qi])
            row_ids, row_dist = ids[qi, :n], dist[qi, :n]
            if mask is not None and self._postfilter:              # filter the vector search's results
                keep = mask[row_ids.astype(np.int64)]
                row_ids, row_dist = row_ids[keep], row_dist[keep]
            sel_ids = row_ids[self._offset:][:lim]
            sel_dist = row_dist[self._offset:][:lim]
            tbl = t._take(sel_ids, self._columns)
            tbl = tbl.append_column("_distance", pa.array(sel_dist, pa.float32()))
            if self._with_row_id:
                tbl = tbl.append_column("_rowid", pa.array(sel_ids, pa.uint64()))
            if self._multi:                                # table/query.rs:360-366
                tbl = tbl.append_column("query_index", pa.array(np.full(len(sel_ids), qi, np.int32)))
            out.append(tbl)
        return pa.concat_tables(out) if len(out) > 1 else out[0]

    def to_batches(self, max_batch_length: Optional[int] = None, *, timeout=None):
        """MaxBatchLengthStream (rust/lancedb/src/utils/mod.rs:395): the result re-chunked to <= 1024 rows."""
        tbl = self.to_arrow(timeout=timeout)
        return pa.RecordBatchReader.from_batches(tbl.schema, tbl.to_batches(max_chunksize=max_batch_length or 1024))

    def to_pandas(self, *, timeout=None, **kw):
        return self.to_arrow(timeout=timeout).to_pandas(**kw)

    def to_list(self, *, timeout=None) -> list:
        return self.to_arrow(timeout=timeout).to_pylist()

"""The remote vector-query wire format (SURVEY.md 8f-4): `POST /v1/table/{name}/query/`, JSON request, Arrow IPC
*file* response -- so that the GPU path can sit behind the reference's own remote client as a query node.

Request schema: what `RemoteTable::apply_query_params` + `apply_vector_query_params` emit
(rust/lancedb/src/remote/table.rs:724-830, 833-929), pinned by the reference's mock-server tests
(`test_query_vector_default_values` :4650-4671, `test_query_vector_all_params` :4798-4873):
    prefilter, k, offset?, filter?, columns?, with_row_id?, fast_search?, version,
    distance_type?, nprobes (= minimum_nprobes, for old servers), minimum_nprobes, maximum_nprobes (0 = unbounded),
    lower_bound, upper_bound, ef, refine_factor, vector_column?, bypass_vector_index?,
    vector: [f32...] or [[f32...], ...] (multi-vector; an empty list = no vector).
`build_query_body` is the client half (what the reference client sends for a given builder state);
`handle_query` is the server half: it turns a body into calls on this package's Table / query builder and returns
the bytes of an Arrow IPC file (content type `application/vnd.apache.arrow.file`), which is what
`RemoteTable::read_arrow_stream` expects (remote/table.rs, ARROW_FILE_CONTENT_TYPE).
Nothing here touches the network: transport, auth and the rest of the REST surface are out of scope.
"""
from __future__ import annotations

import io
import json
from typing import Any, Dict, List, Optional, Union

import numpy as np
import pyarrow as pa

QUERY_PATH = "/v1/table/{name}/query/"
JSON_CONTENT_TYPE = "application/json"
ARROW_FILE_CONTENT_TYPE = "application/vnd.apache.arrow.file"
_ISIZE_MAX = (1 << 63) - 1          # remote/table.rs:741-743: a missing limit travels as isize::MAX


def build_query_body(vector, *, k: Optional[int] = 10, offset: Optional[int] = None, prefilter: bool = True,
                     filter: Optional[str] = None, columns: Optional[List[str]] = None, with_row_id: bool = False,
                     fast_search: bool = False, distance_type: Optional[str] = None, minimum_nprobes: int = 20,
                     maximum_nprobes: Optional[int] = 20, lower_bound: Optional[float] = None,
                     upper_bound: Optional[float] = None, ef: Optional[int] = None, refine_factor: Optional[int] = None,
                     vector_column: Optional[str] = None, bypass_vector_index: bool = False,
                     version: Optional[int] = None) -> Dict[str, Any]:
    """The JSON body the reference's remote client sends for a vector query."""
    body: Dict[str, Any] = {"prefilter": bool(prefilter), "k": _ISIZE_MAX if k is None else int(k), "version": version}
    if offset is not None:
        body["offset"] = int(offset)
    if filter is not None:
        body["filter"] = filter
    if columns is not None:
        body["columns"] = list(columns)
    if fast_search:
        body["fast_search"] = True
    if with_row_id:
        body["with_row_id"] = True
    if distance_type is not None:
        body["distance_type"] = distance_type.lower()
    body["nprobes"] = int(minimum_nprobes)
    body["minimum_nprobes"] = int(minimum_nprobes)
    body["maximum_nprobes"] = 0 if maximum_nprobes is None else int(maximum_nprobes)
    body["lower_bound"] = lower_bound
    body["upper_bound"] = upper_bound
    body["ef"] = ef
    body["refine_factor"] = refine_factor
    if vector_column is not None:
        body["vector_column"] = vector_column
    if bypass_vector_index:
        body["bypass_vector_index"] = True
    v = np.asarray(vector, np.float32)
    if v.size == 0:
        body["vector"] = []                               # "Server takes empty vector, not null or undefined"
    elif v.ndim == 1:
        body["vector"] = [float(x) for x in v]            # f32 widened to f64, as serde_json::Number::from_f64(v as f64)
    else:
        body["vector"] = [[float(x) for x in row] for row in v]
    return body


def _ipc_file(table: pa.Table) -> bytes:
    sink = io.BytesIO()
    with pa.ipc.new_file(sink, table.schema) as w:
        w.write_table(table)
    return sink.getvalue()


def read_ipc_file(data: bytes) -> pa.Table:
    return pa.ipc.open_file(io.BytesIO(data)).read_all()


def handle_query(table, body: Union[str, bytes, Dict[str, Any]]) -> bytes:
    """Serve one `/v1/table/{name}/query/` request against `table` (a lancedb_b200.Table): returns the Arrow IPC
    file bytes of the result.  Unsupported request features raise ValueError / NotImplementedError, which a server
    maps to HTTP 400."""
    if isinstance(body, (str, bytes)):
        body = json.loads(body)
    vec = body.get("vector", [])
    if vec is None or len(vec) == 0:
        raise NotImplementedError("plain (non-vector) queries are not on the GPU hot path")
    if body.get("full_text_query") is not None:
        raise NotImplementedError("full-text queries are out of scope")
    q = table.search(np.asarray(vec, np.float32), vector_column_name=body.get("vector_column"))
    k = body.get("k")
    if k is None or int(k) <= 0:
        raise ValueError("Limit is required for ANN/KNN queries and must be greater than 0")
    q = q.limit(min(int(k), 1 << 20))
    if body.get("offset"):
        q = q.offset(int(body["offset"]))
    if body.get("distance_type"):
        q = q.distance_type(str(body["distance_type"]))
    min_np = body.get("minimum_nprobes", body.get("nprobes"))          # old clients only send nprobes
    if min_np is not None:
        q = q.minimum_nprobes(int(min_np))
    max_np = body.get("maximum_nprobes")
    if max_np is not None:
        q = q.maximum_nprobes(int(max_np))                              # 0 = as many partitions as needed
    elif min_np is not None:
        q = q.maximum_nprobes(int(min_np))
    if body.get("lower_bound") is not None or body.get("upper_bound") is not None:
        q = q.distance_range(body.get("lower_bound"), body.get("upper_bound"))
    if body.get("refine_factor"):
        q = q.refine_factor(int(body["refine_factor"]))
    if body.get("bypass_vector_index"):
        q = q.bypass_vector_index()
    if body.get("fast_search"):
        q = q.fast_search()
    if body.get("filter"):
        q = q.where(str(body["filter"]), prefilter=bool(body.get("prefilter", True)))
    cols = body.get("columns")
    if isinstance(cols, dict):
        raise NotImplementedError("computed (dynamic) columns are out of scope")
    if cols is not None:
        q = q.select(list(cols))
    if body.get("with_row_id"):
        q = q.with_row_id(True)
    out = q.to_arrow()
    if body.get("order_by"):
        keys = [(o["column_name"], "ascending" if o.get("ascending", True) else "descending") for o in body["order_by"]]
        out = out.sort_by(keys)
    return _ipc_file(out)

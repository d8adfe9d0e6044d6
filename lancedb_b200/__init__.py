"""lancedb_b200 -- H100-native (sm_90a) implementation of LanceDB's vector-query hot path.

Scope: `Table.search(...)...to_arrow()` over an IVF_PQ, IVF_SQ, IVF_HNSW_SQ or IVF_RQ index and the flat brute-force path
(SURVEY.md section 8).  Compute lives in hand-written CUDA behind the C ABI of
include/lancedb_b200.h (lancedb_b200/csrc); this package is the Python host-side mirror of
the reference's builder surface plus a ctypes binding.  There is no CPU fallback.
"""
from .index import (IvfPqIndexData, IvfSqIndexData, IvfHnswSqIndexData, IvfRqIndexData, IvfBinaryIndexData,
                    train_ivf_pq, train_ivf_sq, train_ivf_hnsw_sq, train_ivf_rq, train_ivf_binary, suggested_num_sub_vectors, suggested_num_partitions)
from .query import LanceVectorQueryBuilder, DEFAULT_TOP_K, DEFAULT_NPROBES
from .table import DBConnection, DeleteResult, Table, connect
from .aio import AsyncConnection, AsyncTable, HnswSq, IvfFlat, IvfRq, connect_async

__all__ = [
    "connect", "connect_async", "DBConnection", "AsyncConnection", "Table", "AsyncTable", "DeleteResult", "LanceVectorQueryBuilder", "IvfPqIndexData", "train_ivf_pq",
    "IvfSqIndexData", "train_ivf_sq", "IvfHnswSqIndexData", "train_ivf_hnsw_sq", "HnswSq", "IvfRqIndexData", "train_ivf_rq", "IvfRq",
    "IvfBinaryIndexData", "train_ivf_binary", "IvfFlat",
    "suggested_num_sub_vectors", "suggested_num_partitions", "DEFAULT_TOP_K", "DEFAULT_NPROBES",
]
__version__ = "0.1.0"

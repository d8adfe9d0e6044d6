"""ctypes binding of the C ABI in include/lancedb_b200.h.

This is the same binding a non-Python host would write (see INTEGRATION.md for the Rust
`extern "C"` version).  There is no CPU fallback: if the shared library is missing or no
CUDA device is present, every compute call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "liblancedb_b200.so")
_lib = None

LGPU_OK, LGPU_INVALID_INPUT, LGPU_RUNTIME, LGPU_TIMEOUT, LGPU_OOM = 0, 1, 2, 3, 4
METRICS = {"l2": 0, "euclidean": 0, "cosine": 1, "dot": 2}
ABI_VERSION = 2

EXPORTS = [
    "lgpu_last_error", "lgpu_abi_version", "lgpu_device_count",
    "lgpu_index_open", "lgpu_index_close", "lgpu_index_device_bytes", "lgpu_last_scanned_code_bytes",
    "lgpu_search", "lgpu_search_filtered", "lgpu_search_device", "lgpu_merge_topk_device",
    "lgpu_search_async", "lgpu_ticket_poll", "lgpu_ticket_wait", "lgpu_search_coalesced",
    "lgpu_comm_unique_id", "lgpu_comm_init", "lgpu_comm_destroy", "lgpu_search_sharded", "lgpu_search_sharded_device",
    "lgpu_comm_last_stage_ms",
    "lgpu_flat_open", "lgpu_flat_close", "lgpu_flat_search", "lgpu_flat_search_filtered", "lgpu_flat_search_device",
    "lgpu_ivf_assign", "lgpu_pq_encode", "lgpu_kmeans_train", "lgpu_pq_train",
    "lgpu_debug_coarse", "lgpu_debug_partition_distances", "lgpu_debug_filter_bounds", "lgpu_debug_gemm",
    "lgpu_debug_sub_batch_size", "lgpu_last_stage_ms", "lgpu_set_profiling",
    "lgpu_kernel_launch_count", "lgpu_last_filter_stats",
    "lgpu_binary_open", "lgpu_binary_close", "lgpu_binary_search", "lgpu_binary_search_filtered",
    "lgpu_binary_search_device", "lgpu_debug_hamming_gemm",
    "lgpu_multivec_open", "lgpu_multivec_close", "lgpu_multivec_search", "lgpu_multivec_search_filtered",
    "lgpu_multivec_search_device", "lgpu_debug_maxsim_gemm",
    "lgpu_ivf_sq_open", "lgpu_debug_sq_distances",
    "lgpu_ivf_rq_open", "lgpu_debug_rq_distances",
    "lgpu_debug_pq4_sums",
    "lgpu_ivf_binary_open", "lgpu_ivf_binary_close", "lgpu_ivf_binary_search", "lgpu_ivf_binary_search_filtered",
    "lgpu_ivf_binary_search_device", "lgpu_debug_ivf_hamming_scan",
]
MULTIVEC_MAX_NQ = 4096          # vectors per multivector query (include/lancedb_b200.h)
MULTIVEC_MAX_ROW = 1 << 20      # vectors per multivector row
MULTIVEC_MAX_DIM = 65536


class IndexDesc(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("dim", C.c_uint32), ("nlist", C.c_uint32), ("m", C.c_uint32),
        ("nbits", C.c_uint32), ("metric", C.c_int32), ("codes_layout", C.c_int32), ("device", C.c_int32),
        ("nrows", C.c_uint64),
        ("centroids", C.c_void_p), ("codebook", C.c_void_p), ("part_offsets", C.c_void_p),
        ("codes", C.c_void_p), ("row_ids", C.c_void_p), ("vectors", C.c_void_p),
    ]


class SqDesc(C.Structure):
    """lgpu_ivf_sq_desc"""
    _fields_ = [
        ("abi_version", C.c_uint32), ("dim", C.c_uint32), ("nlist", C.c_uint32), ("metric", C.c_int32),
        ("device", C.c_int32), ("reserved", C.c_uint32), ("nrows", C.c_uint64), ("lo", C.c_double), ("hi", C.c_double),
        ("centroids", C.c_void_p), ("part_offsets", C.c_void_p), ("codes", C.c_void_p), ("row_ids", C.c_void_p),
        ("vectors", C.c_void_p),
    ]


class RqDesc(C.Structure):
    """lgpu_ivf_rq_desc"""
    _fields_ = [
        ("abi_version", C.c_uint32), ("dim", C.c_uint32), ("nlist", C.c_uint32), ("metric", C.c_int32),
        ("device", C.c_int32), ("num_bits", C.c_uint32), ("nrows", C.c_uint64),
        ("centroids", C.c_void_p), ("rotation", C.c_void_p), ("part_offsets", C.c_void_p), ("codes", C.c_void_p),
        ("add_factors", C.c_void_p), ("scale_factors", C.c_void_p), ("row_ids", C.c_void_p), ("vectors", C.c_void_p),
    ]


class IvfBinaryDesc(C.Structure):
    """lgpu_ivf_binary_desc"""
    _fields_ = [
        ("abi_version", C.c_uint32), ("nbytes", C.c_uint32), ("nlist", C.c_uint32), ("device", C.c_int32),
        ("nrows", C.c_uint64), ("centroids", C.c_void_p), ("part_offsets", C.c_void_p), ("vectors", C.c_void_p),
        ("row_ids", C.c_void_p),
    ]


class SearchParams(C.Structure):
    _fields_ = [
        ("k", C.c_uint32), ("nprobes", C.c_uint32), ("refine_factor", C.c_uint32),
        ("has_lower", C.c_int32), ("has_upper", C.c_int32), ("lower", C.c_float), ("upper", C.c_float),
        ("flags", C.c_uint32), ("max_nprobes", C.c_uint32), ("timeout_ms", C.c_uint32),
    ]


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    r = subprocess.run(cmd, capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("building liblancedb_b200.so failed:\n" + (r.stdout or "") + (r.stderr or ""))
    return LIB_PATH


def load():
    """Load the shared library; raises ImportError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("LGPU_LIB_PATH") or LIB_PATH      # kernel A/B builds (csrc/Makefile OUT=...)
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(lancedb_b200 has no CPU fallback)")
    lib = C.CDLL(path)
    vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int
    lib.lgpu_last_error.restype = C.c_char_p
    lib.lgpu_abi_version.restype = u32
    lib.lgpu_device_count.argtypes = [C.POINTER(C.c_int)]
    lib.lgpu_index_open.argtypes = [C.POINTER(IndexDesc), C.POINTER(vp)]
    lib.lgpu_index_close.argtypes = [vp]
    lib.lgpu_index_close.restype = None
    lib.lgpu_index_device_bytes.argtypes = [vp, C.POINTER(C.c_uint64)]
    lib.lgpu_last_scanned_code_bytes.argtypes = [C.POINTER(C.c_uint64)]
    lib.lgpu_search.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_search_async.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, C.POINTER(vp)]
    lib.lgpu_ticket_poll.argtypes = [vp, C.POINTER(C.c_int)]
    lib.lgpu_ticket_wait.argtypes = [vp]
    lib.lgpu_search_coalesced.argtypes = [vp, vp, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_search_filtered.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, C.c_uint64, vp, vp, vp]
    lib.lgpu_search_device.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_merge_topk_device.argtypes = [i32, u32, u32, u32, vp, vp, vp, vp, vp, vp]
    lib.lgpu_comm_unique_id.argtypes = [vp, C.c_size_t]
    lib.lgpu_comm_init.argtypes = [vp, C.c_size_t, i32, i32, i32, C.POINTER(vp)]
    lib.lgpu_comm_destroy.argtypes = [vp]
    lib.lgpu_comm_destroy.restype = None
    lib.lgpu_search_sharded.argtypes = [vp, vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_search_sharded_device.argtypes = [vp, vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_comm_last_stage_ms.argtypes = [vp, vp]
    lib.lgpu_flat_open.argtypes = [vp, C.c_uint64, u32, vp, i32, C.POINTER(vp)]
    lib.lgpu_flat_close.argtypes = [vp]
    lib.lgpu_flat_close.restype = None
    lib.lgpu_ivf_assign.argtypes = [vp, u32, u32, i32, vp, C.c_uint64, i32, vp]
    lib.lgpu_pq_encode.argtypes = [vp, vp, u32, u32, u32, i32, vp, vp, C.c_uint64, i32, vp]
    lib.lgpu_kmeans_train.argtypes = [vp, C.c_uint64, u32, vp, u32, u32, i32, C.POINTER(C.c_double)]
    lib.lgpu_pq_train.argtypes = [vp, C.c_uint64, u32, u32, vp, u32, i32]
    lib.lgpu_flat_search.argtypes = [vp, i32, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_flat_search_filtered.argtypes = [vp, i32, vp, u32, C.POINTER(SearchParams), vp, C.c_uint64, vp, vp, vp]
    lib.lgpu_flat_search_device.argtypes = [vp, i32, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_debug_coarse.argtypes = [vp, vp, u32, u32, vp, vp]
    lib.lgpu_debug_partition_distances.argtypes = [vp, vp, u32, vp]
    lib.lgpu_debug_filter_bounds.argtypes = [vp, vp, u32, u32, C.c_uint64, vp, vp, vp, vp, vp]
    lib.lgpu_debug_gemm.argtypes = [vp, vp, u32, C.c_uint64, u32, i32, vp]
    lib.lgpu_debug_sub_batch_size.argtypes = [vp, u32, u32, C.POINTER(u32)]
    lib.lgpu_last_stage_ms.argtypes = [vp]
    lib.lgpu_set_profiling.argtypes = [i32]
    lib.lgpu_kernel_launch_count.argtypes = [C.POINTER(C.c_uint64)]
    lib.lgpu_binary_open.argtypes = [vp, C.c_uint64, u32, vp, i32, C.POINTER(vp)]
    lib.lgpu_binary_close.argtypes = [vp]
    lib.lgpu_binary_close.restype = None
    lib.lgpu_binary_search.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_binary_search_filtered.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, C.c_uint64, vp, vp, vp]
    lib.lgpu_binary_search_device.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_debug_hamming_gemm.argtypes = [vp, vp, u32, C.c_uint64, u32, i32, vp]
    lib.lgpu_multivec_open.argtypes = [vp, vp, C.c_uint64, u32, vp, i32, C.POINTER(vp)]
    lib.lgpu_multivec_close.argtypes = [vp]
    lib.lgpu_multivec_close.restype = None
    lib.lgpu_multivec_search.argtypes = [vp, vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_multivec_search_filtered.argtypes = [vp, vp, vp, u32, C.POINTER(SearchParams), vp, C.c_uint64, vp, vp, vp]
    lib.lgpu_multivec_search_device.argtypes = [vp, vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_debug_maxsim_gemm.argtypes = [vp, u32, vp, vp, C.c_uint64, u32, i32, vp]
    lib.lgpu_ivf_sq_open.argtypes = [C.POINTER(SqDesc), C.POINTER(vp)]
    lib.lgpu_debug_sq_distances.argtypes = [vp, u32, vp, C.c_uint64, u32, i32, vp]
    lib.lgpu_ivf_rq_open.argtypes = [C.POINTER(RqDesc), C.POINTER(vp)]
    lib.lgpu_debug_rq_distances.argtypes = [vp, u32, vp, vp, vp, C.c_uint64, u32, i32, i32, vp, vp]
    lib.lgpu_debug_pq4_sums.argtypes = [vp, u32, vp, C.c_uint64, u32, i32, vp]
    lib.lgpu_ivf_binary_open.argtypes = [C.POINTER(IvfBinaryDesc), C.POINTER(vp)]
    lib.lgpu_ivf_binary_close.argtypes = [vp]
    lib.lgpu_ivf_binary_close.restype = None
    lib.lgpu_ivf_binary_search.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp]
    lib.lgpu_ivf_binary_search_filtered.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, C.c_uint64, vp, vp, vp]
    lib.lgpu_ivf_binary_search_device.argtypes = [vp, vp, u32, C.POINTER(SearchParams), vp, vp, vp, vp]
    lib.lgpu_debug_ivf_hamming_scan.argtypes = [vp, u32, vp, C.c_uint64, u32, i32, vp]
    for name in EXPORTS:
        getattr(lib, name)          # every declared symbol must be exported
    if lib.lgpu_abi_version() != ABI_VERSION:
        raise ImportError("liblancedb_b200.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def check(rc: int) -> None:
    """Map an lgpu_status onto the exception the reference's Python surface raises
    (InvalidInput -> ValueError, Runtime -> RuntimeError: python/python/tests/test_query.py:917-929)."""
    if rc == LGPU_OK:
        return
    msg = (load().lgpu_last_error() or b"").decode("utf-8", "replace")
    if rc == LGPU_INVALID_INPUT:
        raise ValueError(msg)
    if rc == LGPU_TIMEOUT:
        raise TimeoutError(msg)
    if rc == LGPU_OOM:
        raise MemoryError(msg)
    raise RuntimeError(msg)


def device_count() -> int:
    n = C.c_int(0)
    check(load().lgpu_device_count(C.byref(n)))
    return n.value


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def make_params(k=10, nprobes=20, refine_factor=0, lower=None, upper=None, max_nprobes=0,
                timeout_ms=0) -> SearchParams:
    return SearchParams(int(k), int(nprobes), int(refine_factor or 0), lower is not None, upper is not None,
                        0.0 if lower is None else float(lower), 0.0 if upper is None else float(upper), 0,
                        int(max_nprobes or 0), int(timeout_ms or 0))


class _Handle:
    """A library handle (`_h`) that `_close`, the name of its C close function, releases."""
    _close = ""

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            getattr(_lib, self._close)(self._h)
            self._h = None

    __del__ = close


def _host_search(fn: str, head, B: int, k: int, p: SearchParams, allow, allow_bits):
    """Host-buffer search through `fn`, or through `fn`_filtered with `allow` (u32 bitmap over row ids, `allow_bits`
    bits); `head` are the arguments before the params.  Returns (ids [B,k] u64, dist [B,k] f32, count [B] u32)."""
    ids = np.empty((B, k), np.uint64); dist = np.empty((B, k), np.float32); cnt = np.empty(B, np.uint32)
    if allow is None:
        check(getattr(load(), fn)(*head, C.byref(p), _ptr(ids), _ptr(dist), _ptr(cnt)))
    else:
        bm = np.ascontiguousarray(allow, np.uint32)
        if bm.size * 32 < allow_bits:
            raise ValueError("allow bitmap shorter than allow_bits")
        check(getattr(load(), fn + "_filtered")(*head, C.byref(p), _ptr(bm), int(allow_bits), _ptr(ids), _ptr(dist),
                                                _ptr(cnt)))
    return ids, dist, cnt


def binary_components(queries) -> np.ndarray:
    """Query components for a binary vector column: integers in [0, 255] (checked, not wrapped as a cast would) ->
    uint8."""
    a = np.asarray(queries)
    if a.dtype != np.uint8:
        if not (np.issubdtype(a.dtype, np.integer) or np.issubdtype(a.dtype, np.floating)) or (
                a.size and not (np.all(np.isfinite(a)) and np.all(a == np.round(a)) and a.min() >= 0 and
                                a.max() <= 255)):
            raise ValueError("binary query components must be integers in [0, 255]")
    return np.ascontiguousarray(a, np.uint8)


def _query_offsets(q_offsets) -> np.ndarray:
    """Multivector query offsets [B+1] -> u32, checked: they start at 0 and give every query 1..4096 vectors."""
    off = np.asarray(q_offsets, np.int64).reshape(-1)
    if off.size < 1 or off[0] != 0:
        raise ValueError("query offsets must be [B + 1] and start at 0")
    n = np.diff(off)
    if np.any(n < 1):
        raise ValueError("every multivector query needs at least one vector")
    if n.size and int(n.max()) > MULTIVEC_MAX_NQ:
        raise ValueError(f"a multivector query holds at most {MULTIVEC_MAX_NQ} vectors")
    if int(off[-1]) >= 1 << 32:
        raise ValueError("too many query vectors in one call")
    return np.ascontiguousarray(off, np.uint32)


class GpuIvfPq(_Handle):
    """An IVF_PQ index pinned in HBM (lgpu_index), 8-bit or 4-bit codes (data.num_bits)."""
    _close = "lgpu_index_close"

    def __init__(self, data, device: int = 0, with_vectors: bool = True):
        lib = load()
        data.validate()
        self.dim, self.nlist, self.m, self.metric = data.dim, data.nlist, data.m, data.metric
        self.device = device
        vec = data.vectors if with_vectors else None
        keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.codebook, np.float32),
                np.ascontiguousarray(data.part_offsets, np.uint64), np.ascontiguousarray(data.codes_t, np.uint8),
                np.ascontiguousarray(data.row_ids, np.uint64),
                None if vec is None else np.ascontiguousarray(vec, np.float32)]
        self.num_bits = data.num_bits
        desc = IndexDesc(ABI_VERSION, data.dim, data.nlist, data.m, data.num_bits, METRICS[data.metric], 1, device,
                         data.nrows, _ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), _ptr(keep[3]), _ptr(keep[4]),
                         _ptr(keep[5]))
        h = C.c_void_p()
        check(lib.lgpu_index_open(C.byref(desc), C.byref(h)))
        self._h = h
        self.has_vectors = vec is not None

    def device_bytes(self) -> int:
        b = C.c_uint64(0)
        check(load().lgpu_index_device_bytes(self._h, C.byref(b)))
        return b.value

    def search(self, queries, k=10, nprobes=20, refine_factor=0, lower=None, upper=None, allow=None, allow_bits=0,
               max_nprobes=0, timeout_ms=0):
        """Host-buffer search: returns (ids [B,k] u64, dist [B,k] f32, count [B] u32).
        `allow` (u32 bitmap over row ids, `allow_bits` bits) = prefilter allow-list."""
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        p = make_params(k, nprobes, refine_factor, lower, upper, max_nprobes, timeout_ms)
        return _host_search("lgpu_search", (self._h, _ptr(q), q.shape[0]), q.shape[0], k, p, allow, allow_bits)

    def search_into(self, q: np.ndarray, p: SearchParams, ids: np.ndarray, dist: np.ndarray, cnt: np.ndarray):
        """Host-buffer search into caller-owned (e.g. pinned) arrays; no allocation."""
        check(load().lgpu_search(self._h, q.ctypes.data, q.shape[0], C.byref(p), ids.ctypes.data,
                                 dist.ctypes.data, cnt.ctypes.data))

    def search_one(self, query, k=10, nprobes=20, refine_factor=0):
        """One query vector through the micro-batcher (lgpu_search_coalesced): concurrent callers share a batch.
        ctypes releases the GIL for the duration of the call, so Python threads do coalesce."""
        q = np.ascontiguousarray(query, np.float32).reshape(self.dim)
        ids = np.empty(k, np.uint64); dist = np.empty(k, np.float32); cnt = np.zeros(1, np.uint32)
        p = make_params(k, nprobes, refine_factor)
        check(load().lgpu_search_coalesced(self._h, _ptr(q), C.byref(p), _ptr(ids), _ptr(dist), _ptr(cnt)))
        return ids, dist, int(cnt[0])

    def search_async(self, q: np.ndarray, p: SearchParams, ids: np.ndarray, dist: np.ndarray, cnt: np.ndarray):
        """lgpu_search_async into caller-owned (pinned) arrays; returns a ticket for ticket_wait()."""
        t = C.c_void_p()
        check(load().lgpu_search_async(self._h, q.ctypes.data, q.shape[0], C.byref(p), ids.ctypes.data,
                                       dist.ctypes.data, cnt.ctypes.data, C.byref(t)))
        return t

    def search_device(self, d_q: int, B: int, p: SearchParams, d_ids: int, d_dist: int, d_cnt: int, stream: int = 0):
        """Device-pointer search (raw addresses), enqueued on `stream`, not synchronised."""
        check(load().lgpu_search_device(self._h, d_q, B, C.byref(p), d_ids, d_dist, d_cnt, stream))

    def debug_sub_batch_size(self, B: int, nprobes: int) -> int:
        """Queries per sub-batch of a search of B queries over `nprobes` probes under this process's LGPU_WS_BYTES."""
        n = C.c_uint32(0)
        check(load().lgpu_debug_sub_batch_size(self._h, int(B), int(nprobes), C.byref(n)))
        return n.value

    def debug_coarse(self, queries, nprobes):
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        B = q.shape[0]
        nprobes = min(nprobes, self.nlist)
        parts = np.empty((B, nprobes), np.uint32); dists = np.empty((B, nprobes), np.float32)
        check(load().lgpu_debug_coarse(self._h, _ptr(q), B, nprobes, _ptr(parts), _ptr(dists)))
        return parts, dists

    def debug_filter_bounds(self, queries, nprobes, ld):
        """The dense filter scan's own numbers: (parts [B, nprobes] u32, L [B, nprobes, ld] f32 with row r < n_p of
        the slot's partition valid, W [B], E [B] f32 (unscaled), bad [B] u32) -- see lgpu_debug_filter_bounds."""
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        B = q.shape[0]
        nprobes = min(nprobes, self.nlist)
        parts = np.empty((B, nprobes), np.uint32)
        L = np.full((B, nprobes, max(int(ld), 1)), np.nan, np.float32)
        W, E, bad = np.empty(B, np.float32), np.empty(B, np.float32), np.empty(B, np.uint32)
        check(load().lgpu_debug_filter_bounds(self._h, _ptr(q), B, nprobes, L.shape[2], _ptr(parts), _ptr(L), _ptr(W),
                                              _ptr(E), _ptr(bad)))
        return parts, L, W, E, bad

    def debug_partition_distances(self, query, part, n_p):
        q = np.ascontiguousarray(query, np.float32).reshape(self.dim)
        out = np.empty(n_p, np.float32)
        check(load().lgpu_debug_partition_distances(self._h, _ptr(q), int(part), _ptr(out)))
        return out


class GpuIvfSq(GpuIvfPq):
    """An IVF_SQ index pinned in HBM: an lgpu_index opened by lgpu_ivf_sq_open, so every search entry point of GpuIvfPq
    serves it.  _distance is the exact integer sum of squared code differences as f32 (l2 and cosine alike)."""

    def __init__(self, data, device: int = 0, with_vectors: bool = True):
        lib = load()
        if data.metric not in ("l2", "cosine"):
            raise ValueError(f"IVF_SQ supports the l2 and cosine distance types, not {data.metric!r}")
        data.validate()
        self.dim, self.nlist, self.metric = data.dim, data.nlist, data.metric
        self.lo, self.hi = float(data.lo), float(data.hi)
        self.device = device
        vec = data.vectors if with_vectors else None
        keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.part_offsets, np.uint64),
                np.ascontiguousarray(data.codes, np.uint8), np.ascontiguousarray(data.row_ids, np.uint64),
                None if vec is None else np.ascontiguousarray(vec, np.float32)]
        desc = SqDesc(ABI_VERSION, data.dim, data.nlist, METRICS[data.metric], device, 0, data.nrows, self.lo, self.hi,
                      _ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), _ptr(keep[3]), _ptr(keep[4]))
        h = C.c_void_p()
        check(lib.lgpu_ivf_sq_open(C.byref(desc), C.byref(h)))
        self._h = h
        self.has_vectors = vec is not None


class GpuIvfRq(GpuIvfPq):
    """An IVF_RQ index pinned in HBM: an lgpu_index opened by lgpu_ivf_rq_open, so every search entry point of GpuIvfPq
    serves it.  _distance is the RaBitQ estimate of the squared L2 distance (half of it for cosine); refine_factor
    re-ranks by the exact distance."""

    def __init__(self, data, device: int = 0, with_vectors: bool = True):
        lib = load()
        if data.metric not in ("l2", "cosine"):
            raise ValueError(f"IVF_RQ supports the l2 and cosine distance types, not {data.metric!r}")
        data.validate()
        self.dim, self.nlist, self.metric = data.dim, data.nlist, data.metric
        self.device = device
        vec = data.vectors if with_vectors else None
        keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.rotation, np.float32),
                np.ascontiguousarray(data.part_offsets, np.uint64), np.ascontiguousarray(data.codes, np.uint8),
                np.ascontiguousarray(data.add_factors, np.float32), np.ascontiguousarray(data.scale_factors, np.float32),
                np.ascontiguousarray(data.row_ids, np.uint64),
                None if vec is None else np.ascontiguousarray(vec, np.float32)]
        desc = RqDesc(ABI_VERSION, data.dim, data.nlist, METRICS[data.metric], device, data.num_bits, data.nrows,
                      *[_ptr(a) for a in keep])
        h = C.c_void_p()
        check(lib.lgpu_ivf_rq_open(C.byref(desc), C.byref(h)))
        self._h = h
        self.has_vectors = vec is not None


class GpuFlat(_Handle):
    """A raw vector column pinned in HBM (lgpu_flat)."""
    _close = "lgpu_flat_close"

    def __init__(self, vectors, row_ids=None, device: int = 0):
        v = np.ascontiguousarray(vectors, np.float32)
        self.nrows, self.dim = v.shape
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, np.uint64)
        h = C.c_void_p()
        check(load().lgpu_flat_open(_ptr(v), self.nrows, self.dim, _ptr(rid), device, C.byref(h)))
        self._h = h
        self.device = device

    def search(self, queries, k=10, metric="l2", lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        p = make_params(k, 0, 0, lower, upper, 0, timeout_ms)
        return _host_search("lgpu_flat_search", (self._h, METRICS[metric], _ptr(q), q.shape[0]), q.shape[0], k, p,
                            allow, allow_bits)

    def search_into(self, metric: str, q: np.ndarray, p: SearchParams, ids: np.ndarray, dist: np.ndarray,
                    cnt: np.ndarray):
        """Host-buffer flat search into caller-owned (e.g. pinned) arrays; no allocation."""
        check(load().lgpu_flat_search(self._h, METRICS[metric], q.ctypes.data, q.shape[0], C.byref(p),
                                      ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data))

    def search_device(self, metric: str, d_q: int, B: int, p: SearchParams, d_ids: int, d_dist: int, d_cnt: int,
                      stream: int = 0):
        """Device-pointer flat search (raw addresses), enqueued on `stream`, not synchronised."""
        check(load().lgpu_flat_search_device(self._h, METRICS[metric], d_q, B, C.byref(p), d_ids, d_dist, d_cnt,
                                             stream))


class GpuBinary(_Handle):
    """A packed binary vector column (fixed_size_list<uint8, nbytes>) pinned in HBM (lgpu_binary), searched by
    Hamming distance."""
    _close = "lgpu_binary_close"

    def __init__(self, vectors, row_ids=None, device: int = 0):
        v = np.ascontiguousarray(vectors, np.uint8)
        if v.ndim != 2:
            raise ValueError("binary vectors must be a [rows, bytes] uint8 array")
        self.nrows, self.nbytes = v.shape
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, np.uint64)
        h = C.c_void_p()
        check(load().lgpu_binary_open(_ptr(v), self.nrows, self.nbytes, _ptr(rid), device, C.byref(h)))
        self._h = h
        self.device = device

    def search(self, queries, k=10, lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        """Host-buffer search of queries [B, nbytes] (or one [nbytes] query) whose components are integers in
        [0, 255]: returns (ids [B,k] u64, dist [B,k] f32, count [B] u32)."""
        q = self._queries(queries)
        p = make_params(k, 0, 0, lower, upper, 0, timeout_ms)
        return _host_search("lgpu_binary_search", (self._h, _ptr(q), q.shape[0]), q.shape[0], k, p, allow, allow_bits)

    def _queries(self, queries) -> np.ndarray:
        a = np.asarray(queries)
        if a.ndim not in (1, 2) or a.shape[-1] != self.nbytes:
            raise ValueError(f"binary queries must be [B, {self.nbytes}] or [{self.nbytes}], got shape {a.shape}")
        return binary_components(a).reshape(-1, self.nbytes)

    def search_device(self, d_q: int, B: int, p: SearchParams, d_ids: int, d_dist: int, d_cnt: int, stream: int = 0):
        """Device-pointer search (raw addresses; queries [B][nbytes] u8), enqueued on `stream`, not synchronised."""
        check(load().lgpu_binary_search_device(self._h, d_q, B, C.byref(p), d_ids, d_dist, d_cnt, stream))


class GpuIvfBinary(_Handle):
    """A binary IVF_FLAT index (IvfBinaryIndexData) pinned in HBM (lgpu_ivf_binary): the probed partitions of packed
    binary rows scored exactly by Hamming distance."""
    _close = "lgpu_ivf_binary_close"

    def __init__(self, data, device: int = 0):
        lib = load()
        data.validate()
        self.nbytes, self.nlist, self.metric = data.nbytes, data.nlist, data.metric
        self.device = device
        self._keep = [np.ascontiguousarray(data.centroids, np.uint8), np.ascontiguousarray(data.part_offsets, np.uint64),
                      np.ascontiguousarray(data.vectors, np.uint8), np.ascontiguousarray(data.row_ids, np.uint64)]
        desc = IvfBinaryDesc(ABI_VERSION, data.nbytes, data.nlist, device, data.nrows, *[_ptr(a) for a in self._keep])
        h = C.c_void_p()
        check(lib.lgpu_ivf_binary_open(C.byref(desc), C.byref(h)))
        self._h = h
        self._keep = None

    def _queries(self, queries) -> np.ndarray:
        a = np.asarray(queries)
        if a.ndim not in (1, 2) or a.shape[-1] != self.nbytes:
            raise ValueError(f"binary queries must be [B, {self.nbytes}] or [{self.nbytes}], got shape {a.shape}")
        return binary_components(a).reshape(-1, self.nbytes)

    def search(self, queries, k=10, nprobes=20, refine_factor=0, lower=None, upper=None, allow=None, allow_bits=0,
               max_nprobes=0, timeout_ms=0):
        """Host-buffer search of queries [B, nbytes] (or one [nbytes] query): returns (ids [B,k] u64, dist [B,k] f32,
        count [B] u32).  refine_factor is accepted and changes nothing: the distances are exact."""
        q = self._queries(queries)
        p = make_params(k, nprobes, refine_factor, lower, upper, max_nprobes, timeout_ms)
        return _host_search("lgpu_ivf_binary_search", (self._h, _ptr(q), q.shape[0]), q.shape[0], k, p, allow,
                            allow_bits)

    def search_device(self, d_q: int, B: int, p: SearchParams, d_ids: int, d_dist: int, d_cnt: int, stream: int = 0):
        """Device-pointer search (raw addresses; queries [B][nbytes] u8), enqueued on `stream`, not synchronised."""
        check(load().lgpu_ivf_binary_search_device(self._h, d_q, B, C.byref(p), d_ids, d_dist, d_cnt, stream))


def multivec_offsets(lengths) -> np.ndarray:
    """Vector counts per row (or per query) -> the [n+1] offsets the multivector entry points take."""
    n = np.asarray(lengths, np.int64).reshape(-1)
    if n.size and n.min() < 0:
        raise ValueError("vector counts must not be negative")
    return np.concatenate([[0], np.cumsum(n)]).astype(np.uint64)


class GpuMultivec(_Handle):
    """A multivector column (list<fixed_size_list<float, dim>>) pinned in HBM (lgpu_multivec), searched by late
    interaction: _distance = sum over the query's vectors of the smallest cosine distance to the row's vectors."""
    _close = "lgpu_multivec_close"

    def __init__(self, values, offsets, row_ids=None, device: int = 0):
        v = np.ascontiguousarray(values, np.float32)
        off = np.ascontiguousarray(offsets, np.uint64)
        if v.ndim != 2:
            raise ValueError("multivector values must be a [vectors, dim] array")
        if off.ndim != 1 or off.size < 1 or off[0] != 0 or int(off[-1]) != v.shape[0]:
            raise ValueError("row offsets must be [rows + 1], start at 0 and end at the number of vectors")
        if np.any(off[1:] < off[:-1]):
            raise ValueError("row offsets must not decrease")
        if off.size > 1 and int(np.max(off[1:] - off[:-1])) > MULTIVEC_MAX_ROW:
            raise ValueError(f"a multivector row holds at most {MULTIVEC_MAX_ROW} vectors")
        if not 1 <= v.shape[1] <= MULTIVEC_MAX_DIM:
            raise ValueError(f"multivector dimension must be in [1, {MULTIVEC_MAX_DIM}]")
        self.nrows, self.dim = off.size - 1, v.shape[1]
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, np.uint64)
        if rid is not None and rid.shape != (self.nrows,):
            raise ValueError("row_ids must hold one id per row")
        h = C.c_void_p()
        check(load().lgpu_multivec_open(_ptr(v), _ptr(off), self.nrows, self.dim, _ptr(rid), device, C.byref(h)))
        self._h = h
        self.device = device

    def _queries(self, queries, q_offsets):
        """(values [Tq, dim] f32, offsets [B+1] u32).  queries: a list with one [nq_b, dim] (or [dim]) array per
        query, or [Tq, dim] values with q_offsets; a single numpy array is ONE query."""
        if q_offsets is None:
            qs = [queries] if isinstance(queries, np.ndarray) else list(queries)
            arrs = []
            for q in qs:
                a = np.asarray(q, np.float32)
                if a.ndim == 1:
                    a = a[None, :]
                if a.ndim != 2:
                    raise ValueError("a multivector query must be [nq, dim] or [dim]")
                arrs.append(a)
            lens = [a.shape[0] for a in arrs]
            vals = np.concatenate(arrs) if arrs else np.zeros((0, self.dim), np.float32)
            off = multivec_offsets(lens)
        else:
            vals = np.asarray(queries, np.float32)
            off = np.asarray(q_offsets, np.int64).reshape(-1)
        if vals.ndim != 2 or vals.shape[1] != self.dim:
            raise ValueError(f"multivector query vectors must have dimension {self.dim}, got shape {vals.shape}")
        off = _query_offsets(off)
        if int(off[-1]) != vals.shape[0]:
            raise ValueError("query offsets must end at the number of query vectors")
        return np.ascontiguousarray(vals), off

    def search(self, queries, k=10, q_offsets=None, lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        """Host-buffer search of B multivector queries: returns (ids [B,k] u64, dist [B,k] f32, count [B] u32).
        `queries`: a list with one [nq_b, dim] array per query, or [Tq, dim] values with `q_offsets` [B+1]; a single
        numpy array is ONE query.  Shapes are checked before any device call."""
        q, off = self._queries(queries, q_offsets)
        p = make_params(k, 0, 0, lower, upper, 0, timeout_ms)
        return _host_search("lgpu_multivec_search", (self._h, _ptr(q), _ptr(off), off.size - 1), off.size - 1, k, p,
                            allow, allow_bits)

    def search_device(self, d_q: int, q_offsets, p: SearchParams, d_ids: int, d_dist: int, d_cnt: int, stream: int = 0):
        """Device-pointer search: d_q [Tq][dim] f32 and the outputs are raw device addresses, q_offsets [B+1] a host
        array (checked here); enqueued on `stream`, not synchronised."""
        off = _query_offsets(q_offsets)
        check(load().lgpu_multivec_search_device(self._h, d_q, _ptr(off), off.size - 1, C.byref(p), d_ids, d_dist,
                                                 d_cnt, stream))


def ivf_assign(centroids, vectors, metric: str = "l2", device: int = 0) -> np.ndarray:
    """Partition of every row = find_partitions(row, nprobes=1) with the search path's exact kernels."""
    c = np.ascontiguousarray(centroids, np.float32); v = np.ascontiguousarray(vectors, np.float32)
    out = np.empty(v.shape[0], np.uint32)
    check(load().lgpu_ivf_assign(_ptr(c), c.shape[0], c.shape[1], METRICS[metric], _ptr(v), v.shape[0], device, _ptr(out)))
    return out


def pq_encode(centroids, codebook, vectors, parts, metric: str = "l2", device: int = 0) -> np.ndarray:
    """8-bit PQ codes [n, m] of raw rows given their partitions (residual PQ for l2/cosine)."""
    c = np.ascontiguousarray(centroids, np.float32); cb = np.ascontiguousarray(codebook, np.float32)
    v = np.ascontiguousarray(vectors, np.float32); p = np.ascontiguousarray(parts, np.uint32)
    m = cb.shape[0]
    out = np.empty((v.shape[0], m), np.uint8)
    check(load().lgpu_pq_encode(_ptr(c), _ptr(cb), c.shape[0], c.shape[1], m, METRICS[metric], _ptr(v), _ptr(p),
                                v.shape[0], device, _ptr(out)))
    return out


def kmeans_train(vectors, init_centroids, iters: int, device: int = 0, want_inertia: bool = False):
    """Lloyd k-means on the GPU (lgpu_kmeans_train): returns the trained centres (and the inertia)."""
    v = np.ascontiguousarray(vectors, np.float32)
    c = np.array(init_centroids, np.float32, order="C", copy=True)
    inertia = C.c_double(0.0)
    check(load().lgpu_kmeans_train(_ptr(v), v.shape[0], v.shape[1], _ptr(c), c.shape[0], int(iters), device,
                                   C.byref(inertia) if want_inertia else None))
    return (c, inertia.value) if want_inertia else c


def pq_train(vectors, init_codebook, iters: int, device: int = 0) -> np.ndarray:
    """The m x 256 PQ codewords (lgpu_pq_train); vectors = what gets quantised (residuals for l2 / cosine)."""
    v = np.ascontiguousarray(vectors, np.float32)
    cb = np.array(init_codebook, np.float32, order="C", copy=True)
    check(load().lgpu_pq_train(_ptr(v), v.shape[0], v.shape[1], cb.shape[0], _ptr(cb), int(iters), device))
    return cb


def allow_bitmap(row_ids, nbits: int) -> np.ndarray:
    """Row-id allow-list -> the u32 bitmap lgpu_search_filtered takes (bit r & 31 of word r >> 5)."""
    bm = np.zeros((int(nbits) + 31) // 32, np.uint32)
    r = np.asarray(row_ids, np.uint64)
    r = r[r < nbits]
    np.bitwise_or.at(bm, (r >> np.uint64(5)).astype(np.int64), np.uint32(1) << (r & np.uint64(31)).astype(np.uint32))
    return bm


def mask_bitmap(mask) -> np.ndarray:
    """Boolean mask over row ids 0..n-1 -> u32 bitmap."""
    m = np.asarray(mask, bool)
    pad = (-m.size) % 32
    bits = np.packbits(np.concatenate([m, np.zeros(pad, bool)]), bitorder="little")
    return np.ascontiguousarray(bits).view(np.uint32)


COMM_ID_BYTES = 128
# one gathered top-k entry (csrc/kernels.cuh TopkRecord): what crosses NVLink in the sharded search
TOPK_RECORD = np.dtype([("id", "<u8"), ("dist", "<f4"), ("pad", "<u4")])


def comm_unique_id() -> bytes:
    """rank 0: the group's id (an ncclUniqueId) to hand to every rank."""
    buf = (C.c_ubyte * COMM_ID_BYTES)()
    check(load().lgpu_comm_unique_id(buf, COMM_ID_BYTES))
    return bytes(buf)


class Comm(_Handle):
    """One rank of a partition-sharded search group (lgpu_comm): collective constructor."""
    _close = "lgpu_comm_destroy"

    def __init__(self, unique_id: bytes, rank: int, world: int, device: int = 0):
        if len(unique_id) != COMM_ID_BYTES:
            raise ValueError("unique id must be 128 bytes")
        buf = (C.c_ubyte * COMM_ID_BYTES).from_buffer_copy(unique_id)
        h = C.c_void_p()
        check(load().lgpu_comm_init(buf, COMM_ID_BYTES, rank, world, device, C.byref(h)))
        self._h, self.rank, self.world, self.device = h, rank, world, device

    def search(self, shard: "GpuIvfPq", queries, k=10, nprobes=20, lower=None, upper=None):
        """Collective host-buffer search: same queries on every rank, global top-k on every rank."""
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, shard.dim)
        B = q.shape[0]
        ids = np.empty((B, k), np.uint64); dist = np.empty((B, k), np.float32); cnt = np.empty(B, np.uint32)
        p = make_params(k, nprobes, 0, lower, upper)
        check(load().lgpu_search_sharded(shard._h, self._h, _ptr(q), B, C.byref(p), _ptr(ids), _ptr(dist), _ptr(cnt)))
        return ids, dist, cnt

    def search_device(self, shard: "GpuIvfPq", d_q: int, B: int, p: SearchParams, d_ids: int, d_dist: int,
                      d_cnt: int, stream: int = 0):
        check(load().lgpu_search_sharded_device(shard._h, self._h, d_q, B, C.byref(p), d_ids, d_dist, d_cnt, stream))

    def last_stage_ms(self):
        t = (C.c_float * 3)()
        check(load().lgpu_comm_last_stage_ms(self._h, t))
        return dict(zip(["local_search", "allgather", "merge"], list(t)))


def ticket_wait(ticket) -> None:
    check(load().lgpu_ticket_wait(ticket))


def ticket_done(ticket) -> bool:
    d = C.c_int(0)
    check(load().lgpu_ticket_poll(ticket, C.byref(d)))
    return bool(d.value)


def merge_topk_device(device: int, nlists: int, B: int, k: int, d_ids: int, d_dist: int, d_out_ids: int,
                      d_out_dist: int, d_out_cnt: int, stream: int = 0):
    check(load().lgpu_merge_topk_device(device, nlists, B, k, d_ids, d_dist, d_out_ids, d_out_dist, d_out_cnt,
                                        stream))


def debug_gemm(queries, vectors, device: int = 0) -> np.ndarray:
    q = np.ascontiguousarray(queries, np.float32); x = np.ascontiguousarray(vectors, np.float32)
    out = np.empty((q.shape[0], x.shape[0]), np.float32)
    check(load().lgpu_debug_gemm(_ptr(q), _ptr(x), q.shape[0], x.shape[0], q.shape[1], device, _ptr(out)))
    return out


def debug_hamming_gemm(queries, vectors, device: int = 0) -> np.ndarray:
    """The binary tensor-core kernel alone: [B, N] u32 Hamming distances."""
    q = np.ascontiguousarray(queries, np.uint8); x = np.ascontiguousarray(vectors, np.uint8)
    if q.ndim != 2 or x.ndim != 2 or q.shape[1] != x.shape[1]:
        raise ValueError("queries and vectors must be [rows, bytes] arrays with the same bytes per row")
    out = np.empty((q.shape[0], x.shape[0]), np.uint32)
    check(load().lgpu_debug_hamming_gemm(_ptr(q), _ptr(x), q.shape[0], x.shape[0], q.shape[1], device, _ptr(out)))
    return out


def debug_ivf_hamming_scan(queries, vectors, device: int = 0) -> np.ndarray:
    """The binary IVF_FLAT scan kernel alone (lgpu_debug_ivf_hamming_scan), every query one probe slot over one partition
    holding the N rows: [B, N] u32 Hamming distances."""
    q = np.ascontiguousarray(queries, np.uint8); x = np.ascontiguousarray(vectors, np.uint8)
    if q.ndim != 2 or x.ndim != 2 or q.shape[1] != x.shape[1]:
        raise ValueError("queries and vectors must be [rows, bytes] arrays with the same bytes per row")
    out = np.empty((q.shape[0], x.shape[0]), np.uint32)
    check(load().lgpu_debug_ivf_hamming_scan(_ptr(q), q.shape[0], _ptr(x), x.shape[0], q.shape[1], device, _ptr(out)))
    return out


def debug_pq4_sums(tables, codes, device: int = 0) -> np.ndarray:
    """The 4-bit IVF_PQ scan kernel alone (lgpu_debug_pq4_sums): tables [B, m, 16] u8, codes [N, m/2] packed bytes ->
    [B, N] u32 sums of tables[b][i][code_i]."""
    t = np.ascontiguousarray(tables, np.uint8)
    x = np.ascontiguousarray(codes, np.uint8)
    B, m = t.shape[0], t.shape[1]
    if t.shape[2:] != (16,) or x.ndim != 2 or 2 * x.shape[1] != m:
        raise ValueError("tables must be [B, m, 16] and codes [N, m / 2]")
    out = np.empty((B, x.shape[0]), np.uint32)
    check(load().lgpu_debug_pq4_sums(_ptr(t), B, _ptr(x), x.shape[0], m, device, _ptr(out)))
    return out


def debug_sq_distances(q_codes, x_codes, device: int = 0) -> np.ndarray:
    """The IVF_SQ scan kernel alone: [B, N] u32 exact sums of squared code differences."""
    q = np.ascontiguousarray(q_codes, np.uint8); x = np.ascontiguousarray(x_codes, np.uint8)
    if q.ndim != 2 or x.ndim != 2 or q.shape[1] != x.shape[1]:
        raise ValueError("q_codes and x_codes must be [rows, dim] uint8 arrays with the same dim")
    out = np.empty((q.shape[0], x.shape[0]), np.uint32)
    check(load().lgpu_debug_sq_distances(_ptr(q), q.shape[0], _ptr(x), x.shape[0], q.shape[1], device, _ptr(out)))
    return out


def debug_rq_distances(q_res, codes, add_factors, scale_factors, metric: str = "l2", device: int = 0):
    """The IVF_RQ planes and scan kernels alone, each query one probe slot of rotated residual q_res[b] over the N rows:
    (est [B, N] f32, ip [B, N] u32) -- the reported estimates and the exact sum_i b_i u_i."""
    q = np.ascontiguousarray(q_res, np.float32); x = np.ascontiguousarray(codes, np.uint8)
    if q.ndim != 2 or x.ndim != 2 or x.shape[1] != (q.shape[1] + 7) // 8:
        raise ValueError("q_res must be [B, dim] and codes [N, ceil(dim / 8)]")
    add = np.ascontiguousarray(add_factors, np.float32); sc = np.ascontiguousarray(scale_factors, np.float32)
    if add.shape != (x.shape[0],) or sc.shape != (x.shape[0],):
        raise ValueError("add_factors and scale_factors must be [N]")
    est = np.empty((q.shape[0], x.shape[0]), np.float32); ip = np.empty((q.shape[0], x.shape[0]), np.uint32)
    check(load().lgpu_debug_rq_distances(_ptr(q), q.shape[0], _ptr(x), _ptr(add), _ptr(sc), x.shape[0], q.shape[1],
                                         METRICS[metric], device, _ptr(est), _ptr(ip)))
    return est, ip


def debug_maxsim_gemm(queries, values, offsets, device: int = 0) -> np.ndarray:
    """The multivector tensor-core score alone: [nqv, nrows] f32, the largest fp16 normalised similarity of each query
    vector over each row's vectors (NaN for an empty row)."""
    q = np.ascontiguousarray(queries, np.float32); x = np.ascontiguousarray(values, np.float32)
    off = np.ascontiguousarray(offsets, np.uint64)
    if q.ndim != 2 or x.ndim != 2 or q.shape[1] != x.shape[1] or int(off[-1]) != x.shape[0]:
        raise ValueError("queries [nqv, dim], values [T, dim] and offsets [nrows + 1] ending at T are required")
    out = np.empty((q.shape[0], off.size - 1), np.float32)
    check(load().lgpu_debug_maxsim_gemm(_ptr(q), q.shape[0], _ptr(x), _ptr(off), off.size - 1, q.shape[1], device,
                                        _ptr(out)))
    return out


def kernel_launch_count() -> int:
    n = C.c_uint64(0)
    check(load().lgpu_kernel_launch_count(C.byref(n)))
    return n.value


def last_filter_stats():
    t = (C.c_uint64 * 4)()
    check(load().lgpu_last_filter_stats(t))
    return dict(zip(["candidates", "rescored", "flagged_queries", "queries"], [int(x) for x in t]))


def set_profiling(enabled: bool) -> None:
    check(load().lgpu_set_profiling(1 if enabled else 0))


def last_stage_ms():
    t = (C.c_float * 7)()
    check(load().lgpu_last_stage_ms(t))
    return dict(zip(["coarse", "select_probes", "group", "scan", "topk", "refine", "total"], list(t)))


def last_scanned_code_bytes() -> int:
    b = C.c_uint64(0)
    check(load().lgpu_last_scanned_code_bytes(C.byref(b)))
    return b.value

"""ctypes loader for the CPU oracle (oracle/oracle.c and the index kinds' oracles, tests/*_oracle.c).

TEST INFRASTRUCTURE ONLY.  May be imported by tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / ``--impl reference`` legs -- never by
``lancedb_b200`` (the product path).  PARITY STATUS: IVF_PQ parity unpinned
(see oracle/oracle.h); flat path pinned by the reference's doctests.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None

METRICS = {"l2": 0, "cosine": 1, "dot": 2}


class _Index(C.Structure):
    _fields_ = [
        ("dim", C.c_uint32), ("nlist", C.c_uint32), ("m", C.c_uint32), ("metric", C.c_int),
        ("nrows", C.c_uint64),
        ("centroids", C.c_void_p), ("codebook", C.c_void_p), ("part_offsets", C.c_void_p),
        ("codes_t", C.c_void_p), ("row_ids", C.c_void_p), ("vectors", C.c_void_p),
    ]


class _Params(C.Structure):
    _fields_ = [
        ("k", C.c_uint32), ("nprobes", C.c_uint32), ("refine_factor", C.c_uint32),
        ("has_lower", C.c_int), ("has_upper", C.c_int), ("lower", C.c_float), ("upper", C.c_float),
        ("allow", C.c_void_p), ("allow_bits", C.c_uint64), ("max_nprobes", C.c_uint32),
    ]


def allow_bitmap(row_ids, nbits: int) -> np.ndarray:
    """Row-id allow-list -> u32 bitmap of `nbits` bits (the form orc_params.allow / the C ABI take)."""
    bm = np.zeros((int(nbits) + 31) // 32, np.uint32)
    r = np.asarray(row_ids, np.uint64)
    r = r[r < nbits]
    np.bitwise_or.at(bm, (r >> np.uint64(5)).astype(np.int64), (np.uint32(1) << (r & np.uint64(31)).astype(np.uint32)))
    return bm


def _params(k, nprobes, refine_factor, lower, upper, allow=None, allow_bits=0, max_nprobes=0):
    p = _Params(k, nprobes, refine_factor, lower is not None, upper is not None,
                0.0 if lower is None else lower, 0.0 if upper is None else upper, None, 0, int(max_nprobes or 0))
    if allow is not None:
        p.allow = allow.ctypes.data
        p.allow_bits = int(allow_bits)
    return p


def build(force: bool = False) -> str:
    """Compile oracle.c and the index kinds' oracles under tests/ into one library with gcc (flags and sources in
    oracle/Makefile; make rebuilds it when a source is newer)."""
    subprocess.run(["make", "-C", _HERE, "-s"] + (["-B"] if force else []), check=True)
    return _LIB_PATH


_IX, _P = C.POINTER(_Index), C.POINTER(_Params)
_vp, _u8, _u32, _u64, _int, _f, _d, _sz = (C.c_void_p, C.c_uint8, C.c_uint32, C.c_uint64, C.c_int, C.c_float,
                                           C.c_double, C.c_size_t)
# name: (restype, argtypes); every search ends in (queries, B, &params, ids, dist, count, nthreads)
_SIGNATURES = {
    "orc_l2_f32": (_f, [_vp, _vp, _sz]),
    "orc_dot_f32": (_f, [_vp, _vp, _sz]),
    "orc_cosine_f32": (_f, [_vp, _vp, _sz]),
    "orc_distance_f32": (_f, [_int, _vp, _vp, _sz]),
    "orc_l2_subvec": (_f, [_vp, _vp, _sz]),
    "orc_normalize_f32": (None, [_vp, _sz, _vp]),
    "orc_find_partitions": (None, [_IX, _vp, _u32, _vp, _vp, _vp]),
    "orc_build_lut": (None, [_IX, _vp, _vp]),
    "orc_pq_scan": (None, [_vp, _vp, _sz, _u32, _vp]),
    "orc_partition_distances": (None, [_IX, _vp, _u32, _vp]),
    "orc_ivf_assign": (None, [_IX, _vp, _u64, _vp]),
    "orc_pq_encode": (None, [_IX, _vp, _vp, _u64, _vp]),
    "orc_ivfpq_search": (_int, [_IX, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_flat_search": (_int, [_vp, _u64, _u32, _vp, _int, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_sq_encode": (None, [_vp, _u64, _d, _d, _vp]),
    "orc_sq_distance": (_f, [_vp, _vp, _u32]),
    "orc_sq_search": (_int, [_IX, _vp, _d, _d, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_rq_rotate": (None, [_vp, _vp, _u64, _u32, _vp]),
    "orc_rq_slot": (None, [_vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "orc_rq_estimate": (_f, [_vp, _f, _f, _vp, _vp, _u32, _u32, _int]),
    "orc_rq_search": (_int, [_IX, _vp, _vp, _vp, _vp, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_pq4_quant": (_u8, [_f, _f, _f]),
    "orc_pq4_distance": (_f, [_u32, _f, _f, _u32, _int]),
    "orc_pq4_tables": (None, [_IX, _vp, _u32, _vp, _vp]),
    "orc_pq4_partition_distances": (None, [_IX, _vp, _u32, _vp]),
    "orc_pq4_search": (_int, [_IX, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_ivf_binary_search": (_int, [_vp, _u32, _vp, _vp, _vp, _u32, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_hamming_u8": (_int, [_vp, _u32, _vp, _u64, _u32, _vp, _int]),
    "orc_flat_search_u8": (_int, [_vp, _u64, _u32, _vp, _vp, _u32, _P, _vp, _vp, _vp, _int]),
    "orc_multivec_distances": (_int, [_vp, _vp, _u64, _u32, _vp, _vp, _u32, _vp, _int]),
    "orc_multivec_search": (_int, [_vp, _vp, _u64, _u32, _vp, _vp, _vp, _u32, _P, _vp, _vp, _vp, _int]),
}


def load():
    global _lib
    if _lib is not None:
        return _lib
    build()
    lib = C.CDLL(_LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


def threads(nthreads) -> int:
    """nthreads, or every host core for 0"""
    return int(nthreads) if nthreads else (os.cpu_count() or 1)


def search_call(name, args, B, k, nthreads=0, nprobes=0, refine_factor=0, lower=None, upper=None, allow=None,
                allow_bits=0, max_nprobes=0):
    """Runs the C search `name`(*args, B, &orc_params, ids, dist, count, nthreads) and returns (ids [B, k] u64,
    dist [B, k] f32, count [B] u32).  allow: a u32 bitmap of allow_bits bits, or a bool mask over row ids."""
    if allow is not None:
        allow = np.asarray(allow)
        if allow.dtype == bool:
            allow, allow_bits = allow_bitmap(np.nonzero(allow)[0], allow.size), allow.size
        allow = np.ascontiguousarray(allow, np.uint32)
    p = _params(k, nprobes, refine_factor, lower, upper, allow, allow_bits, max_nprobes)
    ids = np.empty((B, k), np.uint64)
    dist = np.empty((B, k), np.float32)
    cnt = np.empty(B, np.uint32)
    if B and getattr(load(), name)(*args, B, C.byref(p), _ptr(ids), _ptr(dist), _ptr(cnt), threads(nthreads)):
        raise RuntimeError(f"{name} failed")
    return ids, dist, cnt


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def l2(x, y) -> float:
    x, y = _f32(x), _f32(y)
    return float(load().orc_l2_f32(_ptr(x), _ptr(y), x.size))


def dot(x, y) -> float:
    x, y = _f32(x), _f32(y)
    return float(load().orc_dot_f32(_ptr(x), _ptr(y), x.size))


def cosine(x, y) -> float:
    x, y = _f32(x), _f32(y)
    return float(load().orc_cosine_f32(_ptr(x), _ptr(y), x.size))


def l2_subvec(x, y) -> float:
    x, y = _f32(x), _f32(y)
    return float(load().orc_l2_subvec(_ptr(x), _ptr(y), x.size))


def normalize(x) -> np.ndarray:
    x = _f32(x)
    out = np.empty_like(x)
    load().orc_normalize_f32(_ptr(x), x.size, _ptr(out))
    return out


class OracleIndex:
    """Wraps the plain index arrays (lancedb_b200.index.IvfPqIndexData fields)."""

    def __init__(self, *, dim, nlist, m, metric, centroids, codebook, part_offsets, codes_t,
                 row_ids, vectors=None):
        self.centroids = _f32(centroids)
        self.codebook = _f32(codebook)
        self.part_offsets = np.ascontiguousarray(part_offsets, dtype=np.uint64)
        self.codes_t = np.ascontiguousarray(codes_t, dtype=np.uint8)
        self.row_ids = np.ascontiguousarray(row_ids, dtype=np.uint64)
        self.vectors = _f32(vectors) if vectors is not None else None
        self.metric = metric if isinstance(metric, int) else METRICS[metric]
        self.dim, self.nlist, self.m = int(dim), int(nlist), int(m)
        self.c = _Index(self.dim, self.nlist, self.m, self.metric, int(self.row_ids.size),
                        _ptr(self.centroids), _ptr(self.codebook), _ptr(self.part_offsets),
                        _ptr(self.codes_t), _ptr(self.row_ids), _ptr(self.vectors))

    @classmethod
    def from_data(cls, d):
        return cls(dim=d.dim, nlist=d.nlist, m=d.m, metric=d.metric, centroids=d.centroids,
                   codebook=d.codebook, part_offsets=d.part_offsets, codes_t=d.codes_t,
                   row_ids=d.row_ids, vectors=d.vectors)

    def find_partitions(self, q, nprobes):
        q = _f32(q)
        nprobes = min(nprobes, self.nlist)
        parts = np.empty(nprobes, np.uint32)
        dists = np.empty(nprobes, np.float32)
        alld = np.empty(self.nlist, np.float32)
        load().orc_find_partitions(C.byref(self.c), _ptr(q), nprobes, _ptr(parts), _ptr(dists), _ptr(alld))
        return parts, dists, alld

    def build_lut(self, resid_or_query):
        r = _f32(resid_or_query)
        lut = np.empty((self.m, 256), np.float32)
        load().orc_build_lut(C.byref(self.c), _ptr(r), _ptr(lut))
        return lut

    def partition_distances(self, q, part):
        q = _f32(q)
        n = int(self.part_offsets[part + 1] - self.part_offsets[part])
        out = np.empty(n, np.float32)
        load().orc_partition_distances(C.byref(self.c), _ptr(q), int(part), _ptr(out))
        return out

    def ivf_assign(self, vectors):
        v = _f32(vectors).reshape(-1, self.dim)
        out = np.empty(v.shape[0], np.uint32)
        load().orc_ivf_assign(C.byref(self.c), _ptr(v), v.shape[0], _ptr(out))
        return out

    def pq_encode(self, vectors, parts):
        v = _f32(vectors).reshape(-1, self.dim)
        p = np.ascontiguousarray(parts, np.uint32)
        out = np.empty((v.shape[0], self.m), np.uint8)
        load().orc_pq_encode(C.byref(self.c), _ptr(v), _ptr(p), v.shape[0], _ptr(out))
        return out

    def search(self, queries, k=10, nprobes=20, refine_factor=0, lower=None, upper=None, nthreads=1,
               allow=None, allow_bits=0, max_nprobes=0):
        q = _f32(queries).reshape(-1, self.dim)
        return search_call("orc_ivfpq_search", (C.byref(self.c), _ptr(q)), q.shape[0], k, nthreads, nprobes,
                           refine_factor, lower, upper, allow, allow_bits, max_nprobes)


def flat_search(vectors, queries, k=10, metric="l2", row_ids=None, lower=None, upper=None, nthreads=1,
                allow=None, allow_bits=0):
    v = _f32(vectors)
    n, dim = v.shape
    q = _f32(queries).reshape(-1, dim)
    rid = np.ascontiguousarray(row_ids, dtype=np.uint64) if row_ids is not None else None
    return search_call("orc_flat_search", (_ptr(v), n, dim, _ptr(rid), METRICS[metric], _ptr(q)), q.shape[0], k,
                       nthreads, lower=lower, upper=upper, allow=allow, allow_bits=allow_bits)


def pq_scan(lut, codes_t, n, m):
    lut = _f32(lut)
    codes_t = np.ascontiguousarray(codes_t, np.uint8)
    out = np.empty(n, np.float32)
    load().orc_pq_scan(_ptr(lut), _ptr(codes_t), n, m, _ptr(out))
    return out

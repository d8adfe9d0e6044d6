"""CPU oracle of binary IVF_FLAT search by Hamming distance: the C ABI's lgpu_ivf_binary_open + lgpu_ivf_binary_search
semantics.

Per query: the nprobes partitions whose packed centroids are nearest by Hamming distance, ties to the lower partition id
(every partition when nprobes >= nlist); every row of those partitions scored exactly, _distance = popcount(q XOR x) as
f32; the allow mask and distance_range [lower, upper) drop rows before the top-k; maximum_nprobes widens under a
prefilter; refine_factor changes nothing.  Results ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (ivf_binary_oracle.c: orc_ivf_binary_search, taking the IVF_PQ oracle's
orc_params), which the GPU tests, smoke() and scripts/bench_ivf_binary.py compare against, and the NumPy mirror below
(search_np, and the k-modes trainer's mirror kmodes_np), which the CPU tests check the C oracle and the trainer against.
`data` is a lancedb_b200.index.IvfBinaryIndexData.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "ivf_binary_oracle.c")
_LIB_PATH = os.path.join(_HERE, "_build", "libivf_binary_oracle.so")
_lib = None
U64_MAX = np.iinfo(np.uint64).max


def build(force: bool = False) -> str:
    """gcc -> tests/_build/libivf_binary_oracle.so (rebuilt when the source or oracle/oracle.h is newer)."""
    deps = [_SRC, os.path.join(_ROOT, "oracle", "oracle.h")]
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        subprocess.run(["gcc", "-O3", "-mpopcnt", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-pthread", "-shared",
                        "-o", _LIB_PATH, _SRC, "-lm"], check=True)
    return _LIB_PATH


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        lib = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        lib.orc_ivf_binary_search.argtypes = [vp, C.c_uint32, vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, vp,
                                              C.c_int]
        _lib = lib
    return _lib


def _allow_bits(allow):
    """bool mask over row ids -> (u32 bitmap, bits)"""
    import oracle
    a = np.asarray(allow, bool)
    return oracle.allow_bitmap(np.nonzero(a)[0], a.size), a.size


def search(data, queries, k: int, nprobes: int, lower=None, upper=None, allow=None, max_nprobes: int = 0,
           nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    import oracle
    q = np.ascontiguousarray(queries, np.uint8).reshape(-1, data.nbytes)
    B = q.shape[0]
    bm, nbits = (None, 0) if allow is None else _allow_bits(allow)
    p = oracle._params(k, nprobes, 0, lower, upper, bm, nbits, max_nprobes)
    ids = np.empty((B, k), np.uint64)
    dist = np.empty((B, k), np.float32)
    cnt = np.empty(B, np.uint32)
    cent = np.ascontiguousarray(data.centroids, np.uint8)
    off = np.ascontiguousarray(data.part_offsets, np.uint64)
    x = np.ascontiguousarray(data.vectors, np.uint8)
    rid = np.ascontiguousarray(data.row_ids, np.uint64)
    if B and load().orc_ivf_binary_search(cent.ctypes.data, data.nlist, off.ctypes.data, x.ctypes.data,
                                          rid.ctypes.data, data.nbytes, q.ctypes.data, B, C.addressof(p),
                                          ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data,
                                          int(nthreads) if nthreads else (os.cpu_count() or 1)) != 0:
        raise RuntimeError("orc_ivf_binary_search failed")
    return ids, dist, cnt


# ---- NumPy mirror ----


def hamming_np(q, x) -> np.ndarray:
    """[B, N] int64 Hamming distances of packed rows (bitwise_count of the XOR)."""
    q = np.asarray(q, np.uint8)
    x = np.asarray(x, np.uint8)
    out = np.empty((q.shape[0], x.shape[0]), np.int64)
    step = max(1, (1 << 26) // max(1, x.shape[0] * x.shape[1]))
    for s in range(0, q.shape[0], step):
        out[s:s + step] = np.bitwise_count(q[s:s + step, None, :] ^ x[None, :, :]).sum(-1, dtype=np.int64)
    return out


def search_np(data, queries, k: int, nprobes: int, lower=None, upper=None, allow=None, max_nprobes: int = 0):
    """The same search, spelled with NumPy one query at a time."""
    q = np.asarray(queries, np.uint8).reshape(-1, data.nbytes)
    B, nlist = q.shape[0], data.nlist
    off = data.part_offsets.astype(np.int64)
    rid = data.row_ids.astype(np.uint64)
    keep = np.ones(data.nrows, bool)
    if allow is not None:
        a = np.asarray(allow, bool)
        inside = rid < a.size
        keep = np.zeros(data.nrows, bool)
        keep[inside] = a[rid[inside].astype(np.int64)]
    D = hamming_np(q, data.vectors) if data.nrows else np.zeros((B, 0), np.int64)
    C_ = hamming_np(q, data.centroids)
    np0 = min(nprobes, nlist)
    npm = min(max_nprobes, nlist) if allow is not None and max_nprobes > np0 else np0
    ids = np.full((B, k), U64_MAX, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    for b in range(B):
        order = np.lexsort((np.arange(nlist), C_[b]))
        for npu in (np0, npm):
            rows = np.concatenate([np.arange(off[p], off[p + 1]) for p in order[:npu]]).astype(np.int64)
            m = keep[rows].copy()
            d = D[b, rows].astype(np.float32)
            if lower is not None:
                m &= d >= np.float32(lower)
            if upper is not None:
                m &= d < np.float32(upper)
            rows, d = rows[m], d[m]
            if len(rows) >= k or npu == npm:
                break
        o = np.lexsort((rid[rows], d))[:k]
        n = len(o)
        ids[b, :n] = rid[rows[o]]
        dist[b, :n] = d[o]
        cnt[b] = n
    return ids, dist, cnt


def kmodes_np(x, centroids, iters: int):
    """The trainer's k-modes rounds, spelled with NumPy: (centroids after `iters` rounds or at convergence, final
    assignment of x).  Nearest centroid by Hamming distance, ties to the lowest index; bit set when 2 ones > members;
    an empty cluster keeps its centroid."""
    c = np.asarray(centroids, np.uint8).copy()
    x = np.asarray(x, np.uint8)
    bits = np.unpackbits(x, axis=1, bitorder="little").astype(np.int64)
    for _ in range(iters):
        a = np.argmin(hamming_np(x, c), axis=1)
        new = c.copy()
        for j in range(c.shape[0]):
            m = a == j
            if m.any():
                new[j] = np.packbits((2 * bits[m].sum(0) > m.sum()).astype(np.uint8), bitorder="little")
        if np.array_equal(new, c):
            break
        c = new
    return c, np.argmin(hamming_np(x, c), axis=1)


def index_from_assignment(x, centroids, assign, row_ids=None):
    """IvfBinaryIndexData of packed rows x [n, nbytes] in the given partitions (ascending row id inside each)."""
    from lancedb_b200.index import IvfBinaryIndexData
    x = np.asarray(x, np.uint8)
    nlist = centroids.shape[0]
    assign = np.asarray(assign, np.int64)
    order = np.argsort(assign, kind="stable")
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(assign, minlength=nlist))
    rid = np.arange(x.shape[0], dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    data = IvfBinaryIndexData(nbytes=x.shape[1], nlist=nlist, centroids=np.ascontiguousarray(centroids, np.uint8),
                              part_offsets=off, vectors=np.ascontiguousarray(x[order]), row_ids=rid[order])
    data.validate()
    return data


def random_index(rng, n: int, nbytes: int, nlist: int, empty=(), patterns: int = 0, row_ids=None):
    """An index over n random packed rows (or rows drawn from `patterns` random patterns: long runs of tied distances),
    centroids = nlist random packed vectors, every row in its nearest centroid; the rows of the partitions in `empty`
    are moved to the lowest partition not in it, so those stay empty (their centroids still attract probes)."""
    if patterns:
        pats = rng.integers(0, 256, (patterns, nbytes), dtype=np.uint8)
        x = pats[rng.integers(0, patterns, n)]
    else:
        x = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    cent = rng.integers(0, 256, (nlist, nbytes), dtype=np.uint8)
    a = np.argmin(hamming_np(x, cent), axis=1) if n else np.zeros(0, np.int64)
    empty = np.asarray(sorted(set(empty)), np.int64)
    full = np.setdiff1d(np.arange(nlist), empty)
    if empty.size and full.size:
        a = np.where(np.isin(a, empty), full[0], a)
    return index_from_assignment(x, cent, a, row_ids)

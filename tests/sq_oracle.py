"""CPU oracle of IVF_SQ search: the C ABI's lgpu_ivf_sq_open + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed), the query's codes sat_u8(((double)v - lo) * 255 / (hi - lo)), and for every row of a probed partition
_distance = (float) sum_i (k_i - q_i)^2 (exact integer sum, one rounding to nearest f32).  distance_range [lower, upper)
and the allow mask drop rows before the top-k; maximum_nprobes widens under a prefilter; refine_factor re-ranks the
k * refine_factor best by the exact f32 distance on the raw vectors.  Results ascend by (_distance, _rowid); unused
slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (sq_oracle.c, built together with oracle/oracle.c so that it calls
orc_find_partitions / orc_normalize_f32 itself), which the GPU tests and scripts/bench_ivf_sq.py compare against and
time, and the NumPy mirror below (sq_encode_np, sq_distances_np, sq_search_np), which the CPU tests check the C oracle
against.  `data` is a lancedb_b200.index.IvfSqIndexData.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "sq_oracle.c")
_ORACLE_SRC = os.path.join(_ROOT, "oracle", "oracle.c")
_LIB_PATH = os.path.join(_HERE, "_build", "libsq_oracle.so")
_lib = None
f32 = np.float32


def build(force: bool = False) -> str:
    """gcc -> tests/_build/libsq_oracle.so with oracle/oracle.c's flags (rebuilt when a source is newer)."""
    deps = [_SRC, _ORACLE_SRC, os.path.join(_ROOT, "oracle", "oracle.h")]
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        subprocess.run(["gcc", "-O3", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fno-fast-math", "-fPIC",
                        "-Wall", "-Wextra", "-std=c11", "-pthread", "-shared", "-o", _LIB_PATH, _SRC, _ORACLE_SRC,
                        "-lm"], check=True)
    return _LIB_PATH


def load():
    global _lib
    if _lib is None:
        import oracle
        if not os.path.exists(_LIB_PATH):
            build()
        lib = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        lib.orc_sq_encode.argtypes = [vp, C.c_uint64, C.c_double, C.c_double, vp]
        lib.orc_sq_encode.restype = None
        lib.orc_sq_distance.argtypes = [vp, vp, C.c_uint32]
        lib.orc_sq_distance.restype = C.c_float
        lib.orc_sq_search.argtypes = [C.POINTER(oracle._Index), vp, C.c_double, C.c_double, vp, C.c_uint32,
                                      C.POINTER(oracle._Params), vp, vp, vp, C.c_int]
        lib.orc_sq_search.restype = C.c_int
        _lib = lib
    return _lib


def sq_encode(x, lo: float, hi: float) -> np.ndarray:
    """The C oracle's quantiser on an f32 array of any shape."""
    v = np.ascontiguousarray(x, np.float32)
    out = np.empty(v.shape, np.uint8)
    if v.size:
        load().orc_sq_encode(v.ctypes.data, v.size, float(lo), float(hi), out.ctypes.data)
    return out


def sq_distance(a, b) -> np.float32:
    """The C oracle's distance of two code rows."""
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return f32(load().orc_sq_distance(a.ctypes.data, b.ctypes.data, a.size))


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    import oracle
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, data.dim)
    B = q.shape[0]
    keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.part_offsets, np.uint64),
            np.ascontiguousarray(data.row_ids, np.uint64),
            None if data.vectors is None else np.ascontiguousarray(data.vectors, np.float32),
            np.ascontiguousarray(data.codes, np.uint8)]
    ix = oracle._Index(data.dim, data.nlist, 0, oracle.METRICS[data.metric], data.nrows, keep[0].ctypes.data, None,
                       keep[1].ctypes.data, None, keep[2].ctypes.data, None if keep[3] is None else keep[3].ctypes.data)
    bm = None
    if allow is not None:
        a = np.asarray(allow, bool)
        bm = oracle.allow_bitmap(np.nonzero(a)[0], a.size)
    p = oracle._params(k, nprobes, refine_factor, lower, upper, bm, 0 if allow is None else np.asarray(allow).size,
                       max_nprobes)
    ids = np.empty((B, k), np.uint64); dist = np.empty((B, k), np.float32); cnt = np.empty(B, np.uint32)
    if B and load().orc_sq_search(C.byref(ix), keep[4].ctypes.data, float(data.lo), float(data.hi), q.ctypes.data, B,
                                  C.byref(p), ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data,
                                  int(nthreads) if nthreads else (os.cpu_count() or 1)) != 0:
        raise MemoryError("orc_sq_search failed")
    return ids, dist, cnt


def random_sq_index(rng, n=600, dim=24, nlist=6, metric="l2", with_vectors=True, empty=(1,), unit_centroids=False):
    """A small IVF_SQ index with empty partitions `empty`, a few duplicate rows and non-contiguous row ids.
    unit_centroids: centroids of length 1, so that a cosine index (rows normalised) fills every partition."""
    x = rng.standard_normal((n, dim)).astype(f32)
    x[5:9] = x[4]                                        # duplicates: equal distances, ordered by row id
    c = rng.standard_normal((nlist, dim)).astype(f32)
    if unit_centroids:
        c /= np.linalg.norm(c, axis=1, keepdims=True).astype(f32)
    for p in empty:
        c[p] += 100.0                                    # nothing lands here
    xs = x / np.linalg.norm(x, axis=1, keepdims=True).astype(f32) if metric == "cosine" else x
    assign = ((c * c).sum(1)[None, :] - 2.0 * (xs @ c.T)).argmin(1)
    order = np.argsort(assign, kind="stable")
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(assign, minlength=nlist))
    lo, hi = float(xs.min()) * 0.9, float(xs.max()) * 0.9      # some components saturate
    from lancedb_b200.index import IvfSqIndexData, sq_encode
    return IvfSqIndexData(dim=dim, nlist=nlist, metric=metric, centroids=c, part_offsets=off,
                          codes=sq_encode(xs[order], lo, hi), row_ids=(np.arange(n, dtype=np.uint64) * 3 + 7)[order],
                          lo=lo, hi=hi, vectors=x[order] if with_vectors else None)


# ---- NumPy mirror ----


def sq_encode_np(x, lo: float, hi: float) -> np.ndarray:
    """sat_u8(((double)v - lo) * 255 / (hi - lo)) with numpy's f64 ops, clipped explicitly (a float -> uint8 cast is
    undefined out of range and for NaN)."""
    v = np.asarray(x, np.float32).astype(np.float64)
    if float(hi) == float(lo):
        return np.zeros(v.shape, np.uint8)
    with np.errstate(invalid="ignore", over="ignore"):
        t = ((v - float(lo)) * 255.0) / (float(hi) - float(lo))
    t = np.where(np.isnan(t), 0.0, t)
    return np.trunc(np.clip(t, 0.0, 255.0)).astype(np.uint8)


def sq_distances_np(codes, qcodes) -> np.ndarray:
    """[B, N] (float) sum_i (k_i - q_i)^2, summed exactly in int64."""
    x = np.asarray(codes, np.int64); q = np.asarray(qcodes, np.int64).reshape(-1, x.shape[1])
    d = (x * x).sum(1)[None, :] + (q * q).sum(1)[:, None] - 2 * (q @ x.T)
    return d.astype(np.float32)                          # int64 -> f32 rounds to nearest


def sq_search_np(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
                 max_nprobes: int = 0):
    """The mirror of orc_sq_search (find_partitions and the refine distances from oracle/oracle_np.py)."""
    from oracle import oracle_np as onp
    q = np.asarray(queries, f32).reshape(-1, data.dim)
    B = q.shape[0]
    nprobes = min(nprobes, data.nlist)
    np_max = max(nprobes, min(max_nprobes, data.nlist)) if allow is not None else nprobes
    kk = k * refine_factor if refine_factor else k
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    a = None if allow is None else np.asarray(allow, bool)
    for b in range(B):
        qn = onp.normalize(q[b]) if data.metric == "cosine" else q[b]
        qc = sq_encode_np(qn, data.lo, data.hi)
        cd = np.array([onp.l2(qn, c) for c in data.centroids], f32)
        order = np.lexsort((np.arange(data.nlist), cd))
        for np_use in (nprobes, np_max):
            cands = []
            for p in order[:np_use]:
                if np.isnan(cd[p]):
                    continue
                s, e = int(data.part_offsets[p]), int(data.part_offsets[p + 1])
                if s == e:
                    continue
                d = sq_distances_np(data.codes[s:e], qc)[0]
                for r in range(e - s):
                    rid = int(data.row_ids[s + r])
                    if lower is not None and not d[r] >= f32(lower):
                        continue
                    if upper is not None and not d[r] < f32(upper):
                        continue
                    if a is not None and not (rid < a.size and a[rid]):
                        continue
                    cands.append((d[r], rid, s + r))
            if len(cands) >= k:
                break
        cands.sort()
        cands = cands[:kk]
        if refine_factor and data.vectors is not None:
            dfun = onp.cosine if data.metric == "cosine" else onp.l2
            cands = sorted((dfun(q[b], data.vectors[pos]), rid, pos) for _, rid, pos in cands)
        n = min(k, len(cands))
        ids[b, :n] = [c[1] for c in cands[:n]]
        dist[b, :n] = [c[0] for c in cands[:n]]
        cnt[b] = n
    return ids, dist, cnt

"""CPU oracle of IVF_SQ search: the C ABI's lgpu_ivf_sq_open + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed), the query's codes sat_u8(((double)v - lo) * 255 / (hi - lo)), and for every row of a probed partition
_distance = (float) sum_i (k_i - q_i)^2 (exact integer sum, one rounding to nearest f32).  distance_range [lower, upper)
and the allow mask drop rows before the top-k; maximum_nprobes widens under a prefilter; refine_factor re-ranks the
k * refine_factor best by the exact f32 distance on the raw vectors.  Results ascend by (_distance, _rowid); unused
slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (sq_oracle.c, built into oracle/'s library and run by its IVF search
driver), which the GPU tests and scripts/bench_ivf_sq.py compare against and
time, and the NumPy mirror below (sq_encode_np, sq_distances_np, sq_search_np), which the CPU tests check the C oracle
against.  `data` is a lancedb_b200.index.IvfSqIndexData.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle

f32 = np.float32


def sq_encode(x, lo: float, hi: float) -> np.ndarray:
    """The C oracle's quantiser on an f32 array of any shape."""
    v = np.ascontiguousarray(x, np.float32)
    out = np.empty(v.shape, np.uint8)
    if v.size:
        oracle.load().orc_sq_encode(v.ctypes.data, v.size, float(lo), float(hi), out.ctypes.data)
    return out


def sq_distance(a, b) -> np.float32:
    """The C oracle's distance of two code rows."""
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return f32(oracle.load().orc_sq_distance(a.ctypes.data, b.ctypes.data, a.size))


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, data.dim)
    keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.part_offsets, np.uint64),
            np.ascontiguousarray(data.row_ids, np.uint64),
            None if data.vectors is None else np.ascontiguousarray(data.vectors, np.float32),
            np.ascontiguousarray(data.codes, np.uint8)]
    ix = oracle._Index(data.dim, data.nlist, 0, oracle.METRICS[data.metric], data.nrows, keep[0].ctypes.data, None,
                       keep[1].ctypes.data, None, keep[2].ctypes.data, None if keep[3] is None else keep[3].ctypes.data)
    return oracle.search_call("orc_sq_search", (C.byref(ix), keep[4].ctypes.data, float(data.lo), float(data.hi),
                                                q.ctypes.data), q.shape[0], k, nthreads, nprobes, refine_factor, lower,
                              upper, allow, max_nprobes=max_nprobes)


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
    """The mirror of orc_sq_search (the search loop, find_partitions and the refine distances from
    oracle/oracle_np.py)."""
    from oracle import oracle_np as onp
    q = np.asarray(queries, f32).reshape(-1, data.dim)
    qn = [onp.query(data.metric, x) for x in q]
    qc = [sq_encode_np(x, data.lo, data.hi) for x in qn]
    off = data.part_offsets.astype(np.int64)
    return onp.ivf_search_np(len(q), data, k, nprobes, lambda b: onp.coarse(data.metric, qn[b], data.centroids),
                             lambda b, p: sq_distances_np(data.codes[off[p]:off[p + 1]], qc[b])[0],
                             None if data.vectors is None else lambda b, r: onp.distance(data.metric, q[b],
                                                                                         data.vectors[r]),
                             refine_factor, lower, upper, allow, max_nprobes)

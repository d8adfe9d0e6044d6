"""CPU oracle of multivector (late-interaction, MaxSim) flat search: the C ABI's lgpu_multivec_* semantics.

A row holds n_r >= 0 vectors, a query nq >= 1.  _distance = sum_i min_j cosd(q_i, v_j), summed over i in order in f32
from 0.0f, with cosd the float oracle's lance cosine (orc_cosine_f32: 1 - xy / |x| / sqrt(yy), lance's lane order).
A NaN cosd is skipped by the min; a query vector with no other pair (an empty row, a zero or NaN vector) makes the
row's distance NaN, and NaN distances are never returned.  Results ascend by (_distance, _rowid); distance_range
[lower, upper) applies to the summed distance; an allow mask over row ids drops rows before the top-k; unused slots are
UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (multivec_oracle.c, built into oracle/'s library, so that it calls
orc_cosine_f32 itself), which the GPU tests, smoke() and scripts/bench_multivector.py compare against and time, and
the NumPy mirror below (cosine_matrix_np, distances_np, flat_search_mv_np), which the CPU tests check the C oracle
against.

Rows are given as (values [T, dim], offsets [N+1]); queries as (values [Tq, dim], q_offsets [B+1]).
"""
from __future__ import annotations

import numpy as np

import oracle

f32 = np.float32


def offsets_of(lengths) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.uint64)


def _rows(values, offsets):
    v = np.ascontiguousarray(values, np.float32)
    off = np.ascontiguousarray(offsets, np.uint64)
    return v, off


def _queries(queries, q_offsets):
    q = np.ascontiguousarray(queries, np.float32)
    qo = np.ascontiguousarray(q_offsets, np.uint32)
    return q, qo


def distances(values, offsets, queries, q_offsets, nthreads: int = 0) -> np.ndarray:
    """[B, N] f32 MaxSim distances from the C oracle (NaN: no distance)."""
    v, off = _rows(values, offsets)
    q, qo = _queries(queries, q_offsets)
    N, B = off.size - 1, qo.size - 1
    out = np.empty((B, N), np.float32)
    if out.size and oracle.load().orc_multivec_distances(v.ctypes.data, off.ctypes.data, N, v.shape[1], q.ctypes.data,
                                                         qo.ctypes.data, B, out.ctypes.data,
                                                         oracle.threads(nthreads)) != 0:
        raise MemoryError("orc_multivec_distances failed")
    return out


def flat_search_mv(values, offsets, queries, q_offsets, k: int, row_ids=None, lower=None, upper=None, allow=None,
                   nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    v, off = _rows(values, offsets)
    q, qo = _queries(queries, q_offsets)
    rid = None if row_ids is None else np.ascontiguousarray(row_ids, np.uint64)
    return oracle.search_call("orc_multivec_search", (v.ctypes.data, off.ctypes.data, off.size - 1,
                                                      v.shape[1] if v.ndim == 2 else 1,
                                                      None if rid is None else rid.ctypes.data, q.ctypes.data,
                                                      qo.ctypes.data), qo.size - 1, k, nthreads, lower=lower,
                              upper=upper, allow=allow)


# ---- NumPy mirror ----


def lance_dot_np(x, Y) -> np.ndarray:
    """dot(x, y) for every row y of Y [n, d] in lance's order: 16 lane sums over whole chunks of 16, the lanes added
    in order, the remainder summed sequentially, result = remainder + lanes.  Every op is one f32 rounding."""
    x = np.asarray(x, f32)
    Y = np.asarray(Y, f32)
    d = x.size
    nch = d // 16
    lanes = np.zeros((Y.shape[0], 16), f32)
    for c in range(nch):
        lanes = (lanes + (x[c * 16:(c + 1) * 16][None, :] * Y[:, c * 16:(c + 1) * 16]).astype(f32)).astype(f32)
    t = np.zeros(Y.shape[0], f32)
    for l in range(16):
        t = (t + lanes[:, l]).astype(f32)
    s = np.zeros(Y.shape[0], f32)
    for i in range(nch * 16, d):
        s = (s + (x[i] * Y[:, i]).astype(f32)).astype(f32)
    return (s + t).astype(f32)


def cosine_matrix_np(Q, V) -> np.ndarray:
    """[nq, n] cosd(Q[i], V[j]) = 1 - xy / |x| / sqrt(yy), as orc_cosine_f32 rounds it."""
    Q = np.asarray(Q, f32)
    V = np.asarray(V, f32)
    yy = np.sqrt(np.stack([lance_dot_np(v, v[None, :])[0] for v in V]) if len(V) else np.zeros(0, f32)).astype(f32)
    out = np.empty((Q.shape[0], V.shape[0]), f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i, x in enumerate(Q):
            xn = np.sqrt(lance_dot_np(x, x[None, :])[0]).astype(f32)
            xy = lance_dot_np(x, V)
            out[i] = (f32(1) - ((xy / xn).astype(f32) / yy).astype(f32)).astype(f32)
    return out


def distances_np(values, offsets, queries, q_offsets) -> np.ndarray:
    """[B, N] MaxSim distances: NaN-skipping min over each row's run, then the in-order f32 sum over query vectors."""
    v, off = _rows(values, offsets)
    q, qo = _queries(queries, q_offsets)
    N, B = off.size - 1, qo.size - 1
    cos = cosine_matrix_np(q, v) if len(q) and len(v) else np.zeros((len(q), len(v)), f32)
    out = np.empty((B, N), f32)
    for r in range(N):
        seg = cos[:, int(off[r]):int(off[r + 1])]
        with np.errstate(all="ignore"):
            m = np.fmin.reduce(seg, axis=1) if seg.shape[1] else np.full(len(q), np.nan, f32)   # fmin skips NaN
        for b in range(B):
            s = f32(0)
            for i in range(int(qo[b]), int(qo[b + 1])):
                s = f32(s + m[i])
            out[b, r] = s
    return out


def flat_search_mv_np(values, offsets, queries, q_offsets, k: int, row_ids=None, lower=None, upper=None, allow=None):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32); allow: optional bool mask over row ids."""
    D = distances_np(values, offsets, queries, q_offsets)
    B, N = D.shape
    rid = np.arange(N, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    keep = np.ones(N, bool)
    if allow is not None:
        a = np.asarray(allow, bool)
        inside = rid < a.size
        keep = np.zeros(N, bool)
        keep[inside] = a[rid[inside].astype(np.int64)]
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    for b in range(B):
        m = keep & ~np.isnan(D[b])
        if lower is not None:
            m &= D[b] >= np.float32(lower)
        if upper is not None:
            m &= D[b] < np.float32(upper)
        cols = np.nonzero(m)[0]
        order = np.lexsort((rid[cols], D[b, cols]))[:k]
        n = len(order)
        ids[b, :n] = rid[cols[order]]
        dist[b, :n] = D[b, cols[order]]
        cnt[b] = n
    return ids, dist, cnt

"""CPU oracle of IVF_RQ search: the C ABI's lgpu_ivf_rq_open + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed), the rotated query rq_i = dot(P row i, q) and per probed partition the 4-bit grid of q' = rq - rc_p (lo, delta,
u, S, qq = l2(rq, rc_p)), and for every row of the partition the RaBitQ estimate
    y = delta * (float)(2 ip - S) + lo * (float)(2 pc - dim),   est = (add + qq) + scale * y
(cosine: 0.5 est), every operation rounded to f32 on its own.  A slot whose delta is not finite has no rows and a NaN
estimate is never returned.  distance_range [lower, upper) and the allow mask drop rows before the top-k;
maximum_nprobes widens under a prefilter; refine_factor re-ranks the k * refine_factor best by the exact f32 distance on
the raw vectors.  Results ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (rq_oracle.c, built into oracle/'s library and run by its IVF search
driver), which the GPU tests and
scripts/bench_ivf_rq.py compare against and time, and the NumPy mirror below (rq_rotate_np, rq_slot_np,
rq_estimates_np, rq_search_np), which the CPU tests check the C oracle against.  `data` is a
lancedb_b200.index.IvfRqIndexData.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle

f32 = np.float32


def rq_rotate(P, x) -> np.ndarray:
    """The C oracle's rotation: out[v][i] = orc_dot_f32(P row i, x[v])."""
    P = np.ascontiguousarray(P, f32); x = np.ascontiguousarray(x, f32).reshape(-1, P.shape[0])
    out = np.empty_like(x)
    if x.size:
        oracle.load().orc_rq_rotate(P.ctypes.data, x.ctypes.data, x.shape[0], P.shape[0], out.ctypes.data)
    return out


def rq_slot(rq, rc):
    """The C oracle's grid of one probe slot: (u [dim] u8, lo, delta, qq as f32, S)."""
    rq = np.ascontiguousarray(rq, f32); rc = np.ascontiguousarray(rc, f32)
    qp = np.empty_like(rq); u = np.empty(rq.size, np.uint8); grid = np.empty(3, f32); S = np.zeros(1, np.uint32)
    oracle.load().orc_rq_slot(rq.ctypes.data, rc.ctypes.data, rq.size, qp.ctypes.data, u.ctypes.data, grid.ctypes.data,
                       S.ctypes.data)
    return u, grid[0], grid[1], grid[2], int(S[0])


def rq_estimates(codes, add, scale, u, lo, delta, qq, S, dim, metric="l2") -> np.ndarray:
    """The C oracle's reported distance of every row of codes [N, ceil(dim / 8)] in one slot."""
    codes = np.ascontiguousarray(codes, np.uint8); u = np.ascontiguousarray(u, np.uint8)
    grid = np.array([lo, delta, qq], f32)
    lib = oracle.load()
    return np.array([lib.orc_rq_estimate(codes[r].ctypes.data, float(add[r]), float(scale[r]), u.ctypes.data,
                                         grid.ctypes.data, int(S), int(dim), oracle.METRICS[metric])
                     for r in range(codes.shape[0])], f32)


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, data.dim)
    keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.part_offsets, np.uint64),
            np.ascontiguousarray(data.row_ids, np.uint64),
            None if data.vectors is None else np.ascontiguousarray(data.vectors, np.float32),
            np.ascontiguousarray(data.codes, np.uint8), np.ascontiguousarray(data.rotation, np.float32),
            np.ascontiguousarray(data.add_factors, np.float32), np.ascontiguousarray(data.scale_factors, np.float32)]
    ix = oracle._Index(data.dim, data.nlist, 0, oracle.METRICS[data.metric], data.nrows, keep[0].ctypes.data, None,
                       keep[1].ctypes.data, None, keep[2].ctypes.data, None if keep[3] is None else keep[3].ctypes.data)
    return oracle.search_call("orc_rq_search", (C.byref(ix), keep[5].ctypes.data, keep[4].ctypes.data,
                                                keep[6].ctypes.data, keep[7].ctypes.data, q.ctypes.data), q.shape[0], k,
                              nthreads, nprobes, refine_factor, lower, upper, allow, max_nprobes=max_nprobes)


def random_rq_index(rng, n=600, dim=24, nlist=6, metric="l2", with_vectors=True, empty=(1,), seed=7,
                    unit_centroids=False):
    """A small IVF_RQ index with empty partitions `empty`, a few duplicate rows and non-contiguous row ids.
    unit_centroids: centroids of length 1, so that a cosine index (rows normalised) fills every partition."""
    from lancedb_b200.index import IvfRqIndexData, rq_encode, rq_rotation
    x = rng.standard_normal((n, dim)).astype(f32)
    if n > 8:
        x[5:9] = x[4]                                    # duplicates: equal estimates, ordered by row id
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
    P = rq_rotation(dim, seed)
    codes, add, scale = rq_encode(xs[order], c, assign[order], P)
    return IvfRqIndexData(dim=dim, nlist=nlist, metric=metric, centroids=c, rotation=P, part_offsets=off, codes=codes,
                          add_factors=add, scale_factors=scale,
                          row_ids=(np.arange(n, dtype=np.uint64) * 3 + 7)[order],
                          vectors=x[order] if with_vectors else None)


# ---- NumPy mirror ----


def rq_rotate_np(P, x) -> np.ndarray:
    """dot(P row i, x[v]) in lance's lane order (remainder first, 16 lane sums over the chunks, lanes summed in
    order), vectorised over the rows of P: every addition is one f32 rounding in the same order as orc_dot_f32."""
    P = np.asarray(P, f32); x = np.asarray(x, f32).reshape(-1, P.shape[0])
    dim = P.shape[0]
    nch = dim // 16
    out = np.empty((x.shape[0], dim), f32)
    for v in range(x.shape[0]):
        s = np.zeros(dim, f32)
        for i in range(nch * 16, dim):
            s = (s + P[:, i] * x[v, i]).astype(f32)
        sums = np.zeros((dim, 16), f32)
        for c in range(nch):
            sums = (sums + P[:, c * 16:(c + 1) * 16] * x[v, c * 16:(c + 1) * 16]).astype(f32)
        t = np.zeros(dim, f32)
        for lane in range(16):
            t = (t + sums[:, lane]).astype(f32)
        out[v] = s + t
    return out


def rq_slot_np(rq, rc):
    """(u [dim] u8, lo, delta, qq as f32, S) of one probe slot with numpy's f32 operations."""
    from oracle import oracle_np as onp
    qp = (np.asarray(rq, f32) - np.asarray(rc, f32)).astype(f32)
    if np.isnan(qp).any():
        lo = hi = f32(np.nan)
    else:
        lo, hi = f32(qp.min()), f32(qp.max())
        zero = qp == 0
        if lo == 0:                                      # -0 orders below +0
            lo = f32(-0.0) if np.any(zero & np.signbit(qp)) else f32(0.0)
        if hi == 0:
            hi = f32(0.0) if np.any(zero & ~np.signbit(qp)) else f32(-0.0)
    with np.errstate(invalid="ignore", over="ignore"):
        delta = f32(f32(hi - lo) / f32(15))
    if delta > 0 and np.isfinite(delta):
        with np.errstate(over="ignore"):
            f = ((qp - lo).astype(f32) / delta).astype(f32) + f32(0.5)
        u = np.minimum(np.trunc(f), 15).astype(np.uint8)
    else:
        u = np.zeros(qp.size, np.uint8)
    return u, lo, delta, f32(onp.l2(rq, rc)), int(u.astype(np.int64).sum())


def rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, metric="l2", ip_only=False) -> np.ndarray:
    """[N] reported estimates of the rows of codes [N, ceil(dim / 8)] in one slot (ip = sum b_i u_i in int64);
    ip_only: the integers ip themselves."""
    bits = np.unpackbits(np.asarray(codes, np.uint8), axis=1, bitorder="little")[:, :dim].astype(np.int64)
    ip = bits @ np.asarray(u, np.int64)
    if ip_only:
        return ip
    pc = bits.sum(1)
    with np.errstate(invalid="ignore", over="ignore"):
        y = (f32(delta) * (2 * ip - S).astype(f32)).astype(f32) + (f32(lo) * (2 * pc - dim).astype(f32)).astype(f32)
        est = (np.asarray(add, f32) + f32(qq)).astype(f32) + (np.asarray(scale, f32) * y.astype(f32)).astype(f32)
        est = est.astype(f32)
        if metric == "cosine":
            est = (f32(0.5) * est).astype(f32)
    return est if np.isfinite(delta) else np.full(est.shape, np.nan, f32)


def rq_search_np(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
                 max_nprobes: int = 0):
    """The mirror of orc_rq_search (the search loop, find_partitions, normalisation and the refine distances from
    oracle/oracle_np.py)."""
    from oracle import oracle_np as onp
    q = np.asarray(queries, f32).reshape(-1, data.dim)
    qn = [onp.query(data.metric, x) for x in q]
    rq = [rq_rotate_np(data.rotation, x)[0] for x in qn]
    rc = rq_rotate_np(data.rotation, data.centroids)
    off = data.part_offsets.astype(np.int64)

    def partition(b, p):
        s, e = off[p], off[p + 1]
        return rq_estimates_np(data.codes[s:e], data.add_factors[s:e], data.scale_factors[s:e],
                               *rq_slot_np(rq[b], rc[p]), data.dim, data.metric)

    return onp.ivf_search_np(len(q), data, k, nprobes, lambda b: onp.coarse(data.metric, qn[b], data.centroids),
                             partition, None if data.vectors is None else lambda b, r: onp.distance(data.metric, q[b],
                                                                                                    data.vectors[r]),
                             refine_factor, lower, upper, allow, max_nprobes)

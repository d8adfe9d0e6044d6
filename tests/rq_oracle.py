"""CPU oracle of IVF_RQ search: the C ABI's lgpu_ivf_rq_open + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed), the rotated query rq_i = dot(P row i, q) and per probed partition the 4-bit grid of q' = rq - rc_p (lo, delta,
u, S, qq = l2(rq, rc_p)), and for every row of the partition the RaBitQ estimate
    y = delta * (float)(2 ip - S) + lo * (float)(2 pc - dim),   est = (add + qq) + scale * y
(cosine: 0.5 est), every operation rounded to f32 on its own.  A slot whose delta is not finite has no rows and a NaN
estimate is never returned.  distance_range [lower, upper) and the allow mask drop rows before the top-k;
maximum_nprobes widens under a prefilter; refine_factor re-ranks the k * refine_factor best by the exact f32 distance on
the raw vectors.  Results ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (rq_oracle.c, built together with oracle/oracle.c so that it calls
orc_find_partitions / orc_normalize_f32 / orc_dot_f32 / orc_l2_f32 / orc_distance_f32 itself), which the GPU tests and
scripts/bench_ivf_rq.py compare against and time, and the NumPy mirror below (rq_rotate_np, rq_slot_np,
rq_estimates_np, rq_search_np), which the CPU tests check the C oracle against.  `data` is a
lancedb_b200.index.IvfRqIndexData.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "rq_oracle.c")
_ORACLE_SRC = os.path.join(_ROOT, "oracle", "oracle.c")
_LIB_PATH = os.path.join(_HERE, "_build", "librq_oracle.so")
_lib = None
f32 = np.float32


def build(force: bool = False) -> str:
    """gcc -> tests/_build/librq_oracle.so with oracle/oracle.c's flags (rebuilt when a source is newer)."""
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
        lib.orc_rq_rotate.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp]
        lib.orc_rq_rotate.restype = None
        lib.orc_rq_slot.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
        lib.orc_rq_slot.restype = None
        lib.orc_rq_estimate.argtypes = [vp, C.c_float, C.c_float, vp, vp, C.c_uint32, C.c_uint32, C.c_int]
        lib.orc_rq_estimate.restype = C.c_float
        lib.orc_rq_search.argtypes = [C.POINTER(oracle._Index), vp, vp, vp, vp, vp, C.c_uint32,
                                      C.POINTER(oracle._Params), vp, vp, vp, C.c_int]
        lib.orc_rq_search.restype = C.c_int
        _lib = lib
    return _lib


def rq_rotate(P, x) -> np.ndarray:
    """The C oracle's rotation: out[v][i] = orc_dot_f32(P row i, x[v])."""
    P = np.ascontiguousarray(P, f32); x = np.ascontiguousarray(x, f32).reshape(-1, P.shape[0])
    out = np.empty_like(x)
    if x.size:
        load().orc_rq_rotate(P.ctypes.data, x.ctypes.data, x.shape[0], P.shape[0], out.ctypes.data)
    return out


def rq_slot(rq, rc):
    """The C oracle's grid of one probe slot: (u [dim] u8, lo, delta, qq as f32, S)."""
    rq = np.ascontiguousarray(rq, f32); rc = np.ascontiguousarray(rc, f32)
    qp = np.empty_like(rq); u = np.empty(rq.size, np.uint8); grid = np.empty(3, f32); S = np.zeros(1, np.uint32)
    load().orc_rq_slot(rq.ctypes.data, rc.ctypes.data, rq.size, qp.ctypes.data, u.ctypes.data, grid.ctypes.data,
                       S.ctypes.data)
    return u, grid[0], grid[1], grid[2], int(S[0])


def rq_estimates(codes, add, scale, u, lo, delta, qq, S, dim, metric="l2") -> np.ndarray:
    """The C oracle's reported distance of every row of codes [N, ceil(dim / 8)] in one slot."""
    import oracle
    codes = np.ascontiguousarray(codes, np.uint8); u = np.ascontiguousarray(u, np.uint8)
    grid = np.array([lo, delta, qq], f32)
    lib = load()
    return np.array([lib.orc_rq_estimate(codes[r].ctypes.data, float(add[r]), float(scale[r]), u.ctypes.data,
                                         grid.ctypes.data, int(S), int(dim), oracle.METRICS[metric])
                     for r in range(codes.shape[0])], f32)


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    import oracle
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, data.dim)
    B = q.shape[0]
    keep = [np.ascontiguousarray(data.centroids, np.float32), np.ascontiguousarray(data.part_offsets, np.uint64),
            np.ascontiguousarray(data.row_ids, np.uint64),
            None if data.vectors is None else np.ascontiguousarray(data.vectors, np.float32),
            np.ascontiguousarray(data.codes, np.uint8), np.ascontiguousarray(data.rotation, np.float32),
            np.ascontiguousarray(data.add_factors, np.float32), np.ascontiguousarray(data.scale_factors, np.float32)]
    ix = oracle._Index(data.dim, data.nlist, 0, oracle.METRICS[data.metric], data.nrows, keep[0].ctypes.data, None,
                       keep[1].ctypes.data, None, keep[2].ctypes.data, None if keep[3] is None else keep[3].ctypes.data)
    bm = None
    if allow is not None:
        a = np.asarray(allow, bool)
        bm = oracle.allow_bitmap(np.nonzero(a)[0], a.size)
    p = oracle._params(k, nprobes, refine_factor, lower, upper, bm, 0 if allow is None else np.asarray(allow).size,
                       max_nprobes)
    ids = np.empty((B, k), np.uint64); dist = np.empty((B, k), np.float32); cnt = np.empty(B, np.uint32)
    if B and load().orc_rq_search(C.byref(ix), keep[5].ctypes.data, keep[4].ctypes.data, keep[6].ctypes.data,
                                  keep[7].ctypes.data, q.ctypes.data, B, C.byref(p), ids.ctypes.data,
                                  dist.ctypes.data, cnt.ctypes.data,
                                  int(nthreads) if nthreads else (os.cpu_count() or 1)) != 0:
        raise MemoryError("orc_rq_search failed")
    return ids, dist, cnt


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
    """The mirror of orc_rq_search (find_partitions, normalisation and the refine distances from oracle/oracle_np.py)."""
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
    rc = rq_rotate_np(data.rotation, data.centroids)
    for b in range(B):
        qn = onp.normalize(q[b]) if data.metric == "cosine" else q[b]
        rq = rq_rotate_np(data.rotation, qn)[0]
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
                u, lo, delta, qq, S = rq_slot_np(rq, rc[p])
                if not np.isfinite(delta):
                    continue
                d = rq_estimates_np(data.codes[s:e], data.add_factors[s:e], data.scale_factors[s:e], u, lo, delta,
                                    qq, S, data.dim, data.metric)
                for r in range(e - s):
                    rid = int(data.row_ids[s + r])
                    if np.isnan(d[r]):
                        continue
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
            cands = [(dfun(q[b], data.vectors[pos]), rid, pos) for _, rid, pos in cands]
            cands = sorted(c for c in cands if not np.isnan(c[0]))     # a NaN distance is never returned
        n = min(k, len(cands))
        ids[b, :n] = [c[1] for c in cands[:n]]
        dist[b, :n] = [c[0] for c in cands[:n]]
        cnt[b] = n
    return ids, dist, cnt

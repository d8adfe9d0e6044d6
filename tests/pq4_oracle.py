"""CPU oracle of 4-bit IVF_PQ search: the C ABI's lgpu_index_open(nbits = 4) + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed).  Per probed partition, with r = q - c_p (l2, cosine) or q (dot): the float table T [m][16] of the 8-bit path on
the 16 codewords, qmin = min T, qmax = max over adjacent sub-space pairs of the summed row maxima (NaN skipped), the u8
table Q = sat_u8(round_half_away(((T - qmin) * 255) / (qmax - qmin))), and per row
d = ((float) S * (qmax - qmin)) / 255 + qmin * (float) m with S = sum_i Q[i][code_i] (cosine 0.5 d, dot d - (m - 1)).
A NaN d is never returned; distance_range [lower, upper) and the allow mask drop rows before the top-k;
maximum_nprobes widens under a prefilter; refine_factor re-ranks the k * refine_factor best by the exact f32 distance on
the raw vectors.  Results ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (pq4_oracle.c, built together with oracle/oracle.c so that it calls
orc_find_partitions / orc_normalize_f32 / orc_l2_subvec / orc_dot_f32 itself), which the GPU tests and
scripts/bench_ivf_pq4.py compare against and time, and the NumPy mirror below (quant_np, distance_np, tables_np,
pq4_search_np), which the CPU tests check the C oracle against.  `data` is a lancedb_b200.index.IvfPqIndexData with
num_bits = 4.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "pq4_oracle.c")
_ORACLE_SRC = os.path.join(_ROOT, "oracle", "oracle.c")
_LIB_PATH = os.path.join(_HERE, "_build", "libpq4_oracle.so")
_lib = None
f32 = np.float32


def build(force: bool = False) -> str:
    """gcc -> tests/_build/libpq4_oracle.so with oracle/oracle.c's flags (rebuilt when a source is newer)."""
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
        vp, u32 = C.c_void_p, C.c_uint32
        lib.orc_pq4_quant.argtypes = [C.c_float, C.c_float, C.c_float]
        lib.orc_pq4_quant.restype = C.c_uint8
        lib.orc_pq4_distance.argtypes = [u32, C.c_float, C.c_float, u32, C.c_int]
        lib.orc_pq4_distance.restype = C.c_float
        lib.orc_pq4_tables.argtypes = [C.POINTER(oracle._Index), vp, u32, vp, vp]
        lib.orc_pq4_tables.restype = None
        lib.orc_pq4_partition_distances.argtypes = [C.POINTER(oracle._Index), vp, u32, vp]
        lib.orc_pq4_partition_distances.restype = None
        lib.orc_pq4_search.argtypes = [C.POINTER(oracle._Index), vp, u32, C.POINTER(oracle._Params), vp, vp, vp,
                                       C.c_int]
        lib.orc_pq4_search.restype = C.c_int
        _lib = lib
    return _lib


def _index(data):
    """(orc_index, arrays it points into)"""
    import oracle
    assert data.num_bits == 4
    keep = [np.ascontiguousarray(data.centroids, f32), np.ascontiguousarray(data.codebook, f32),
            np.ascontiguousarray(data.part_offsets, np.uint64), np.ascontiguousarray(data.codes_t, np.uint8),
            np.ascontiguousarray(data.row_ids, np.uint64),
            None if data.vectors is None else np.ascontiguousarray(data.vectors, f32)]
    ix = oracle._Index(data.dim, data.nlist, data.m, oracle.METRICS[data.metric], data.nrows,
                       *[None if a is None else a.ctypes.data for a in keep])
    return ix, keep


def quant(t, qmin, qmax) -> np.ndarray:
    """The C oracle's orc_pq4_quant, element-wise."""
    lib = load()
    t = np.asarray(t, f32)
    return np.array([lib.orc_pq4_quant(float(v), float(qmin), float(qmax)) for v in t.ravel()],
                    np.uint8).reshape(t.shape)


def distance(S, qmin, qmax, m, metric) -> np.ndarray:
    """The C oracle's orc_pq4_distance, element-wise."""
    import oracle
    lib = load()
    S = np.asarray(S, np.uint32)
    return np.array([lib.orc_pq4_distance(int(s), float(qmin), float(qmax), int(m), oracle.METRICS[metric])
                     for s in S.ravel()], f32).reshape(S.shape)


def tables(data, qn, part):
    """(Q [m, 16] u8, qmin, qmax) of one probe slot from the C oracle; qn normalised for cosine."""
    ix, keep = _index(data)
    q = np.ascontiguousarray(qn, f32)
    Q = np.empty((data.m, 16), np.uint8)
    qmm = np.empty(2, f32)
    load().orc_pq4_tables(C.byref(ix), q.ctypes.data, int(part), Q.ctypes.data, qmm.ctypes.data)
    return Q, qmm[0], qmm[1]


def partition_distances(data, q, part) -> np.ndarray:
    """d of every row of partition `part` from the C oracle (q: the raw query)."""
    ix, keep = _index(data)
    q = np.ascontiguousarray(q, f32)
    n = int(data.part_offsets[part + 1] - data.part_offsets[part])
    out = np.empty(max(n, 1), f32)
    load().orc_pq4_partition_distances(C.byref(ix), q.ctypes.data, int(part), out.ctypes.data)
    return out[:n]


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    import oracle
    q = np.ascontiguousarray(queries, f32).reshape(-1, data.dim)
    B = q.shape[0]
    ix, keep = _index(data)
    bm = None
    if allow is not None:
        a = np.asarray(allow, bool)
        bm = oracle.allow_bitmap(np.nonzero(a)[0], a.size)
    p = oracle._params(k, nprobes, refine_factor, lower, upper, bm, 0 if allow is None else np.asarray(allow).size,
                       max_nprobes)
    ids = np.empty((B, k), np.uint64); dist = np.empty((B, k), f32); cnt = np.empty(B, np.uint32)
    if B and load().orc_pq4_search(C.byref(ix), q.ctypes.data, B, C.byref(p), ids.ctypes.data, dist.ctypes.data,
                                   cnt.ctypes.data, int(nthreads) if nthreads else (os.cpu_count() or 1)) != 0:
        raise MemoryError("orc_pq4_search failed")
    return ids, dist, cnt


def random_pq4_index(rng, n=600, dim=32, nlist=6, m=8, metric="l2", with_vectors=True, empty=(1,), sizes=None,
                     scale=1.0):
    """A small 4-bit IVF_PQ index: partitions `empty` hold no rows (or explicit `sizes`), a few duplicate rows, random
    nibble codes and non-contiguous ascending row ids."""
    from lancedb_b200.index import IvfPqIndexData
    dsub = dim // m
    c = (rng.standard_normal((nlist, dim)) * scale).astype(f32)
    if metric == "cosine":
        c /= np.linalg.norm(c, axis=1, keepdims=True)
    if sizes is None:
        w = rng.random(nlist) + 0.2
        for p in empty:
            w[p] = 0.0
        sizes = np.floor(w / w.sum() * n).astype(np.int64)
        sizes[int(np.argmax(w))] += n - sizes.sum()
    sizes = np.asarray(sizes, np.int64)
    n = int(sizes.sum())
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    cb = (rng.standard_normal((m, 16, dsub)) * 0.5 * scale).astype(f32)
    codes = rng.integers(0, 256, (n, m // 2), dtype=np.uint8)          # row-major packed bytes
    if n > 9:
        codes[5:9] = codes[4]                                          # duplicates: tied sums, ordered by row id
    codes_t = np.empty(n * (m // 2), np.uint8)
    for p in range(nlist):
        a, b = int(off[p]), int(off[p + 1])
        codes_t[a * (m // 2):b * (m // 2)] = codes[a:b].T.reshape(-1)
    perm = rng.permutation(n).astype(np.uint64) * 3 + 7
    ids = np.empty(n, np.uint64)
    for p in range(nlist):
        a, b = int(off[p]), int(off[p + 1])
        ids[a:b] = np.sort(perm[a:b])
    vec = (rng.standard_normal((n, dim)) * scale).astype(f32) if with_vectors else None
    ix = IvfPqIndexData(dim, nlist, m, metric, c, cb, off, codes_t, ids, vec, num_bits=4)
    ix.validate()
    return ix


def row_major_codes(data) -> np.ndarray:
    """[n, m/2] packed bytes in partition order (the LGPU_CODES_ROW_MAJOR form of data.codes_t)."""
    w = data.code_bytes
    out = np.empty((data.nrows, w), np.uint8)
    for p in range(data.nlist):
        a, b = int(data.part_offsets[p]), int(data.part_offsets[p + 1])
        out[a:b] = data.codes_t[a * w:b * w].reshape(w, b - a).T
    return out


# ---- NumPy mirror ----


def quant_np(T, qmin, qmax) -> np.ndarray:
    """sat_u8(round_half_away(((T - qmin) * 255) / (qmax - qmin))) with each op an f32 op; the rounding is done in f64,
    where x + 0.5 is exact, and NaN / below 0 -> 0, above 255 -> 255."""
    T = np.asarray(T, f32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        x = ((T - f32(qmin)).astype(f32) * f32(255)).astype(f32) / f32(f32(qmax) - f32(qmin))
        x = x.astype(f32).astype(np.float64)
        r = np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5))
    r = np.where(np.isnan(r) | (r <= 0), 0.0, np.minimum(r, 255.0))
    return r.astype(np.uint8)


def distance_np(S, qmin, qmax, m, metric) -> np.ndarray:
    """((float) S * (qmax - qmin)) / 255 + qmin * (float) m, each op in f32, then cosine 0.5 d / dot d - (m - 1)."""
    S = np.asarray(S, np.uint32).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = ((S * f32(f32(qmax) - f32(qmin))).astype(f32) / f32(255)).astype(f32) + f32(f32(qmin) * f32(m))
        d = d.astype(f32)
        if metric == "cosine":
            d = (d * f32(0.5)).astype(f32)
        elif metric == "dot":
            d = (d - f32(m - 1)).astype(f32)
    return d


def fold_np(T):
    """(qmin, qmax) of T [m, 16]: NaN-skipping min of every entry; NaN-skipping max over i < m - 1 of the f32 sum of the
    row maxima of sub-spaces i and i + 1 (an all-NaN fold is +inf / -inf)."""
    T = np.asarray(T, f32)
    ok = ~np.isnan(T)
    qmin = f32(T[ok].min()) if ok.any() else f32(np.inf)
    rmax = np.where(ok, T, f32(-np.inf)).max(1).astype(f32)
    with np.errstate(invalid="ignore"):
        w = (rmax[:-1] + rmax[1:]).astype(f32)
    w = w[~np.isnan(w)]
    qmax = f32(w.max()) if w.size else f32(-np.inf)
    return qmin, qmax


def float_table_np(data, qn, part) -> np.ndarray:
    """T [m, 16]: the 8-bit path's table entries on the 16 codewords (oracle_np.l2_subvec_batch / 1 - dot)."""
    from oracle import oracle_np as onp
    qn = np.asarray(qn, f32)
    r = qn if data.metric == "dot" else (qn - data.centroids[part]).astype(f32)
    d = data.dsub
    T = np.empty((data.m, 16), f32)
    for i in range(data.m):
        sub = r[i * d:(i + 1) * d]
        if data.metric == "dot":
            T[i] = [f32(f32(1) - onp.dot(sub, c)) for c in data.codebook[i]]
        else:
            T[i] = onp.l2_subvec_batch(sub, data.codebook[i])
    return T


def tables_np(data, qn, part):
    """(Q [m, 16] u8, qmin, qmax) of one probe slot; qn normalised for cosine."""
    T = float_table_np(data, qn, part)
    qmin, qmax = fold_np(T)
    return quant_np(T, qmin, qmax), qmin, qmax


def sums_np(Q, packed) -> np.ndarray:
    """[B, N] sum_i Q[b][i][code_i] of packed rows [N, m/2] (Q: [B, m, 16] or [m, 16]), exact in int64."""
    from lancedb_b200.index import unpack_pq4
    Q = np.asarray(Q, np.int64)
    if Q.ndim == 2:
        Q = Q[None]
    codes = unpack_pq4(packed).astype(np.int64)                  # [N, m]
    m = codes.shape[1]
    return np.stack([Q[b][np.arange(m)[None, :], codes].sum(1) for b in range(Q.shape[0])])


def partition_distances_np(data, qn, part) -> np.ndarray:
    Q, qmin, qmax = tables_np(data, qn, part)
    a, b = int(data.part_offsets[part]), int(data.part_offsets[part + 1])
    w = data.code_bytes
    packed = data.codes_t[a * w:b * w].reshape(w, b - a).T
    return distance_np(sums_np(Q, packed)[0], qmin, qmax, data.m, data.metric)


def pq4_search_np(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
                  max_nprobes: int = 0):
    """The mirror of orc_pq4_search (find_partitions and the refine distances from oracle/oracle_np.py)."""
    from oracle import oracle_np as onp
    q = np.asarray(queries, f32).reshape(-1, data.dim)
    B = q.shape[0]
    nprobes = min(nprobes, data.nlist)
    np_max = max(nprobes, min(max_nprobes, data.nlist)) if allow is not None else nprobes
    kk = k * refine_factor if refine_factor else k
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, f32)
    cnt = np.zeros(B, np.uint32)
    a = None if allow is None else np.asarray(allow, bool)
    for b in range(B):
        qn = onp.normalize(q[b]) if data.metric == "cosine" else q[b]
        if data.metric == "dot":
            cd = np.array([f32(f32(1) - onp.dot(qn, c)) for c in data.centroids], f32)
        else:
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
                d = partition_distances_np(data, qn, p)
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
            dfun = {"cosine": onp.cosine, "l2": onp.l2, "dot": lambda x, y: f32(f32(1) - onp.dot(x, y))}[data.metric]
            cands = [(dfun(q[b], data.vectors[pos]), rid, pos) for _, rid, pos in cands]
            cands = sorted(c for c in cands if not np.isnan(c[0]))     # a NaN distance is never returned
        n = min(k, len(cands))
        ids[b, :n] = [c[1] for c in cands[:n]]
        dist[b, :n] = [c[0] for c in cands[:n]]
        cnt[b] = n
    return ids, dist, cnt

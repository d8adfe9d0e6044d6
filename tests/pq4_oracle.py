"""CPU oracle of 4-bit IVF_PQ search: the C ABI's lgpu_index_open(nbits = 4) + lgpu_search semantics.

Per query (normalised first for cosine): the nprobes nearest partitions (find_partitions; a NaN centroid distance is not
probed).  Per probed partition, with r = q - c_p (l2, cosine) or q (dot): the float table T [m][16] of the 8-bit path on
the 16 codewords, qmin = min T, qmax = max over adjacent sub-space pairs of the summed row maxima (NaN skipped), the u8
table Q = sat_u8(round_half_away(((T - qmin) * 255) / (qmax - qmin))), and per row
d = ((float) S * (qmax - qmin)) / 255 + qmin * (float) m with S = sum_i Q[i][code_i] (cosine 0.5 d, dot d - (m - 1)).
A NaN d is never returned; distance_range [lower, upper) and the allow mask drop rows before the top-k;
maximum_nprobes widens under a prefilter; refine_factor re-ranks the k * refine_factor best by the exact f32 distance on
the raw vectors.  Results ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (pq4_oracle.c, built into oracle/'s library and run by its IVF search
driver), which the GPU tests and
scripts/bench_ivf_pq4.py compare against and time, and the NumPy mirror below (quant_np, distance_np, tables_np,
pq4_search_np), which the CPU tests check the C oracle against.  `data` is a lancedb_b200.index.IvfPqIndexData with
num_bits = 4.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle

f32 = np.float32


def _index(data):
    """(orc_index, arrays it points into)"""
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
    lib = oracle.load()
    t = np.asarray(t, f32)
    return np.array([lib.orc_pq4_quant(float(v), float(qmin), float(qmax)) for v in t.ravel()],
                    np.uint8).reshape(t.shape)


def distance(S, qmin, qmax, m, metric) -> np.ndarray:
    """The C oracle's orc_pq4_distance, element-wise."""
    lib = oracle.load()
    S = np.asarray(S, np.uint32)
    return np.array([lib.orc_pq4_distance(int(s), float(qmin), float(qmax), int(m), oracle.METRICS[metric])
                     for s in S.ravel()], f32).reshape(S.shape)


def tables(data, qn, part):
    """(Q [m, 16] u8, qmin, qmax) of one probe slot from the C oracle; qn normalised for cosine."""
    ix, keep = _index(data)
    q = np.ascontiguousarray(qn, f32)
    Q = np.empty((data.m, 16), np.uint8)
    qmm = np.empty(2, f32)
    oracle.load().orc_pq4_tables(C.byref(ix), q.ctypes.data, int(part), Q.ctypes.data, qmm.ctypes.data)
    return Q, qmm[0], qmm[1]


def partition_distances(data, q, part) -> np.ndarray:
    """d of every row of partition `part` from the C oracle (q: the raw query)."""
    ix, keep = _index(data)
    q = np.ascontiguousarray(q, f32)
    n = int(data.part_offsets[part + 1] - data.part_offsets[part])
    out = np.empty(max(n, 1), f32)
    oracle.load().orc_pq4_partition_distances(C.byref(ix), q.ctypes.data, int(part), out.ctypes.data)
    return out[:n]


def search(data, queries, k: int, nprobes: int, refine_factor: int = 0, lower=None, upper=None, allow=None,
           max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    q = np.ascontiguousarray(queries, f32).reshape(-1, data.dim)
    ix, keep = _index(data)
    return oracle.search_call("orc_pq4_search", (C.byref(ix), q.ctypes.data), q.shape[0], k, nthreads, nprobes,
                              refine_factor, lower, upper, allow, max_nprobes=max_nprobes)


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
    """The mirror of orc_pq4_search (the search loop, find_partitions and the refine distances from
    oracle/oracle_np.py)."""
    from oracle import oracle_np as onp
    q = np.asarray(queries, f32).reshape(-1, data.dim)
    qn = [onp.query(data.metric, x) for x in q]
    return onp.ivf_search_np(len(q), data, k, nprobes, lambda b: onp.coarse(data.metric, qn[b], data.centroids),
                             lambda b, p: partition_distances_np(data, qn[b], p),
                             None if data.vectors is None else lambda b, r: onp.distance(data.metric, q[b],
                                                                                         data.vectors[r]),
                             refine_factor, lower, upper, allow, max_nprobes)

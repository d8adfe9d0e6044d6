"""NumPy mirror of oracle.c (small cases only) -- an independent second statement of
the same arithmetic, used by tests to cross-check the C oracle.

TEST INFRASTRUCTURE ONLY (never imported by lancedb_b200).  Every operation is an
explicit float32 op so the order of roundings is exactly the one oracle.c states;
see oracle.c for the reference citations of each function.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def l2(x, y):
    """l2_scalar::<f32,f32,16> [lance, recalled]"""
    x = np.asarray(x, f32); y = np.asarray(y, f32)
    d = x.size; nch = d // 16
    s = f32(0)
    for i in range(nch * 16, d):
        diff = f32(x[i] - y[i]); s = f32(s + f32(diff * diff))
    sums = np.zeros(16, f32)
    for c in range(nch):
        diff = (x[c * 16:(c + 1) * 16] - y[c * 16:(c + 1) * 16]).astype(f32)
        sums = (sums + (diff * diff).astype(f32)).astype(f32)
    t = f32(0)
    for l in range(16):
        t = f32(t + sums[l])
    return f32(s + t)


def dot(x, y):
    x = np.asarray(x, f32); y = np.asarray(y, f32)
    d = x.size; nch = d // 16
    s = f32(0)
    for i in range(nch * 16, d):
        s = f32(s + f32(x[i] * y[i]))
    sums = np.zeros(16, f32)
    for c in range(nch):
        sums = (sums + (x[c * 16:(c + 1) * 16] * y[c * 16:(c + 1) * 16]).astype(f32)).astype(f32)
    t = f32(0)
    for l in range(16):
        t = f32(t + sums[l])
    return f32(s + t)


def cosine(x, y):
    xn = np.sqrt(dot(x, x)).astype(f32)
    yy = dot(y, y)
    return f32(f32(1) - f32(f32(dot(x, y) / xn) / np.sqrt(yy).astype(f32)))


def normalize(x):
    x = np.asarray(x, f32)
    return (x / np.sqrt(dot(x, x)).astype(f32)).astype(f32)


def l2_subvec_batch(sub, cb):
    """l2_once::<f32x8,8> reduce tree for dsub == 8; cb: [256, dsub] -> [256]"""
    sub = np.asarray(sub, f32); cb = np.asarray(cb, f32)
    dsub = sub.size
    if dsub == 8 or dsub == 16:
        d = (sub[None, :] - cb).astype(f32)
        s = (d * d).astype(f32)
        if dsub == 16:
            s = (s[:, :8] + s[:, 8:]).astype(f32)
        t = (s[:, :4] + s[:, 4:]).astype(f32)          # s0+s4, s1+s5, s2+s6, s3+s7
        u0 = (t[:, 0] + t[:, 2]).astype(f32)
        u1 = (t[:, 1] + t[:, 3]).astype(f32)
        return (u0 + u1).astype(f32)
    return np.array([l2(sub, c) for c in cb], f32)


def build_lut(codebook, rq, metric):
    m, _, dsub = codebook.shape
    lut = np.empty((m, 256), f32)
    for i in range(m):
        sub = rq[i * dsub:(i + 1) * dsub]
        if metric == "dot":
            lut[i] = [f32(f32(1) - dot(sub, c)) for c in codebook[i]]
        else:
            lut[i] = l2_subvec_batch(sub, codebook[i])
    return lut


def pq_scan(lut, codes_t):
    """codes_t: [m, n] -> sequential f32 accumulate over sub-vectors"""
    m, n = codes_t.shape
    acc = np.zeros(n, f32)
    for i in range(m):
        acc = (acc + lut[i][codes_t[i]]).astype(f32)
    return acc


def ivf_assign(ix, v):
    """find_partitions(row, nprobes = 1) per row"""
    out = np.empty(len(v), np.uint32)
    for r, x in enumerate(np.asarray(v, f32)):
        qn = normalize(x) if ix.metric == "cosine" else x
        if ix.metric == "dot":
            cd = np.array([f32(f32(1) - dot(qn, c)) for c in ix.centroids], f32)
        else:
            cd = np.array([l2(qn, c) for c in ix.centroids], f32)
        out[r] = np.lexsort((np.arange(ix.nlist), cd))[0]
    return out


def pq_encode(ix, v, parts):
    """ProductQuantizer::transform [lance, recalled]: first minimum of each distance-table row"""
    dsub = ix.dim // ix.m
    out = np.empty((len(v), ix.m), np.uint8)
    for r, x in enumerate(np.asarray(v, f32)):
        qn = normalize(x) if ix.metric == "cosine" else x
        rq = qn if ix.metric == "dot" else (qn - ix.centroids[parts[r]]).astype(f32)
        out[r] = build_lut(ix.codebook, rq, ix.metric).argmin(axis=1)
    return out


def distance(metric, x, y):
    """orc_distance_f32: the exact distance refine re-ranks by"""
    if metric == "cosine":
        return cosine(x, y)
    return f32(f32(1) - dot(x, y)) if metric == "dot" else l2(x, y)


def query(metric, q):
    """the query the coarse step and the tables see: normalised for cosine"""
    q = np.asarray(q, f32)
    return normalize(q) if metric == "cosine" else q


def coarse(metric, qn, centroids):
    """find_partitions' distances: 1 - x.y for dot, l2 otherwise (cosine: on the normalised query)"""
    if metric == "dot":
        return np.array([f32(f32(1) - dot(qn, c)) for c in centroids], f32)
    return np.array([l2(qn, c) for c in centroids], f32)


def ivf_search_np(B, data, k, nprobes, coarse_of, partition_of, refine_of=None, refine_factor=0, lower=None,
                  upper=None, allow=None, max_nprobes=0):
    """The IVF search every index kind shares (DESIGN.md section 0), the mirror of orc_ivf_search.  data: nlist,
    part_offsets, row_ids.  Per query b: coarse_of(b) -> the [nlist] coarse distances (a NaN one is never probed);
    partition_of(b, p) -> the distances of partition p's rows; refine_of(b, pos) -> the exact distance of row pos
    (None: no refine).  allow: bool mask over row ids.  Returns (ids [B, k] u64, dist [B, k] f32, count [B] u32)."""
    nlist = data.nlist
    off = np.asarray(data.part_offsets, np.int64)
    rid = np.asarray(data.row_ids, np.uint64)
    keep = np.ones(rid.size, bool)
    if allow is not None:                               # ids beyond the mask are excluded
        a = np.asarray(allow, bool)
        inside = rid < a.size
        keep = np.zeros(rid.size, bool)
        keep[inside] = a[rid[inside].astype(np.int64)]
    nprobes = min(nprobes, nlist)
    np_max = max(nprobes, min(max_nprobes, nlist)) if allow is not None else nprobes
    kk = k * refine_factor if refine_factor else k
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, f32)
    cnt = np.zeros(B, np.uint32)
    for b in range(B):
        cd = np.asarray(coarse_of(b))
        order = np.lexsort((np.arange(nlist), cd))     # ties by partition id, NaN last
        for np_use in (nprobes, np_max):                # maximum_nprobes: again, wider, when fewer than k rows remain
            pos, ds = [np.zeros(0, np.int64)], [np.zeros(0, f32)]
            for p in order[:np_use]:
                if np.isnan(cd[p]) or off[p] == off[p + 1]:
                    continue
                d = np.asarray(partition_of(b, p), f32)
                m = keep[off[p]:off[p + 1]] & ~np.isnan(d)            # _distance IS NOT NULL
                if lower is not None:
                    m &= d >= f32(lower)
                if upper is not None:
                    m &= d < f32(upper)
                pos.append(np.arange(off[p], off[p + 1])[m])
                ds.append(d[m])
            pos, d = np.concatenate(pos), np.concatenate(ds)
            if len(pos) >= k:
                break
        o = np.lexsort((rid[pos], d))[:kk]              # (_distance, _rowid)
        pos, d = pos[o], d[o]
        if refine_factor and refine_of is not None:
            d = np.array([refine_of(b, r) for r in pos], f32)
            pos, d = pos[~np.isnan(d)], d[~np.isnan(d)]               # a NaN distance is never returned
            o = np.lexsort((rid[pos], d))
            pos, d = pos[o], d[o]
        n = min(k, len(pos))
        ids[b, :n] = rid[pos[:n]]
        dist[b, :n] = d[:n]
        cnt[b] = n
    return ids, dist, cnt


def partition_distances(ix, qn, p):
    """the 8-bit IVF_PQ distances of partition p's rows: table sums, then cosine L2^2 / 2 or dot sum - (m - 1)"""
    a, b = int(ix.part_offsets[p]), int(ix.part_offsets[p + 1])
    rq = qn if ix.metric == "dot" else (qn - ix.centroids[p]).astype(f32)
    d = pq_scan(build_lut(ix.codebook, rq, ix.metric), ix.codes_t[a * ix.m:b * ix.m].reshape(ix.m, b - a))
    if ix.metric == "cosine":
        return (d * f32(0.5)).astype(f32)
    return (d - f32(ix.m - 1)).astype(f32) if ix.metric == "dot" else d


def ivfpq_search_one(ix, q, k, nprobes, lower=None, upper=None, allowed=None):
    """ix: lancedb_b200.index.IvfPqIndexData; returns (ids, dists) sorted by (dist, id).
    allowed: optional set of row ids (prefilter: other rows are dropped before the top-k)"""
    qn = query(ix.metric, q)
    allow = None
    if allowed is not None:
        allow = np.zeros(int(ix.row_ids.max(initial=0)) + 1, bool)
        allow[[r for r in allowed if r < allow.size]] = True
    ids, dist, cnt = ivf_search_np(1, ix, k, nprobes, lambda b: coarse(ix.metric, qn, ix.centroids),
                                   lambda b, p: partition_distances(ix, qn, p), lower=lower, upper=upper, allow=allow)
    return ids[0, :cnt[0]], dist[0, :cnt[0]]

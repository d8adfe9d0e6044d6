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


def ivfpq_search_one(ix, q, k, nprobes, lower=None, upper=None, allowed=None):
    """ix: lancedb_b200.index.IvfPqIndexData; returns (ids, dists) sorted by (dist, id).
    allowed: optional set of row ids (prefilter: other rows are dropped before the top-k)"""
    q = np.asarray(q, f32)
    qn = normalize(q) if ix.metric == "cosine" else q
    if ix.metric == "dot":
        cd = np.array([f32(f32(1) - dot(qn, c)) for c in ix.centroids], f32)
    else:
        cd = np.array([l2(qn, c) for c in ix.centroids], f32)
    order = np.lexsort((np.arange(ix.nlist), cd))[:min(nprobes, ix.nlist)]     # NaN last
    cands = []
    for p in order:
        if np.isnan(cd[p]):                 # a NaN coarse distance is never probed
            continue
        a, b = int(ix.part_offsets[p]), int(ix.part_offsets[p + 1])
        if a == b:
            continue
        rq = qn if ix.metric == "dot" else (qn - ix.centroids[p]).astype(f32)
        lut = build_lut(ix.codebook, rq, ix.metric)
        codes_t = ix.codes_t[a * ix.m:b * ix.m].reshape(ix.m, b - a)
        d = pq_scan(lut, codes_t)
        if ix.metric == "cosine":
            d = (d * f32(0.5)).astype(f32)
        elif ix.metric == "dot":
            d = (d - f32(ix.m - 1)).astype(f32)
        for r in range(b - a):
            if np.isnan(d[r]):                  # _distance IS NOT NULL
                continue
            if lower is not None and not d[r] >= f32(lower):
                continue
            if upper is not None and not d[r] < f32(upper):
                continue
            if allowed is not None and int(ix.row_ids[a + r]) not in allowed:
                continue
            cands.append((d[r], int(ix.row_ids[a + r])))
    cands.sort()
    cands = cands[:k]
    return np.array([c[1] for c in cands], np.uint64), np.array([c[0] for c in cands], f32)

"""CPU oracle of IVF_HNSW_SQ search: the C ABI's lgpu_ivf_hnsw_sq_open + lgpu_search semantics.

Per query: IVF_SQ's preparation and coarse step (tests/sq_oracle.py), then in every probed partition the graph search
stated in tests/hnsw_sq_oracle.c [lance, recalled]: a greedy descent through the upper levels, the level-0 loop over W
(the ef' = max(ef, kk) best rows seen, ef = 0 meaning ceil(1.5 k)), and the partition's result R, the kk best
evaluated rows that pass the row filter, ordered by (distance, position).  The driver merges the R lists by
(_distance, _rowid); refine, distance_range and maximum_nprobes are IVF_SQ's.

Two statements of it: the threaded C oracle (hnsw_sq_oracle.c, compiled here against oracle/'s library and run by its
IVF search driver), which the GPU tests and scripts/bench_ivf_hnsw_sq.py compare against and time, and the NumPy mirror
below (level0_np, search_np), which the CPU tests check the C oracle against.  `data` is a
lancedb_b200.index.IvfHnswSqIndexData.
"""
from __future__ import annotations

import ctypes as C
import heapq
import math
import os
import subprocess

import numpy as np

import oracle
from oracle import oracle_np as onp
from tests.sq_oracle import sq_encode_np

f32 = np.float32
NONE = 0xFFFFFFFF

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "hnsw_sq_oracle.c")
_lib = None


def _load():
    """liboracle.so (oracle.load) plus this kind, compiled with the oracle's flags into oracle/_build/."""
    global _lib
    if _lib is not None:
        return _lib
    base = oracle.build()
    oracle.load()
    out = os.path.join(os.path.dirname(base), "libhnsw_sq_oracle.so")
    tmp = f"{out}.{os.getpid()}.tmp"
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(_SRC), os.path.getmtime(base)):
        subprocess.run(["gcc", "-O3", "-mavx2", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                        "-Wextra", "-std=c11", "-shared", "-o", tmp, _SRC, "-L", os.path.dirname(base),
                        "-loracle", "-Wl,-rpath,$ORIGIN", "-lm"], check=True)
        os.replace(tmp, out)                              # atomic: concurrent test processes never see a partial file
    lib = C.CDLL(out)
    vp = C.c_void_p
    lib.orc_hnsw_sq_search.restype = C.c_int
    lib.orc_hnsw_sq_search.argtypes = [C.POINTER(oracle._Index), vp, C.c_double, C.c_double, C.c_uint32, vp, vp, vp,
                                       vp, vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(oracle._Params), vp, vp, vp,
                                       C.c_int]
    oracle.load().orc_hnsw_sq_search = lib.orc_hnsw_sq_search     # so that oracle.search_call finds it
    _lib = lib
    return lib


def ef_prime(k: int, ef: int, refine_factor: int = 0) -> int:
    kk = k * refine_factor if refine_factor else k
    return max(ef if ef else math.ceil(1.5 * k), kk)


def search(data, queries, k: int, nprobes: int, ef: int = 0, refine_factor: int = 0, lower=None, upper=None,
           allow=None, max_nprobes: int = 0, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    sq = data.sq
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, sq.dim)
    keep = [np.ascontiguousarray(sq.centroids, np.float32), np.ascontiguousarray(sq.part_offsets, np.uint64),
            np.ascontiguousarray(sq.row_ids, np.uint64),
            None if sq.vectors is None else np.ascontiguousarray(sq.vectors, np.float32),
            np.ascontiguousarray(sq.codes, np.uint8)]
    g = [np.ascontiguousarray(a) for a in (data.levels, data.adj0, data.upper_index, data.upper_adj, data.entry,
                                           data.top_level)]
    ix = oracle._Index(sq.dim, sq.nlist, 0, oracle.METRICS[sq.metric], sq.nrows, keep[0].ctypes.data, None,
                       keep[1].ctypes.data, None, keep[2].ctypes.data, None if keep[3] is None else keep[3].ctypes.data)
    _load()
    return oracle.search_call("orc_hnsw_sq_search",
                              (C.byref(ix), keep[4].ctypes.data, float(sq.lo), float(sq.hi), int(data.m),
                               *[a.ctypes.data for a in g], int(ef), q.ctypes.data), q.shape[0], k, nthreads,
                              nprobes, refine_factor, lower, upper, allow, max_nprobes=max_nprobes)


# ---- NumPy mirror ----


def descend_np(dist, upper_index_p, upper_adj, levels_p, entry: int, top: int, m: int) -> int:
    """The upper-level descent from `entry`: the start row of level 0.  dist(pos) -> f32."""
    cur, dc = int(entry), dist(int(entry))
    for L in range(top, 0, -1):
        while True:
            nb = upper_adj[int(upper_index_p[cur]) + L - 1]
            best, bd = cur, dc
            for v in (int(x) for x in nb if x != NONE):
                d = dist(v)
                if (d, v) < (bd, best):
                    best, bd = v, d
            if best == cur:
                break
            cur, dc = best, bd
    return cur


def level0_np(dist, adj0_p, start: int, efp: int, rng=None, forget=None):
    """The level-0 list loop.  Returns {pos: distance} of every evaluated row.  rng: offer each expanded row's
    neighbours to W in a shuffled order; forget(pos) -> True: the visited check misses pos (a lossy cache), so it is
    evaluated and offered again."""
    ev = {start: dist(start)}
    W = [(ev[start], start, False)]                       # sorted by (d, pos), with the expanded flag
    while True:
        c = next((i for i, w in enumerate(W) if not w[2]), None)
        if c is None:
            break
        W[c] = (W[c][0], W[c][1], True)
        nbs = [int(v) for v in adj0_p[W[c][1]] if v != NONE]
        if rng is not None:
            rng.shuffle(nbs)
        for v in nbs:
            if v in ev and not (forget and forget(v)):
                continue
            ev[v] = d = dist(v)
            if any(w[1] == v for w in W):                 # W rejects a duplicate
                continue
            if len(W) == efp and not (d, v) < W[-1][:2]:
                continue
            W.append((d, v, False))
            W.sort(key=lambda w: w[:2])
            del W[efp:]
    return ev


def two_heap_np(dist, adj0_p, start: int, efp: int):
    """The usual two-heap form: pop the nearest candidate, stop when it is farther than W's farthest.  Returns the
    evaluated rows as level0_np does."""
    ev = {start: dist(start)}
    cand = [(ev[start], start)]
    W = [(-ev[start], -start)]                            # max-heap of (d, pos)
    while cand:
        d, c = heapq.heappop(cand)
        if (d, c) > (-W[0][0], -W[0][1]):
            break
        for v in (int(x) for x in adj0_p[c] if x != NONE):
            if v in ev:
                continue
            ev[v] = dv = dist(v)
            if len(W) < efp or (dv, v) < (-W[0][0], -W[0][1]):
                heapq.heappush(cand, (dv, v))
                heapq.heappush(W, (-dv, -v))
                if len(W) > efp:
                    heapq.heappop(W)
    return ev


def partition_np(data, p: int, qc, efp: int, kk: int, keep, **loop):
    """The distances of partition p's rows for query codes qc: R's rows carry their distance, every other row NaN.
    keep(pos, d) -> bool is the row filter."""
    off = data.part_offsets.astype(np.int64)
    a, b = off[p], off[p + 1]
    codes = data.sq.codes[a:b].astype(np.int64)
    q = np.asarray(qc, np.int64)
    dist = lambda r: f32(int(((codes[r] - q) ** 2).sum()))
    start = descend_np(dist, data.upper_index[a:b], data.upper_adj, data.levels[a:b], int(data.entry[p]),
                       int(data.top_level[p]), data.m)
    ev = level0_np(dist, data.adj0[a:b], start, efp, **loop)
    r = sorted((d, v) for v, d in ev.items() if keep(a + v, d))[:kk]
    out = np.full(b - a, np.nan, f32)
    for d, v in r:
        out[v] = d
    return out


def search_np(data, queries, k: int, nprobes: int, ef: int = 0, refine_factor: int = 0, lower=None, upper=None,
              allow=None, max_nprobes: int = 0):
    """The mirror of orc_hnsw_sq_search (the search loop, find_partitions and the refine distances from
    oracle/oracle_np.py)."""
    sq = data.sq
    q = np.asarray(queries, f32).reshape(-1, sq.dim)
    qn = [onp.query(sq.metric, x) for x in q]
    qc = [sq_encode_np(x, sq.lo, sq.hi) for x in qn]
    efp = ef_prime(k, ef, refine_factor)
    kk = k * refine_factor if refine_factor else k
    rid = np.asarray(sq.row_ids, np.uint64)
    mask = None if allow is None else np.asarray(allow, bool)

    def keep(pos, d):
        if lower is not None and not d >= f32(lower):
            return False
        if upper is not None and not d < f32(upper):
            return False
        return mask is None or (int(rid[pos]) < mask.size and bool(mask[int(rid[pos])]))

    return onp.ivf_search_np(len(q), sq, k, nprobes, lambda b: onp.coarse(sq.metric, qn[b], sq.centroids),
                             lambda b, p: partition_np(data, p, qc[b], efp, kk, keep),
                             None if sq.vectors is None else lambda b, r: onp.distance(sq.metric, q[b], sq.vectors[r]),
                             refine_factor, lower, upper, allow, max_nprobes)


def complete_graph(sq, m: int | None = None):
    """An IvfHnswSqIndexData over `sq` whose level-0 graph is complete (every row adjacent to every other) and has no
    upper level: with ef' >= the partition size every row is evaluated, so the search returns IVF_SQ's results."""
    from lancedb_b200.index import IvfHnswSqIndexData
    off = sq.part_offsets.astype(np.int64)
    big = int(np.diff(off).max(initial=1))
    m = m or max(1, big // 2)                             # 2m >= big - 1 neighbours
    adj0 = np.full((sq.nrows, 2 * m), NONE, np.uint32)
    for p in range(sq.nlist):
        a, b = off[p], off[p + 1]
        for r in range(b - a):
            nb = [v for v in range(b - a) if v != r]
            adj0[a + r, :len(nb)] = nb
    entry = np.where(np.diff(off) > 0, 0, NONE).astype(np.uint32)
    return IvfHnswSqIndexData(sq, m, np.zeros(sq.nrows, np.uint8), adj0, np.full(sq.nrows, NONE, np.uint32),
                              np.zeros((0, m), np.uint32), entry, np.zeros(sq.nlist, np.uint8))


def random_hnsw_index(rng, n=600, dim=24, nlist=6, metric="l2", m=6, ef_construction=40, with_vectors=True,
                      empty=(1,), seed=45):
    """random_sq_index (empty partitions, duplicate rows, non-contiguous row ids) with HNSW graphs built over its
    codes."""
    from lancedb_b200.index import IvfHnswSqIndexData, build_hnsw_graph
    from tests.sq_oracle import random_sq_index
    sq = random_sq_index(rng, n=n, dim=dim, nlist=nlist, metric=metric, with_vectors=with_vectors, empty=empty,
                         unit_centroids=metric == "cosine")
    data = IvfHnswSqIndexData(sq, m, *build_hnsw_graph(sq.codes, sq.part_offsets, m, ef_construction, seed))
    data.validate()
    return data


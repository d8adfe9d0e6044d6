"""CPU oracle of binary-vector flat search by Hamming distance (the C ABI's lgpu_binary_* semantics).

_distance = popcount(q XOR x) over the row's bytes, as f32; results ascending by (_distance, _rowid); distance_range
[lower, upper); an allow mask over row ids drops rows before the top-k; unused slots are UINT64_MAX / +inf.

Two statements of it: the threaded C oracle (hamming_oracle.c: orc_hamming_u8, orc_flat_search_u8, built into
oracle/'s library), which the GPU tests, smoke() and scripts/bench_binary.py compare against and time, and the NumPy
mirror below (hamming_u8_np, flat_search_u8_np), which the CPU tests check the C oracle against.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor
import os

import numpy as np

import oracle

def hamming_u8(queries, vectors, nthreads: int = 0) -> np.ndarray:
    """[B, N] uint32 Hamming distances of packed uint8 rows (C oracle, `nthreads` threads, 0 = all)."""
    q = np.ascontiguousarray(queries, np.uint8)
    x = np.ascontiguousarray(vectors, np.uint8)
    out = np.empty((q.shape[0], x.shape[0]), np.uint32)
    if out.size:
        if oracle.load().orc_hamming_u8(q.ctypes.data, q.shape[0], x.ctypes.data, x.shape[0], q.shape[1],
                                        out.ctypes.data, oracle.threads(nthreads)) != 0:
            raise MemoryError("orc_hamming_u8 failed")
    return out


def flat_search_u8(vectors, queries, k: int, row_ids=None, lower=None, upper=None, allow=None, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32) from the C oracle; allow: optional bool mask over row ids."""
    x = np.ascontiguousarray(vectors, np.uint8)
    q = np.ascontiguousarray(queries, np.uint8)
    rid = None if row_ids is None else np.ascontiguousarray(row_ids, np.uint64)
    return oracle.search_call("orc_flat_search_u8", (x.ctypes.data, x.shape[0], x.shape[1],
                                                     None if rid is None else rid.ctypes.data, q.ctypes.data),
                              q.shape[0], k, nthreads, lower=lower, upper=upper, allow=allow)


# ---- NumPy mirror ----


def hamming_u8_np(queries, vectors, nthreads: int = 0) -> np.ndarray:
    """[B, N] uint32 Hamming distances of packed uint8 rows (numpy's bitwise_count of the XOR, in row chunks; the
    chunks run on `nthreads` threads, numpy releasing the GIL inside the ufuncs)."""
    q = np.ascontiguousarray(queries, np.uint8)
    x = np.ascontiguousarray(vectors, np.uint8)
    B, nb = q.shape
    N = x.shape[0]
    out = np.empty((B, N), np.uint32)
    if B == 0 or N == 0:
        return out
    step = max(1, (1 << 24) // max(1, B * nb))

    def run(c0):
        xs = x[c0:c0 + step]
        out[:, c0:c0 + len(xs)] = np.bitwise_count(q[:, None, :] ^ xs[None, :, :]).sum(-1, dtype=np.uint32)

    starts = range(0, N, step)
    if nthreads and nthreads > 1:
        with ThreadPoolExecutor(nthreads) as ex:
            list(ex.map(run, starts))
    else:
        for c0 in starts:
            run(c0)
    return out


def hamming_unpackbits(q, x) -> int:
    """One distance, spelled the slow way: np.unpackbits(q ^ x).sum()."""
    return int(np.unpackbits(np.asarray(q, np.uint8) ^ np.asarray(x, np.uint8)).sum())


def flat_search_u8_np(vectors, queries, k: int, row_ids=None, lower=None, upper=None, allow=None, nthreads: int = 0):
    """(ids [B, k] u64, dist [B, k] f32, count [B] u32); allow: optional bool mask over row ids."""
    x = np.ascontiguousarray(vectors, np.uint8)
    q = np.ascontiguousarray(queries, np.uint8)
    N, B = x.shape[0], q.shape[0]
    rid = np.arange(N, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    D = hamming_u8_np(q, x, nthreads or (os.cpu_count() or 1)).astype(np.float32)
    keep = np.ones(N, bool)
    if allow is not None:                     # ids beyond the mask are excluded
        a = np.asarray(allow, bool)
        inside = rid < a.size
        keep = np.zeros(N, bool)
        keep[inside] = a[rid[inside].astype(np.int64)]
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    for b in range(B):
        m = keep.copy()
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

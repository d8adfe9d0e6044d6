"""CPU reference of the GPU index-training kernels (lgpu_kmeans_train, lgpu_pq_train), exact to the bit.

lloyd(x, init, iters) restates lgpu_kmeans_train: max(iters, 1) Lloyd iterations.  Each assigns every row to its nearest
centre with the C oracle's find_partitions(row, nprobes = 1) in L2 (lance's arithmetic, ties to the lowest centre), which
is what the kernels compute.  Each non-empty centre then becomes np.float32(sum / cnt), with the sum taken in f64 over the
cluster's rows in ascending row order, starting from +0.0 as the kernels' accumulators do (so values that are all -0.0
sum to +0.0).  An empty centre keeps its value bit for bit, and a row with no finite distance to any centre (one holding
a NaN or an infinity, which the C ABI refuses) is in no cluster.
pq_lloyd(x, init_cb, iters) restates lgpu_pq_train: codes from the oracle's pq_encode against one all-zero centroid, then
each used codeword becomes the f64 mean of its sub-vectors rounded to f32; unused codewords are kept.

Why a bit-exact comparison with the GPU is legitimate.  km_update_kernel sorts a cluster of at most KM_SORT_MAX = 4096
rows and sums it in ascending row order, as lloyd does, so those centres agree on any data.  A larger cluster, and every
PQ codeword, is summed in whatever order the kernel's threads or atomics run.  For those the tests use dyadic data:
multiples of 2^-10 no larger than 8 in magnitude (`dyadic`).  Every partial sum of fewer than 2^32 such values is a
multiple of 2^-10 below 2^36 in magnitude, so it needs at most 46 significant bits and f64 adds it exactly, in any order.
The sums run over data rows only, never over centres, so this holds at every iteration, not only the first.

KMEANS_CASES and PQ_CASES are the GPU comparisons of tests/test_gpu_train.py; tests/test_train_host.py rehearses them here and checks that
each reaches the kernel branch it names.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor
import math

import numpy as np

import oracle

KM_SORT_MAX = 4096            # kmeans.cu: clusters up to this many rows are summed in ascending row order
KM_MAX_DIM = 4096             # kmeans.cu: KM_THREADS * KM_DPT
KM_THREADS = 256              # kmeans.cu: dims KM_THREADS apart share one thread (slot j = t // 256)
PQ_DSUB = (1, 2, 4, 8, 16, 32)


def assign_chunk_rows(k: int) -> int:
    """Rows per chunk of the assignment (assign_nearest and lgpu_ivf_assign in api.cu): the [rows][ld] distance matrix
    is kept to 2^28 bytes, with ld = k rounded up to a multiple of 4."""
    ld = (k + 3) & ~3
    return max(256, min(65536, (1 << 28) // (ld * 4)))


def tensor_core_assignment(dim: int, k: int) -> bool:
    """assign_nearest takes the tensor-core GEMM (gemm_shape_supported: dim % 8 == 0) when k >= 256"""
    return dim % 8 == 0 and k >= 256


def dyadic(rng, shape) -> np.ndarray:
    """Multiples of 2^-10 in [-8, 8]: every sum of fewer than 2^32 of them is exact in f64, in any order"""
    return (np.clip(np.round(rng.standard_normal(shape) * 2 ** 10) / 2 ** 10, -8, 8)).astype(np.float32)


def _l2_index(c, codebook=None, m=1):
    c = np.ascontiguousarray(c, np.float32)
    k, dim = c.shape
    cb = np.zeros(0, np.float32) if codebook is None else np.ascontiguousarray(codebook, np.float32)
    return oracle.OracleIndex(dim=dim, nlist=k, m=m, metric="l2", centroids=c, codebook=cb,
                              part_offsets=np.zeros(k + 1, np.uint64), codes_t=np.zeros(0, np.uint8),
                              row_ids=np.zeros(0, np.uint64))


def threaded(fn, n: int, nthreads: int = 0, step: int = 2048):
    """fn(r0, r1) over row chunks on a thread pool (the oracle's ctypes calls release the GIL)"""
    starts = range(0, n, step)
    with ThreadPoolExecutor(oracle.threads(nthreads)) as ex:
        list(ex.map(lambda r0: fn(r0, min(n, r0 + step)), starts))


def nearest(x, c, nthreads: int = 0) -> np.ndarray:
    """u32 [n]: the oracle's ivf_assign in L2 (find_partitions(row, 1), ties to the lowest centre)"""
    x = np.ascontiguousarray(x, np.float32)
    ix = _l2_index(c)
    out = np.empty(x.shape[0], np.uint32)

    def run(r0, r1):
        out[r0:r1] = ix.ivf_assign(x[r0:r1])
    threaded(run, x.shape[0], nthreads)
    return out


def _means(x, groups, n_groups, old):
    """old with every non-empty group replaced by np.float32(f64 sum in ascending row order / count); also the counts"""
    out = old.copy()
    order = np.argsort(groups, kind="stable")                 # rows of each group, ascending
    counts = np.bincount(groups, minlength=n_groups)[:n_groups]
    ends = np.cumsum(counts)
    for g in np.nonzero(counts)[0]:
        rows = order[ends[g] - counts[g]:ends[g]]
        # sequential, not np.sum's pairwise order; "+ 0.0": the kernels' sums start from +0.0, so the sum of values
        # that are all -0.0 is +0.0, not -0.0 (in every other case adding +0.0 first or last changes nothing)
        s = np.cumsum(x[rows].astype(np.float64), axis=0)[-1] + 0.0
        out[g] = (s / np.float64(counts[g])).astype(np.float32)
    return out, counts


def lloyd(x, init, iters: int, trace: list | None = None, nthreads: int = 0) -> np.ndarray:
    """lgpu_kmeans_train restated: the trained centres [k, dim] f32.  trace: if given, gets (assignment, counts) of
    every iteration."""
    x = np.ascontiguousarray(x, np.float32)
    c = np.array(init, np.float32, order="C", copy=True)
    k = c.shape[0]
    finite = np.isfinite(x).all(axis=1)
    for _ in range(max(iters, 1)):
        a = nearest(x, c, nthreads).astype(np.int64)
        a[~finite] = k                                         # no finite distance: in no cluster
        c, counts = _means(x, a, k, c)
        if trace is not None:
            trace.append((a, counts))
    return c


def inertia(x, c) -> float:
    """math.fsum of every row's distance to its nearest centre (the oracle's find_partitions(row, 1))"""
    ix = _l2_index(c)
    return math.fsum(float(ix.find_partitions(row, 1)[1][0]) for row in np.asarray(x, np.float32))


def pq_codes(x, cb, nthreads: int = 0) -> np.ndarray:
    """u8 [n, m]: the oracle's pq_encode of the rows against one all-zero centroid (residual = row), ties to the
    lowest code"""
    x = np.ascontiguousarray(x, np.float32)
    m = cb.shape[0]
    ix = _l2_index(np.zeros((1, x.shape[1]), np.float32), cb, m)
    out = np.empty((x.shape[0], m), np.uint8)
    zero = np.zeros(x.shape[0], np.uint32)

    def run(r0, r1):
        out[r0:r1] = ix.pq_encode(x[r0:r1], zero[r0:r1])
    threaded(run, x.shape[0], nthreads, step=512)
    return out


def pq_lloyd(x, init_cb, iters: int, trace: list | None = None, nthreads: int = 0) -> np.ndarray:
    """lgpu_pq_train restated: the trained codebook [m, 256, dsub] f32.  trace: if given, gets the codes of every
    iteration."""
    x = np.ascontiguousarray(x, np.float32)
    cb = np.array(init_cb, np.float32, order="C", copy=True)
    m, _, dsub = cb.shape
    xs = x.reshape(x.shape[0], m, dsub)
    for _ in range(max(iters, 1)):
        codes = pq_codes(x, cb, nthreads)
        for i in range(m):
            cb[i], _ = _means(xs[:, i, :], codes[:, i].astype(np.int64), 256, cb[i])
        if trace is not None:
            trace.append(codes)
    return cb


# ---- the GPU cases ----


def _clustered(rng, n, dim, k=24):
    """n rows around k Gaussian centres (not dyadic: only for clusters of at most KM_SORT_MAX rows)"""
    cen = rng.standard_normal((k, dim)).astype(np.float32) * 3
    return (cen[rng.integers(0, k, n)] + rng.standard_normal((n, dim))).astype(np.float32)


def _rows(rng, x, k):
    return x[rng.choice(len(x), k, replace=False)].copy()


def _case_dim(dim, n):
    def make(rng):
        x = _clustered(rng, n, dim)
        return x, _rows(rng, x, 256), 2
    return make


def _case_k(k):
    def make(rng):
        x = _clustered(rng, 4000, 32)
        return x, _rows(rng, x, k), 3
    return make


def _case_chunks(rng):
    x = dyadic(rng, (40000, 64))
    return x, _rows(rng, x, 2048), 2


def _case_big_clusters(rng):
    x = dyadic(rng, (20000, 16))
    return x, _rows(rng, x, 4), 3


def _case_empty(rng):
    x = _clustered(rng, 3000, 32)
    c = _rows(rng, x, 64)
    c[5] = 1e3
    return x, c, 3


def _case_tie(rng):
    x = _clustered(rng, 3000, 32)
    c = _rows(rng, x, 64)
    c[41] = c[7]
    return x, c, 2


def _case_k_above_n(rng):
    x = _clustered(rng, 100, 32)
    return x, rng.standard_normal((300, 32)).astype(np.float32) * 3, 3


def _case_one_row(rng):
    return rng.standard_normal((1, 24)).astype(np.float32), rng.standard_normal((4, 24)).astype(np.float32), 2


def _case_ragged(rng):
    x = _clustered(rng, 1037, 40)
    return x, _rows(rng, x, 20), 3


def _case_bf16_exact(rng):
    x = (rng.integers(-8, 9, (3000, 64)) / 4).astype(np.float32)   # small integers / 4: exact in bf16, many ties
    return x, _rows(rng, x, 256), 3


def _case_dyadic_fine(rng):
    x = dyadic(rng, (3000, 64))                                   # 2^-10 steps: not exact in bf16's 8-bit mantissa
    return x, _rows(rng, x, 256), 3


def _case_iters0(rng):
    x = _clustered(rng, 2000, 32)
    return x, _rows(rng, x, 50), 0


# name -> (data(rng) -> (x, init, iters), what it reaches).  Claims (checked on the CPU by test_train_host.py):
#   "tc" / "exact": the tensor-core assignment or the exact kernels; "dpt": KM_DPT slots j > 0 (dim > 256);
#   "big": a cluster above KM_SORT_MAX rows; "empty": an empty cluster; "tie": two identical initial centres;
#   "chunks": more rows than one assignment chunk; "scan2": k > 1024 (two counts per km_scan thread);
#   "k>n", "n=1", "ragged": degenerate counts; "bf16": data exact in bf16; "iters0": iters = 0 runs one iteration.
KMEANS_CASES = {
    "dim8": (_case_dim(8, 3000), {"tc"}),
    "dim64": (_case_dim(64, 3000), {"tc"}),
    "dim100": (_case_dim(100, 3000), {"exact"}),
    "dim260": (_case_dim(260, 3000), {"exact", "dpt"}),
    "dim768": (_case_dim(768, 2000), {"tc", "dpt"}),
    "dim4096": (_case_dim(4096, 1200), {"tc", "dpt"}),
    "k1": (_case_k(1), {"exact"}),
    "k2": (_case_k(2), {"exact"}),
    "k255": (_case_k(255), {"exact"}),
    "k256": (_case_k(256), {"tc"}),
    "k300": (_case_k(300), {"tc"}),
    "k2048": (_case_k(2048), {"tc", "scan2"}),
    "chunks": (_case_chunks, {"tc", "chunks", "scan2"}),
    "big_clusters": (_case_big_clusters, {"exact", "big"}),
    "empty": (_case_empty, {"empty"}),
    "tie": (_case_tie, {"tie", "empty"}),
    "k_above_n": (_case_k_above_n, {"tc", "k>n", "empty"}),
    "one_row": (_case_one_row, {"n=1", "k>n", "empty"}),
    "ragged": (_case_ragged, {"ragged", "empty"}),
    "bf16_exact": (_case_bf16_exact, {"tc", "bf16"}),
    "dyadic_fine": (_case_dyadic_fine, {"tc"}),
    "iters0": (_case_iters0, {"iters0"}),
}


def kmeans_case(name):
    """(x, init, iters) of a KMEANS_CASES entry, from its own seed"""
    return KMEANS_CASES[name][0](np.random.default_rng([71, *name.encode()]))


def _pq_init(rng, x, m, n_init=256):
    rows = x[rng.choice(len(x), n_init, replace=n_init > len(x))]
    return np.ascontiguousarray(rows.reshape(n_init, m, -1).transpose(1, 0, 2))


def _case_pq(dim, m, n):
    def make(rng):
        x = dyadic(rng, (n, dim))
        return x, _pq_init(rng, x, m), 2, m
    return make


def _case_pq_unused(rng):
    x = dyadic(rng, (150, 64))
    return x, dyadic(rng, (16, 256, 4)), 3, 16


def _case_pq_tie(rng):
    x = dyadic(rng, (2000, 64))
    cb = _pq_init(rng, x, 8)
    cb[:, 200] = cb[:, 9]
    return x, cb, 1, 8


# name -> data(rng) -> (x, init codebook [m, 256, dsub], iters, m); dyadic data throughout
PQ_CASES = {
    "d32m32": _case_pq(32, 32, 3000),      # dsub 1
    "d64m32": _case_pq(64, 32, 3000),      # dsub 2
    "d64m16": _case_pq(64, 16, 3000),      # dsub 4
    "d768m96": _case_pq(768, 96, 1500),    # dsub 8
    "d48m3": _case_pq(48, 3, 3000),        # dsub 16
    "d96m3": _case_pq(96, 3, 3000),        # dsub 32
    "d32m1": _case_pq(32, 1, 3000),        # dsub 32, one sub-space
    "unused": _case_pq_unused,             # n < 256: unused codewords kept
    "tie": _case_pq_tie,                   # codeword 200 = codeword 9: the tie goes to 9
}


def pq_case(name):
    return PQ_CASES[name](np.random.default_rng([72, *name.encode()]))

"""Every search kind at high dimensions and wide codes, up to the limit each kind declares: one case table, each case
compared with its kind's C oracle bit for bit (ids, counts, distance bits), and the route each case claims proven with
the library's counters (lgpu_last_filter_stats, lgpu_last_scanned_code_bytes, lgpu_kernel_launch_count).  The
width-dependent switches -- the small path's shared-memory bytes, the filter scan's m <= 512, the tensor-core shapes,
the multivector host re-score's 4096-byte slots, the IVF host refine's chunks -- each get a case on either side.
tests/test_wide_host.py restates every route predicate and checks that each case lands where it says, without a GPU.

Then the tensor-core and integer debug kernels at the same widths against float64 or integer NumPy."""
from dataclasses import dataclass, field

import numpy as np
import pytest

import oracle
from lancedb_b200 import _native
from lancedb_b200.index import IvfSqIndexData
from tests import hnsw_sq_oracle, ivf_binary_oracle, pq4_oracle, rq_oracle, sq_oracle
from tests.hamming_oracle import flat_search_u8
from tests.hnsw_sq_oracle import random_hnsw_index
from tests.multivec_oracle import flat_search_mv, offsets_of
from tests.pq4_oracle import random_pq4_index
from tests.rq_oracle import random_rq_index
from tests.sq_oracle import random_sq_index
from tests.util import assert_same, bf16, random_index, same_result, split_support_case, tc_band

f32 = np.float32
NT = 16                                         # oracle threads


@dataclass(frozen=True)
class Case:
    """kind: flat, pq8, pq4, sq, hnsw_sq, rq, multivec, binary, ivf_binary.  w: the widths (dim, m, nbytes, dtype,
    metrics, placement), N rows (multivec: stored vectors), B queries, k, env: environment of the open and the search,
    route: the route the case claims (test_wide_host.py derives it from the shape)."""
    kind: str
    w: dict
    N: int
    B: int
    k: int
    route: str
    env: dict = field(default_factory=dict)


SMALL = {"LGPU_SMALL_SLOTS": "1024"}               # the library's default for the small path
_FLAT = {}
for _dt in ("f32", "f16"):
    for _d in (3072, 4096):
        _FLAT[f"flat_{_dt}_simt_{_d}"] = Case("flat", dict(dim=_d, dtype=_dt, metrics=("l2", "cosine", "dot")),
                                              2000, 5, 10, "simt")
        _FLAT[f"flat_{_dt}_tc_dense_{_d}"] = Case("flat", dict(dim=_d, dtype=_dt, metrics=("l2",)), 4096, 16, 10,
                                                  "tc_dense")
    _FLAT[f"flat_{_dt}_tc_sampled_2056"] = Case("flat", dict(dim=2056, dtype=_dt, metrics=("l2",)), 262144, 8, 10,
                                                "tc_sampled")
    _FLAT[f"flat_{_dt}_exact_4099"] = Case("flat", dict(dim=4099, dtype=_dt, metrics=("l2", "cosine", "dot")), 5000, 16,
                                           10, "simt")

CASES = {
    **_FLAT,
    # 8-bit IVF_PQ: the small path's (256 m + dim) 4 <= 200 KiB, the filter scan's m <= 512, dsub 32 (codebook from L2)
    # (the suite turns the small path off, tests/conftest.py: these four turn it back on)
    "pq8_small_m192_d1536": Case("pq8", dict(dim=1536, m=192, nlist=16), 6000, 2, 10, "small", SMALL),
    "pq8_filter_m192_d3072": Case("pq8", dict(dim=3072, m=192, nlist=16), 6000, 2, 10, "filter", SMALL),
    "pq8_small_m199_d199": Case("pq8", dict(dim=199, m=199, nlist=16), 6000, 2, 10, "small", SMALL),
    "pq8_filter_m200_d200": Case("pq8", dict(dim=200, m=200, nlist=16), 6000, 2, 10, "filter", SMALL),
    "pq8_filter_m512_d4096": Case("pq8", dict(dim=4096, m=512, nlist=32), 8000, 16, 10, "filter"),
    "pq8_exact_m1024_d4096": Case("pq8", dict(dim=4096, m=1024, nlist=32), 8000, 16, 10, "exact"),
    "pq8_filter_m512_d16384": Case("pq8", dict(dim=16384, m=512, nlist=8), 3000, 16, 10, "filter"),
    "pq8_exact_m1024_d32768": Case("pq8", dict(dim=32768, m=1024, nlist=8), 2000, 8, 10, "exact"),
    "pq8_exact_m2048_d32768": Case("pq8", dict(dim=32768, m=2048, nlist=8), 2000, 8, 10, "exact"),
    "pq8_refine_hbm_d4096": Case("pq8", dict(dim=4096, m=512, nlist=32, refine=4), 6000, 16, 10, "filter"),
    "pq8_refine_host_d4096": Case("pq8", dict(dim=4096, m=512, nlist=32, refine=4), 6000, 16, 10, "filter",
                                  {"LGPU_VECTORS_HBM_BYTES": "0"}),
    "pq4_m256_d8192": Case("pq4", dict(dim=8192, m=256, nlist=16), 6000, 16, 10, "pq4"),
    "sq_d4096": Case("sq", dict(dim=4096, nlist=16), 6000, 16, 10, "sq"),
    "sq_d65536_extreme": Case("sq", dict(dim=65536, nlist=2, extreme=True), 300, 3, 300, "sq"),
    "hnsw_sq_d4096": Case("hnsw_sq", dict(dim=4096, nlist=4), 1500, 8, 10, "hnsw"),
    "rq_l2_d4096": Case("rq", dict(dim=4096, nlist=16, metric="l2"), 4000, 16, 10, "rq"),
    "rq_cosine_d4096": Case("rq", dict(dim=4096, nlist=16, metric="cosine"), 4000, 16, 10, "rq"),
    "binary_simt_4096": Case("binary", dict(nbytes=4096), 3000, 9, 10, "simt"),
    "binary_simt_4100": Case("binary", dict(nbytes=4100), 3000, 9, 10, "simt"),
    "binary_tc_dense_4096": Case("binary", dict(nbytes=4096), 4096, 128, 10, "tc_dense"),
    "binary_tc_dense_4100": Case("binary", dict(nbytes=4100), 4096, 128, 10, "tc_dense"),
    "binary_list_4096": Case("binary", dict(nbytes=4096), 70000, 5, 10, "list"),
    "binary_list_4100": Case("binary", dict(nbytes=4100), 70000, 5, 10, "list"),
    "binary_2mib": Case("binary", dict(nbytes=1 << 21, extreme=True), 6, 3, 6, "simt"),
    "ivf_binary_4096": Case("ivf_binary", dict(nbytes=4096, nlist=16), 4000, 16, 10, "ivf_ham"),
    "ivf_binary_4100": Case("ivf_binary", dict(nbytes=4100, nlist=16), 4000, 16, 10, "ivf_ham"),
    "ivf_binary_2mib": Case("ivf_binary", dict(nbytes=1 << 21, nlist=2, extreme=True), 6, 3, 6, "ivf_ham"),
}
for _dt in ("f32", "f16"):
    for _pl in ("hbm", "host"):
        env = {"LGPU_MULTIVEC_HBM_BYTES": "0"} if _pl == "host" else {}
        for _d in (2048, 4096):
            CASES[f"multivec_{_dt}_{_pl}_exact_{_d}"] = Case("multivec", dict(dim=_d, dtype=_dt), 3000, 3, 10, "exact",
                                                             env)
            CASES[f"multivec_{_dt}_{_pl}_tc_{_d}"] = Case("multivec", dict(dim=_d, dtype=_dt), 65536, 3, 10, "tc", env)
        CASES[f"multivec_{_dt}_{_pl}_exact_2049"] = Case("multivec", dict(dim=2049, dtype=_dt), 65536, 3, 10, "exact",
                                                         env)

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def _profiled(fn):
    """(fn(), filter stats, scanned code bytes) of one profiled call"""
    _native.set_profiling(True)
    try:
        out = fn()
        return out, _native.last_filter_stats(), _native.last_scanned_code_bytes()
    finally:
        _native.set_profiling(False)


def _launches(fn):
    n0 = _native.kernel_launch_count()
    out = fn()
    return out, _native.kernel_launch_count() - n0


# ---- flat ----
def _flat_rows(dim, N):
    def make():
        rng = np.random.default_rng(dim * 7 + N)
        x = rng.standard_normal((N, dim), dtype=f32)
        x[N // 2] = x[3]                                  # a duplicate: a tie ordered by row id
        q = rng.standard_normal((16, dim), dtype=f32)
        q[0] = x[3]
        return x, q
    return _cached(("flat", dim, N), make)


def _run_flat(c, monkeypatch):
    dim, B = c.w["dim"], c.B
    x, q = _flat_rows(dim, c.N)
    q = q[:B]
    rows = x.astype(np.float16) if c.w["dtype"] == "f16" else x
    ref = rows.astype(f32) if c.w["dtype"] == "f16" else rows
    fl = _native.GpuFlat(rows)
    try:
        for metric in c.w["metrics"]:
            (got, st, _) = _profiled(lambda: fl.search(q, k=c.k, metric=metric))
            assert_same(got, oracle.flat_search(ref, q, k=c.k, metric=metric, nthreads=NT), f"{metric}")
            route = "simt" if st["rescored"] == 0 else ("tc_sampled" if c.N >= 262144 else "tc_dense")
            assert route == c.route, (metric, route, st)
            if route == "tc_sampled":
                # the same search on the dense shortlist: another launch sequence, the same bits
                again, n_sampled = _launches(lambda: fl.search(q, k=c.k, metric=metric))
                monkeypatch.setenv("LGPU_FLAT_DENSE", "1")
                dense, n_dense = _launches(lambda: fl.search(q, k=c.k, metric=metric))
                monkeypatch.delenv("LGPU_FLAT_DENSE")
                assert n_sampled != n_dense, "the sampled route ran the dense route's launches"
                assert same_result(again, got) and same_result(dense, got)
    finally:
        fl.close()


# ---- 8-bit IVF_PQ ----
def _run_pq8(c, monkeypatch):
    w = c.w
    refine = w.get("refine", 0)
    rng = np.random.default_rng(w["dim"] + w["m"] + c.N)
    ix = random_index(rng, dim=w["dim"], nlist=w["nlist"], m=w["m"], n=c.N, with_vectors=bool(refine))
    q = rng.standard_normal((c.B, w["dim"]), dtype=f32)
    if refine:
        q[0] = ix.vectors[11]
    kw = dict(k=c.k, nprobes=4, refine_factor=refine)
    gpu = _native.GpuIvfPq(ix)
    try:
        if "LGPU_VECTORS_HBM_BYTES" in c.env:
            assert gpu.vectors_on_host
        elif refine:
            assert not gpu.vectors_on_host
        got, st, scanned = _profiled(lambda: gpu.search(q, **kw))
    finally:
        gpu.close()
    assert_same(got, oracle.OracleIndex.from_data(ix).search(q, nthreads=NT, **kw), "pq8")
    route = "filter" if st["queries"] == c.B else ("small" if scanned == 0 else "exact")
    assert route == c.route, (route, st, scanned)


# ---- the other IVF kinds ----
def _sq_extreme(N, dim, nlist):
    """Rows of codes 0 and queries of codes 255 in every component: l2 distances up to dim x 255^2 (4,261,478,400 at
    dim 65536, above 2^31).  Row r < 8 moves r components to code 1, so its distance is 255^2 - 254^2 = 509 smaller
    per component: distinct integers that round to the same f32 (ulp 256 there) except across steps."""
    rng = np.random.default_rng(65536)
    codes = np.zeros((N, dim), np.uint8)
    for r in range(8):
        codes[r, :r * 40] = 1
    codes[8:] = rng.integers(0, 256, (N - 8, dim), dtype=np.uint8)
    codes[8:N // 2, : dim - 64] = 0                       # most components at the extreme
    lo, hi = -1.0, 1.0
    cent = np.zeros((nlist, dim), f32)
    cent[1:] = 5.0
    off = np.array([0, N] + [N] * (nlist - 1), np.uint64)
    ix = IvfSqIndexData(dim=dim, nlist=nlist, metric="l2", centroids=cent, part_offsets=off, codes=codes,
                        row_ids=np.arange(N, dtype=np.uint64)[::-1].copy(), lo=lo, hi=hi, vectors=None)
    q = np.full((3, dim), 2.0, f32)                       # saturates at code 255
    q[1, :100] = -2.0                                     # code 0 on 100 components
    return ix, q


def _run_ivf(c, monkeypatch):
    w = c.w
    rng = np.random.default_rng(w["dim"] + c.N + len(c.kind))
    extreme = w.get("extreme", False)
    q = rng.standard_normal((c.B, w["dim"]), dtype=f32)
    if c.kind == "pq4":
        ix = random_pq4_index(rng, n=c.N, dim=w["dim"], nlist=w["nlist"], m=w["m"], with_vectors=False)
        handle, orc = _native.GpuIvfPq, pq4_oracle
    elif c.kind == "sq":
        ix, q = (_sq_extreme(c.N, w["dim"], w["nlist"]) if extreme
                 else (random_sq_index(rng, n=c.N, dim=w["dim"], nlist=w["nlist"]), q))
        handle, orc = _native.GpuIvfSq, sq_oracle
    elif c.kind == "hnsw_sq":
        ix = random_hnsw_index(rng, n=c.N, dim=w["dim"], nlist=w["nlist"])
        handle, orc = _native.GpuIvfHnswSq, hnsw_sq_oracle
    else:
        ix = random_rq_index(rng, n=c.N, dim=w["dim"], nlist=w["nlist"], metric=w["metric"])
        handle, orc = _native.GpuIvfRq, rq_oracle
    nprobes = w["nlist"] if extreme else 4
    gpu = handle(ix)
    try:
        got, st, scanned = _profiled(lambda: gpu.search(q, k=c.k, nprobes=nprobes))
    finally:
        gpu.close()
    want = orc.search(ix, q, k=c.k, nprobes=nprobes, nthreads=NT)
    assert_same(got, want, c.kind)
    assert st["queries"] == 0, st                                     # the kind's own scan, never the filter scan
    if c.kind != "hnsw_sq":
        assert scanned > 0 and scanned % {"pq4": w.get("m", 0) // 2 or 1}.get(c.kind, 1) == 0, scanned
    if extreme:
        top = float(want[1][0, -1])
        assert top == w["dim"] * 255.0 ** 2, top                      # 4,261,478,400: above 2^31, exact in f32
        assert (got[1][0] > 2.0 ** 31).sum() >= c.N // 2                # every row with most codes at 0


# ---- binary ----
def _binary_extreme(nbytes, n):
    """rows at Hamming distance 8 nbytes (2^24 at 2 MiB), 8 nbytes - 1 and a few below from query 0 (all ones)"""
    x = np.zeros((n, nbytes), np.uint8)
    x[1, 0] = 1                                           # 8 nbytes - 1
    x[2, : nbytes // 2] = 0xFF                            # 4 nbytes
    x[3] = 0xFF                                           # 0
    x[4, -1] = 0x80
    x[5:, 7] = 0x0F
    q = np.zeros((3, nbytes), np.uint8)
    q[0] = 0xFF
    q[1, ::3] = 0xAA
    return x, q


def _run_binary(c, monkeypatch):
    nb = c.w["nbytes"]
    rng = np.random.default_rng(nb + c.N)
    if c.w.get("extreme"):
        x, q = _binary_extreme(nb, c.N)
    else:
        x = rng.integers(0, 256, (c.N, nb), dtype=np.uint8)
        x[c.N // 2] = x[5]
        q = rng.integers(0, 256, (c.B, nb), dtype=np.uint8)
        q[0] = x[5]
    bx = _native.GpuBinary(x)
    try:
        got, st, _ = _profiled(lambda: bx.search(q, k=c.k))
    finally:
        bx.close()
    want = flat_search_u8(x, q, k=c.k, nthreads=NT)
    assert_same(got, want, "binary")
    route = "list" if st["candidates"] > 0 else ("tc_dense" if st["rescored"] > 0 else "simt")
    assert route == c.route, (route, st)
    if c.w.get("extreme"):
        assert want[1][0, -1] == f32(8 * nb) and want[1][0, -2] == f32(8 * nb - 1)


def _run_ivf_binary(c, monkeypatch):
    nb, nlist = c.w["nbytes"], c.w["nlist"]
    rng = np.random.default_rng(nb + c.N + 1)
    if c.w.get("extreme"):
        x, q = _binary_extreme(nb, c.N)
        cent = np.stack([np.zeros(nb, np.uint8), np.full(nb, 0xFF, np.uint8)])
        assign = np.array([0, 0, 1, 1, 0, 1])[: c.N]
    else:
        x = rng.integers(0, 256, (c.N, nb), dtype=np.uint8)
        q = x[rng.integers(0, c.N, c.B)].copy()
        q[1] ^= 0x10
        cent = rng.integers(0, 256, (nlist, nb), dtype=np.uint8)
        assign = rng.integers(0, nlist, c.N)              # not the nearest centroid: parity does not need it
    ix = ivf_binary_oracle.index_from_assignment(x, cent, assign)
    nprobes = nlist if c.w.get("extreme") else 5
    gpu = _native.GpuIvfBinary(ix)
    try:
        got = gpu.search(q, k=c.k, nprobes=nprobes)
    finally:
        gpu.close()
    want = ivf_binary_oracle.search(ix, q, k=c.k, nprobes=nprobes, nthreads=NT)
    assert_same(got, want, "ivf_binary")
    if c.w.get("extreme"):
        assert want[1][0, -1] == f32(8 * nb) and want[1][0, -2] == f32(8 * nb - 1)


# ---- multivector ----
def _mv_data(dim, T):
    """T stored vectors (fp16-exact, so the f32 and fp16 handles hold the same rows) in rows of 0..15, three queries
    of 1, 3 and 5 vectors; the oracle's result"""
    def make():
        rng = np.random.default_rng(dim + T)
        lens = np.full(T // 8, 8)
        n2 = lens.size // 2
        r = rng.integers(-8, 9, n2)
        lens[0:2 * n2:2] += r                                          # 0..16 vectors a row, T in all
        lens[1:2 * n2:2] -= r
        off = offsets_of(lens)
        x = rng.standard_normal((T, dim), dtype=f32).astype(np.float16).astype(f32)
        qoff = offsets_of([1, 3, 5])
        q = rng.standard_normal((9, dim), dtype=f32)
        q[0] = x[int(off[7])]                                         # on a stored vector
        return x, off, q, qoff, flat_search_mv(x, off, q, qoff, k=10, nthreads=NT)
    return _cached(("mv", dim, T), make)


def _run_multivec(c, monkeypatch):
    x, off, q, qoff, want = _mv_data(c.w["dim"], c.N)
    rows = x.astype(np.float16) if c.w["dtype"] == "f16" else x
    mv = _native.GpuMultivec(rows, off)
    try:
        assert mv.rows_on_host == ("LGPU_MULTIVEC_HBM_BYTES" in c.env)
        got, st, _ = _profiled(lambda: mv.search(q, k=c.k, q_offsets=qoff))
    finally:
        mv.close()
    assert_same(got, want, "multivec")
    nrows = off.size - 1
    route = "tc" if st["rescored"] < c.B * nrows else "exact"
    assert route == c.route, (route, st)


RUN = {"flat": _run_flat, "pq8": _run_pq8, "pq4": _run_ivf, "sq": _run_ivf, "hnsw_sq": _run_ivf, "rq": _run_ivf,
       "binary": _run_binary, "ivf_binary": _run_ivf_binary, "multivec": _run_multivec}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_wide_search_vs_oracle(name, monkeypatch):
    c = CASES[name]
    for var, value in c.env.items():
        monkeypatch.setenv(var, value)
    RUN[c.kind](c, monkeypatch)


@pytest.mark.gpu
def test_wide_pq8_tensor_core_coarse_step(monkeypatch):
    """dim 4096, nlist 1024, B 32 (B x nlist below 2^16): the exact coarse kernels by default, the tensor-core coarse
    step with LGPU_FORCE_TC_COARSE; both equal the oracle, and their launch sequences differ"""
    rng = np.random.default_rng(4096)
    ix = random_index(rng, dim=4096, nlist=1024, m=256, n=20000)
    q = rng.standard_normal((32, 4096), dtype=f32)
    q[:3] = ix.centroids[[0, 511, 1023]]
    want = oracle.OracleIndex.from_data(ix).search(q, k=10, nprobes=20, nthreads=NT)
    gpu = _native.GpuIvfPq(ix)
    try:
        launches = []
        for force in (False, True):
            if force:
                monkeypatch.setenv("LGPU_FORCE_TC_COARSE", "1")
            gpu.search(q, k=10, nprobes=20)
            got, n = _launches(lambda: gpu.search(q, k=10, nprobes=20))
            assert_same(got, want, f"LGPU_FORCE_TC_COARSE={force}")
            launches.append(n)
    finally:
        gpu.close()
    assert launches[0] != launches[1], "LGPU_FORCE_TC_COARSE changed no launch"


# ---- debug kernels at width ----
@pytest.mark.gpu
@pytest.mark.parametrize("d", [4096, 16384, 65528])
def test_wide_gemm_within_tc_band(d):
    """debug_gemm (bf16 wgmma, f32 accumulation) against float64: every score within tc_band of its exact value"""
    rng = np.random.default_rng(d)
    q = rng.standard_normal((8, d), dtype=f32)
    x = rng.standard_normal((300, d), dtype=f32)
    x[7] = q[1]
    got = _native.debug_gemm(q, x).astype(np.float64)
    q64, x64 = q.astype(np.float64), x.astype(np.float64)
    exact = (x64 ** 2).sum(1)[None, :] - 2.0 * q64 @ x64.T                           # |q - x|^2 - |q|^2
    for i in range(8):
        assert np.all(np.abs(got[i] - exact[i]) <= tc_band(q[i], x)), i


@pytest.mark.gpu
@pytest.mark.parametrize("d", [4096, 16384, 65528])
def test_wide_gemm_split_support_and_midpoints(d):
    """test_gemm_band's constructions at width: split support (the true nearest row scored high by ~2^-7 |q||x|, k
    decoys low by as much) and queries one f32 ulp beside bf16 midpoints; the GEMM stays within tc_band"""
    q, X = split_support_case(d, 1.0, 128, 10)
    got = _native.debug_gemm(q[None, :], X)[0].astype(np.float64)
    exact = (X.astype(np.float64) ** 2).sum(1) - 2.0 * X.astype(np.float64) @ q.astype(np.float64)
    e = tc_band(q, X)
    assert np.all(np.abs(got - exact) <= e)
    assert bf16(q).tolist() != q.tolist()                                            # the query does round


@pytest.mark.gpu
def test_wide_flat_split_support_end_to_end():
    """the split-support rows at d 4096 through the dense tensor-core route: the true nearest row comes back first"""
    q, X = split_support_case(4096, 1.0, 4096, 10)
    Q = np.tile(q, (8, 1))
    fl = _native.GpuFlat(X)
    try:
        got, st, _ = _profiled(lambda: fl.search(Q, k=10))
    finally:
        fl.close()
    want = oracle.flat_search(X, Q, k=10, nthreads=NT)
    assert want[0][0][0] == 4095 and st["rescored"] > 0
    assert_same(got, want, "split support d 4096")


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True])
@pytest.mark.parametrize("d", [4096, 65536])
def test_wide_maxsim_gemm_within_band(d, f16):
    """debug_maxsim_gemm(_f16) against the float64 similarity: within mv_band / mv_band_f16 at d 4096 and 65536"""
    from tests.test_multivec_f16_host import mv_band_f16
    from tests.test_multivec_host import mv_band
    rng = np.random.default_rng(d + f16)
    off = offsets_of([3, 0, 5, 1, 2])
    x = rng.standard_normal((11, d), dtype=f32)
    if f16:
        x = x.astype(np.float16)
    q = rng.standard_normal((4, d), dtype=f32)
    q[0] = x[2]
    got = _native.debug_maxsim_gemm(q, x, off).astype(np.float64)
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    sim = (q64 @ x64.T) / np.linalg.norm(q64, axis=1)[:, None] / np.linalg.norm(x64, axis=1)[None, :]
    e = float(mv_band_f16(1, d) if f16 else mv_band(1, d))
    for r in range(off.size - 1):
        a, b = int(off[r]), int(off[r + 1])
        if a == b:
            assert np.isnan(got[:, r]).all()
            continue
        assert np.all(np.abs(got[:, r] - sim[:, a:b].max(1)) <= e), r


@pytest.mark.gpu
@pytest.mark.parametrize("nbytes", [4096, 4100, 1 << 21])
def test_wide_hamming_gemm_exact(nbytes):
    """debug_hamming_gemm (b1 wgmma, K = 8 nbytes) against integer NumPy, distances up to 2^24"""
    rng = np.random.default_rng(nbytes)
    n = 6 if nbytes == 1 << 21 else 300
    x = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    x[0] = 0
    x[1] = 0
    x[1, 5] = 0x01
    q = rng.integers(0, 256, (3, nbytes), dtype=np.uint8)
    q[0] = 0xFF
    got = _native.debug_hamming_gemm(q, x)
    want = ivf_binary_oracle.hamming_np(q, x)
    assert np.array_equal(got.astype(np.int64), want)
    assert want[0, 0] == 8 * nbytes and want[0, 1] == 8 * nbytes - 1


@pytest.mark.gpu
def test_wide_pq4_sums_m256():
    """debug_pq4_sums at m 256 against integer NumPy: sums up to 255 x 256"""
    rng = np.random.default_rng(256)
    t = rng.integers(0, 256, (5, 256, 16), dtype=np.uint8)
    t[0] = 255
    codes = rng.integers(0, 256, (700, 128), dtype=np.uint8)
    got = _native.debug_pq4_sums(t, codes)
    nib = np.stack([codes & 0x0F, codes >> 4], 2).reshape(700, 256).astype(np.int64)
    want = t.astype(np.int64)[:, np.arange(256)[None, :], nib].sum(2)
    assert np.array_equal(got.astype(np.int64), want)
    assert (want[0] == 255 * 256).all()


@pytest.mark.gpu
@pytest.mark.parametrize("m", [512, 1024])
def test_wide_partition_distances(m):
    """debug_partition_distances at dim 4096, m 512 (dsub 8) and 1024 (dsub 4), against the oracle's"""
    rng = np.random.default_rng(m)
    ix = random_index(rng, dim=4096, nlist=4, m=m, n=3000)
    orc = oracle.OracleIndex.from_data(ix)
    gpu = _native.GpuIvfPq(ix)
    try:
        q = rng.standard_normal(4096, dtype=f32)
        for p in range(4):
            n_p = int(ix.part_offsets[p + 1] - ix.part_offsets[p])
            got = gpu.debug_partition_distances(q, p, n_p)
            assert np.array_equal(got.view(np.uint32), orc.partition_distances(q, p).view(np.uint32)), p
    finally:
        gpu.close()

"""CPU companion of tests/test_gpu_wide.py: every route predicate the wide cases rely on, restated from the host code
(small_scan_smem and the IVF plan in api.cu, gemm_shape_supported in gemm.cu, the flat, binary and multivector route
choices), and each case asserted to reach the route it claims -- and each width-dependent switch to be reached from
both sides.  Then the refusals one past each declared width limit, which come before any device work and so pass
without a GPU, and the oracles at wide shapes against their NumPy mirrors."""
import ctypes as C

import numpy as np
import pytest

from lancedb_b200 import _native
from tests import hamming_oracle, multivec_oracle, sq_oracle
from tests.sq_oracle import random_sq_index
from tests.test_gpu_wide import CASES

f32 = np.float32

# ---- the route predicates, restated ----
SMALL_SMEM_MAX = 200 * 1024        # api.cu ivf_plan: the small path's shared memory
SMALL_SLOTS = 1024                 # LGPU_SMALL_SLOTS default
FILTER_MAX_M = 512                 # api.cu ivf_plan: the filter scan's m
FLAT_TC_MIN_N, FLAT_TC_MIN_B, FLAT_SAMPLED_MIN_N = 4096, 8, 262144    # flat_tc_route, flat_score
HAM_SAMPLE, HAM_TC_MIN_B, HAM_TC_MIN_N = 65536, 128, 4096             # api.cu, binary routes
MV_TC_MIN_T = 65536                # multivector tensor-core path from this many stored vectors
MH_SLOT_BYTES = 4096               # dist.cu: the multivector host re-score's ring slots
RH_CHUNK_MAX = 1024                # the IVF host refine's floats per chunk
PQ8_NPROBES = 4                    # the nprobes of the wide PQ8 cases


def small_scan_smem(m, dim):
    return (256 * m + dim) * 4


def gemm_shape_supported(d):
    return d >= 8 and d % 8 == 0


def flat_route(dim, N, B, metric):
    if gemm_shape_supported(dim) and metric == "l2" and B >= FLAT_TC_MIN_B and N >= FLAT_TC_MIN_N:
        return "tc_sampled" if N >= FLAT_SAMPLED_MIN_N else "tc_dense"
    return "simt"


def pq8_route(dim, m, B, small_slots, nprobes=PQ8_NPROBES):
    if B * nprobes <= small_slots and small_scan_smem(m, dim) <= SMALL_SMEM_MAX:
        return "small"
    return "filter" if m <= FILTER_MAX_M and dim // m <= 32 else "exact"


def binary_route(N, B):
    if N > HAM_SAMPLE:
        return "list"
    return "tc_dense" if B >= HAM_TC_MIN_B and N >= HAM_TC_MIN_N else "simt"


def multivec_route(dim, T):
    return "tc" if T >= MV_TC_MIN_T and gemm_shape_supported(dim) else "exact"


def route(c):
    w = c.w
    if c.kind == "flat":
        routes = {flat_route(w["dim"], c.N, c.B, metric) for metric in w["metrics"]}
        assert len(routes) == 1, routes
        return routes.pop()
    if c.kind == "pq8":
        # the suite runs with LGPU_SMALL_SLOTS=0 (tests/conftest.py) unless a case sets it
        return pq8_route(w["dim"], w["m"], c.B, int(c.env.get("LGPU_SMALL_SLOTS", 0)))
    if c.kind == "binary":
        return binary_route(c.N, c.B)
    if c.kind == "multivec":
        return multivec_route(w["dim"], c.N)
    return {"pq4": "pq4", "sq": "sq", "hnsw_sq": "hnsw", "rq": "rq", "ivf_binary": "ivf_ham"}[c.kind]


@pytest.mark.parametrize("name", list(CASES))
def test_case_reaches_its_route(name):
    assert route(CASES[name]) == CASES[name].route


def _cases(kind, **match):
    return [c for c in CASES.values() if c.kind == kind and all(c.w.get(a) == v for a, v in match.items())]


def test_every_width_switch_is_reached_from_both_sides():
    pq8 = _cases("pq8")
    smem = {(c.w["m"], c.w["dim"]): small_scan_smem(c.w["m"], c.w["dim"]) for c in pq8}
    # the small path's shared memory: m 192 in at dim 1536 and out at 3072; m 199 in and m 200 out at dsub 1
    assert smem[(192, 1536)] == 202752 <= SMALL_SMEM_MAX < smem[(192, 3072)] == 208896
    assert smem[(199, 199)] <= SMALL_SMEM_MAX < smem[(200, 200)]
    assert all(int(c.env["LGPU_SMALL_SLOTS"]) == SMALL_SLOTS for c in pq8 if (c.w["m"], c.w["dim"]) in
               ((192, 1536), (192, 3072), (199, 199), (200, 200)))
    # the filter scan's m <= 512: m 512 and m 1024 at dim 4096; dsub 32 at dim 16384 (the table floor's widest)
    assert {(c.w["m"], c.route) for c in pq8 if c.w["dim"] == 4096} >= {(512, "filter"), (1024, "exact")}
    assert any(c.w["dim"] == 16384 and c.w["m"] == 512 and c.route == "filter" for c in pq8)
    # no dimension limit on PQ8: the exact scan at dim 32768, m 1024 (dsub 32) and 2048 (dsub 16)
    assert {c.w["m"] for c in pq8 if c.w["dim"] == 32768} == {1024, 2048}
    # the refine over raw vectors, in HBM and on the host, reads rows in several host-refine chunks
    refine = [c for c in pq8 if c.w.get("refine")]
    assert {"LGPU_VECTORS_HBM_BYTES" in c.env for c in refine} == {False, True}
    assert all(c.w["dim"] > 2 * RH_CHUNK_MAX for c in refine)
    # flat: each route at dims 3072 and 4096 or beyond, one dim that is a multiple of 8 but not of 64 on the sampled
    # route, one that is not a multiple of 8 on the exact kernels; both row types
    flat = _cases("flat")
    for dt in ("f32", "f16"):
        routes = {(c.w["dim"], c.route) for c in flat if c.w["dtype"] == dt}
        assert routes >= {(3072, "simt"), (4096, "simt"), (3072, "tc_dense"), (4096, "tc_dense"),
                          (2056, "tc_sampled"), (4099, "simt")}
    assert 2056 % 8 == 0 and 2056 % 64 != 0 and not gemm_shape_supported(4099)
    assert any(c.w["dim"] == 4099 and c.N >= FLAT_TC_MIN_N and c.B >= FLAT_TC_MIN_B for c in flat)
    # multivector: vectors of one ring slot or fewer and of several, both routes, both placements, both row types
    mv = _cases("multivec")
    slots = {(c.w["dtype"], (c.w["dim"] * (2 if c.w["dtype"] == "f16" else 4) + MH_SLOT_BYTES - 1) // MH_SLOT_BYTES)
             for c in mv}
    assert {("f16", 1), ("f16", 2), ("f32", 2), ("f32", 4)} <= slots
    assert {(c.w["dtype"], "LGPU_MULTIVEC_HBM_BYTES" in c.env, c.route) for c in mv} == {
        (dt, host, r) for dt in ("f32", "f16") for host in (False, True) for r in ("tc", "exact")}
    assert any(c.route == "exact" and c.N >= MV_TC_MIN_T and not gemm_shape_supported(c.w["dim"]) for c in mv)
    # binary: nbytes 4096 and 4100 on every route; 2 MiB (2^24 bits) flat and indexed
    bins = _cases("binary")
    assert {(c.w["nbytes"], c.route) for c in bins} >= {(nb, r) for nb in (4096, 4100)
                                                         for r in ("simt", "tc_dense", "list")}
    assert max(c.w["nbytes"] for c in bins) * 8 == 1 << 24
    assert max(c.w["nbytes"] for c in _cases("ivf_binary")) * 8 == 1 << 24
    # the integer kinds at their limits
    assert max(c.w["dim"] for c in _cases("sq")) == 65536 and 65536 * 255 ** 2 == 4261478400 < 1 << 32
    assert max(c.w["dim"] for c in _cases("rq")) == 4096
    assert {c.w["metric"] for c in _cases("rq")} == {"l2", "cosine"}
    assert max(c.w["m"] for c in _cases("pq4")) == 256


# ---- one past each declared limit: LGPU_INVALID_INPUT before any device work ----
def _refused(rc, what):
    assert rc == _native.LGPU_INVALID_INPUT, rc
    assert what.encode() in _native.load().lgpu_last_error(), _native.load().lgpu_last_error()


def test_sq_and_hnsw_sq_refuse_dim_65537():
    lib = _native.load()
    c, off = np.zeros((1, 16), f32), np.zeros(2, np.uint64)
    sq = _native.SqDesc(_native.ABI_VERSION, 65537, 1, 0, 0, 0, 0, 0.0, 1.0, c.ctypes.data, off.ctypes.data, None, None,
                        None)
    h = C.c_void_p()
    _refused(lib.lgpu_ivf_sq_open(C.byref(sq), C.byref(h)), "up to 65536")
    hn = _native.HnswSqDesc(sq, 8, 0, 0, None, None, None, None, None, None)
    _refused(lib.lgpu_ivf_hnsw_sq_open(C.byref(hn), C.byref(h)), "up to 65536")
    assert h.value is None


def test_rq_refuses_dim_4097():
    lib = _native.load()
    c, off, P = np.zeros((1, 16), f32), np.zeros(2, np.uint64), np.eye(16, dtype=f32)
    d = _native.RqDesc(_native.ABI_VERSION, 4097, 1, 0, 0, 1, 0, c.ctypes.data, P.ctypes.data, off.ctypes.data, None,
                       None, None, None, None)
    h = C.c_void_p()
    _refused(lib.lgpu_ivf_rq_open(C.byref(d), C.byref(h)), "up to 4096")
    assert h.value is None


@pytest.mark.parametrize("opener", ["lgpu_multivec_open", "lgpu_multivec_open_f16"])
def test_multivec_refuses_dim_65537(opener):
    off = np.zeros(2, np.uint64)
    h = C.c_void_p()
    _refused(getattr(_native.load(), opener)(None, off.ctypes.data, 1, 65537, None, 0, C.byref(h)), "[1, 65536]")
    assert h.value is None
    with pytest.raises(ValueError, match="65536"):                       # the Python handle refuses it first
        _native.GpuMultivec(np.zeros((0, 65537), f32), off)


def test_binary_refuses_2_24_plus_8_bits():
    lib = _native.load()
    nb = (1 << 21) + 1                                                    # 2^24 + 8 bits
    x = np.zeros((1, nb), np.uint8)
    h = C.c_void_p()
    _refused(lib.lgpu_binary_open(x.ctypes.data, 1, nb, None, 0, C.byref(h)), "above 2^24 bits")
    c, off, ids = np.zeros((1, nb), np.uint8), np.array([0, 1], np.uint64), np.zeros(1, np.uint64)
    d = _native.IvfBinaryDesc(_native.ABI_VERSION, nb, 1, 0, 1, c.ctypes.data, off.ctypes.data, x.ctypes.data,
                              ids.ctypes.data)
    _refused(lib.lgpu_ivf_binary_open(C.byref(d), C.byref(h)), "above 2^24 bits")
    assert h.value is None


def test_pq4_refuses_m_258():
    lib = _native.load()
    m, dim = 258, 516
    c, off = np.zeros((1, dim), f32), np.zeros(2, np.uint64)
    cb = np.zeros((m, 16, 2), f32)
    d = _native.IndexDesc(_native.ABI_VERSION, dim, 1, m, 4, 0, 1, 0, 0, c.ctypes.data, cb.ctypes.data,
                          off.ctypes.data, None, None, None)
    h = C.c_void_p()
    _refused(lib.lgpu_index_open(C.byref(d), C.byref(h)), "up to 256")
    assert h.value is None


# ---- the oracles at wide shapes against their NumPy mirrors ----
def test_sq_oracle_at_dim_4096_matches_numpy():
    rng = np.random.default_rng(4096)
    ix = random_sq_index(rng, n=300, dim=4096, nlist=4)
    q = rng.standard_normal((3, 4096), dtype=f32)
    got = sq_oracle.search(ix, q, k=10, nprobes=2, nthreads=4)
    want = sq_oracle.sq_search_np(ix, q, k=10, nprobes=2)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_sq_oracle_distance_at_dim_65536_extremes():
    """the largest IVF_SQ l2 distance, 65536 x 255^2 = 4,261,478,400 (above 2^31, exact in f32), and one 509 below it,
    which rounds to the same f32"""
    a, b = np.zeros(65536, np.uint8), np.full(65536, 255, np.uint8)
    assert sq_oracle.sq_distance(a, b) == f32(4261478400)
    a[0] = 1
    assert sq_oracle.sq_distance(a, b) == f32(4261478400 - 509) == sq_oracle.sq_distances_np(a[None], b)[0, 0]


def test_hamming_oracle_at_4100_bytes_and_2_24_bits_matches_numpy():
    rng = np.random.default_rng(4100)
    x = rng.integers(0, 256, (200, 4100), dtype=np.uint8)
    q = rng.integers(0, 256, (3, 4100), dtype=np.uint8)
    got = hamming_oracle.flat_search_u8(x, q, k=10, nthreads=4)
    want = hamming_oracle.flat_search_u8_np(x, q, k=10)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    x = np.zeros((2, 1 << 21), np.uint8)
    x[1, 9] = 0x40
    q = np.full((1, 1 << 21), 0xFF, np.uint8)
    ids, dist, cnt = hamming_oracle.flat_search_u8(x, q, k=2, nthreads=4)
    assert dist[0].tolist() == [float((1 << 24) - 1), float(1 << 24)] and ids[0].tolist() == [1, 0]


def test_multivec_oracle_at_dim_2049_matches_numpy():
    rng = np.random.default_rng(2049)
    off = multivec_oracle.offsets_of([3, 0, 2, 5, 1])
    x = rng.standard_normal((11, 2049), dtype=f32)
    qoff = multivec_oracle.offsets_of([2, 1])
    q = rng.standard_normal((3, 2049), dtype=f32)
    got = multivec_oracle.flat_search_mv(x, off, q, qoff, k=4, nthreads=4)
    want = multivec_oracle.flat_search_mv_np(x, off, q, qoff, k=4)
    assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want))

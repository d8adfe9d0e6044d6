"""Tensor-core (wgmma) GEMM shortlist: numerics of the GEMM itself (tolerance: it is bf16), and bit-exact
parity of the paths that use it as a candidate generator (flat L2, IVF coarse step) -- the
exact re-score decides, so ids/distances must still equal the oracle's bit for bit."""
import numpy as np
import pytest
import torch

import oracle
from lancedb_b200 import _native
from tests.util import queries, random_index, same_result, split_support_case

pytestmark = pytest.mark.gpu


def _bf16(a):
    return torch.from_numpy(a).to(torch.bfloat16).to(torch.float32).numpy()


@pytest.mark.parametrize("B,N,d", [(128, 256, 64), (1, 1, 8), (130, 300, 72), (1000, 5000, 768), (16, 70000, 128)])
def test_gemm_numerics(B, N, d):
    rng = np.random.default_rng(B + N + d)
    q = queries(rng, B, d); x = queries(rng, N, d)
    got = _native.debug_gemm(q, x)
    qb, xb = _bf16(q).astype(np.float64), _bf16(x).astype(np.float64)
    want = (x.astype(np.float64) ** 2).sum(1)[None, :] - 2.0 * qb @ xb.T
    scale = np.abs(want).max() + 1.0
    err = np.abs(got - want).max()
    assert err <= 2e-5 * scale * max(1.0, d / 256), f"max abs err {err} (scale {scale})"


@pytest.mark.parametrize("n,dim,B,k", [(20000, 128, 64, 10), (6000, 1536, 33, 10), (9000, 64, 200, 100)])
def test_flat_tensorcore_path_bit_exact(n, dim, B, k):
    rng = np.random.default_rng(n)
    v = queries(rng, n, dim)
    v[n // 2] = v[3]; v[n // 3] = v[3]                    # exact duplicates -> ties by row id
    rid = rng.permutation(n).astype(np.uint64)
    q = queries(rng, B, dim)
    q[0] = v[3]
    fl = _native.GpuFlat(v, row_ids=rid)
    gi, gd, gc = fl.search(q, k=k, metric="l2")
    oi, od, oc = oracle.flat_search(v, q, k=k, metric="l2", row_ids=rid, nthreads=8)
    fl.close()
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


def test_flat_tensorcore_filtered_epilogue_large_n():
    """N >= 256k takes the sampled-threshold + filtering-epilogue path (no dense score matrix)"""
    rng = np.random.default_rng(31)
    n, dim = 300_000, 64
    v = queries(rng, n, dim)
    v[200_000] = v[7]; v[299_999] = v[7]                  # ties across the sampled and unsampled parts
    q = queries(rng, 24, dim)
    q[0] = v[7]
    fl = _native.GpuFlat(v)
    for k in (10, 40):
        gi, gd, gc = fl.search(q, k=k)
        oi, od, oc = oracle.flat_search(v, q, k=k, nthreads=8)
        assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
        assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    fl.close()


def test_coarse_filtered_path_large_nlist(monkeypatch):
    """nlist >= 4096: sampled threshold + filtering epilogue picks the probes; result must equal the oracle"""
    monkeypatch.setenv("LGPU_FORCE_TC_COARSE", "1")
    rng = np.random.default_rng(17)
    sizes = np.full(4200, 3, np.int64); sizes[::7] = 0
    ix = random_index(rng, dim=64, nlist=4200, m=8, sizes=sizes)
    q = queries(rng, 40, 64)
    gpu = _native.GpuIvfPq(ix)
    orc = oracle.OracleIndex.from_data(ix)
    for nprobes in (20, 50):
        gi, gd, gc = gpu.search(q, k=10, nprobes=nprobes)
        oi, od, oc = orc.search(q, k=10, nprobes=nprobes, nthreads=8)
        assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
        assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    gpu.close()

@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_coarse_sampled_list_path(metric, monkeypatch):
    """Many lists (default from nlist 8192, here forced at 4200): dense scores of every 8th centroid give a per-query
    bound, the full GEMM's filtering epilogue appends (column, score) of the columns under it to a list, and the
    finishing kernel works on the list.  Probe sets -- hence results -- must equal the oracle's, including for queries
    that sit ON a centroid (distance 0, ties in the band) and with clustered centroids (a loose sample bound)."""
    monkeypatch.setenv("LGPU_FORCE_TC_COARSE", "1")
    monkeypatch.setenv("LGPU_COARSE_LIST_MIN", "1024")
    rng = np.random.default_rng(19)
    sizes = np.full(4200, 3, np.int64); sizes[::5] = 0
    ix = random_index(rng, dim=64, nlist=4200, m=8, metric=metric, sizes=sizes)
    # the first 600 centroids in one tight cluster (consecutive ids, like a hierarchical trainer leaves them)
    ix.centroids[:600] = ix.centroids[0] + 0.01 * rng.standard_normal((600, 64)).astype(np.float32)
    if metric == "cosine":
        ix.centroids /= np.linalg.norm(ix.centroids, axis=1, keepdims=True)
    q = queries(rng, 48, 64)
    q[:6] = ix.centroids[[5, 100, 599, 700, 2000, 4199]]
    q[6:9] = ix.centroids[3] * np.float32(1.0001)
    gpu = _native.GpuIvfPq(ix)
    orc = oracle.OracleIndex.from_data(ix)
    for nprobes in (1, 20, 50):
        gi, gd, gc = gpu.search(q, k=10, nprobes=nprobes)
        oi, od, oc = orc.search(q, k=10, nprobes=nprobes, nthreads=8)
        assert np.array_equal(gc, oc) and np.array_equal(gi, oi), nprobes
        assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    gpu.close()

def test_coarse_sampled_list_path_default_switch():
    """nlist 8192 with B x nlist >= 1M takes the sampled-bound + list-epilogue coarse step by default (no environment
    switch): probe sets, hence ids and distance bits, equal the oracle's; empty partitions interleaved."""
    rng = np.random.default_rng(29)
    sizes = np.full(8192, 2, np.int64); sizes[::3] = 0
    ix = random_index(rng, dim=64, nlist=8192, m=8, sizes=sizes)
    q = queries(rng, 160, 64)
    q[:4] = ix.centroids[[0, 8, 4097, 8191]]                     # on a sampled / unsampled centroid
    gpu = _native.GpuIvfPq(ix)
    gi, gd, gc = gpu.search(q, k=10, nprobes=20)
    oi, od, oc = oracle.OracleIndex.from_data(ix).search(q, k=10, nprobes=20, nthreads=8)
    gpu.close()
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


def test_coarse_default_path_c2_shape():
    """B x nlist >= 1M with nlist >= 1024 (BASELINE config 2's coarse shape) takes the tensor-core
    shortlist by default; probes and final results must equal the oracle."""
    rng = np.random.default_rng(23)
    sizes = rng.integers(0, 9, 1024).astype(np.int64)
    ix = random_index(rng, dim=64, nlist=1024, m=8, sizes=sizes)
    q = queries(rng, 1100, 64)
    gpu = _native.GpuIvfPq(ix)
    gi, gd, gc = gpu.search(q, k=10, nprobes=20)
    oi, od, oc = oracle.OracleIndex.from_data(ix).search(q, k=10, nprobes=20, nthreads=8)
    gpu.close()
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


def test_flat_tensorcore_clustered_fallback():
    """near-duplicate rows make the error band overflow the shortlist -> exact fix-up path"""
    rng = np.random.default_rng(5)
    base = queries(rng, 1, 64)
    v = (base + 1e-3 * rng.standard_normal((8192, 64))).astype(np.float32)
    q = (base + 1e-3 * rng.standard_normal((16, 64))).astype(np.float32)
    fl = _native.GpuFlat(v)
    gi, gd, gc = fl.search(q, k=10)
    oi, od, oc = oracle.flat_search(v, q, k=10, nthreads=8)
    fl.close()
    assert np.array_equal(gi, oi) and np.array_equal(gd.view(np.uint32), od.view(np.uint32))


@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("nprobes", [20, 37])
def test_coarse_tensorcore_path_bit_exact(metric, nprobes, monkeypatch):
    monkeypatch.setenv("LGPU_FORCE_TC_COARSE", "1")
    rng = np.random.default_rng(11)
    ix = random_index(rng, dim=128, nlist=700, m=16, metric=metric, n=30000)
    q = queries(rng, 70, 128)
    gpu = _native.GpuIvfPq(ix)
    orc = oracle.OracleIndex.from_data(ix)
    parts, dists = gpu.debug_coarse(q, nprobes)              # exact reference path
    gi, gd, gc = gpu.search(q, k=10, nprobes=nprobes)        # tensor-core shortlist path inside
    oi, od, oc = orc.search(q, k=10, nprobes=nprobes, nthreads=8)
    gpu.close()
    for i in range(q.shape[0]):
        qn = oracle.normalize(q[i]) if metric == "cosine" else q[i]
        op, _, _ = orc.find_partitions(qn, nprobes)
        assert np.array_equal(parts[i], op)
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


# ---- adversarial bf16 rounding (tests/util.py split_support_case, tests/test_gemm_band.py): the true nearest row is
# scored ~2^-7 |q||x| too high and k decoys as much too low, so only a band that allows for BOTH operands' rounding
# keeps it.  Each path must still return the oracle's result bit for bit (directly, or through its exact fix-up).
def _split_support_flat(n):
    q, X = split_support_case(64, 1.0, n, 10)
    Q = np.tile(q, (8, 1))
    fl = _native.GpuFlat(X)
    got = fl.search(Q, k=10)
    fl.close()
    want = oracle.flat_search(X, Q, k=10, nthreads=8)
    assert want[0][0][0] == n - 1                                   # the construction's true nearest row
    assert same_result(got, want)


def test_flat_dense_shortlist_adversarial_rounding():
    """N = 4096: the kp = 256 shortlist + band check"""
    _split_support_flat(4096)


def test_flat_filtered_adversarial_rounding():
    """N = 262144: threshold from the first Ns rows (the decoys are there, the true nearest row is not) + filtering"""
    _split_support_flat(262144)


@pytest.mark.parametrize("list_path", [False, True])
def test_coarse_adversarial_rounding(list_path, monkeypatch):
    """IVF coarse step (dense finishing kernel, or the sampled bound + list with the decoys on sampled centroids): only
    the true nearest centroid's partition holds rows, so a missed probe changes the counts"""
    monkeypatch.setenv("LGPU_FORCE_TC_COARSE", "1")
    if list_path:
        monkeypatch.setenv("LGPU_COARSE_LIST_MIN", "1024")
    nlist = 1024
    q, C = split_support_case(64, 1.0, nlist, 10)
    sizes = np.zeros(nlist, np.int64); sizes[-1] = 5
    ix = random_index(np.random.default_rng(3), dim=64, nlist=nlist, m=8, sizes=sizes)
    ix.centroids = C
    Q = np.tile(q, (8, 1))
    gpu = _native.GpuIvfPq(ix)
    got = gpu.search(Q, k=10, nprobes=10)
    gpu.close()
    want = oracle.OracleIndex.from_data(ix).search(Q, k=10, nprobes=10, nthreads=8)
    assert (want[2] == 5).all()
    assert same_result(got, want)


@pytest.mark.parametrize("d", [64, 768, 1536])
def test_gemm_accumulation_rounding(d):
    """tc_band's 4 d 2^-24 (|q| + xmax)^2 term for the f32 sums.  bf16-exact operands make every product exact, so only
    the accumulation (and |x|^2) rounds; the rows are ordered adversarially: one large product then many 3/4-ulp ones,
    the same with alternating signs, and random signs.  The error against the exact score must stay within that term.
    This holds whether wgmma rounds to nearest or truncates (either errs by <= 2 u per addition); the bound does not tell
    them apart, test_gemm_accumulation_of_sub_ulp_products measures which.  The largest error is printed."""
    rng = np.random.default_rng(d)
    q = np.ones((8, d), np.float32)
    q[1::2, 1::2] = -1                                       # queries 1, 3, ..: alternating signs
    X = np.zeros((256, d), np.float32)
    X[:, 0] = 2.0 ** 8
    X[:128, 1:] = 0.75 * 2.0 ** -15                          # 3/4 of an f32 ulp of 2^8
    X[128:192, 1:] = 0.75 * 2.0 ** -15 * np.where(np.arange(1, d) % 2, 1, -1)
    X[192:, 1:] = _bf16(rng.standard_normal((64, d - 1)).astype(np.float32))
    got = _native.debug_gemm(q, X).astype(np.float64)
    qx = q.astype(np.float64) @ X.astype(np.float64).T                                     # exact
    want = (X.astype(np.float64) ** 2).sum(1).astype(np.float32).astype(np.float64)[None, :] - 2.0 * qx
    s = np.sqrt((q.astype(np.float64) ** 2).sum(1))[:, None] + np.sqrt((X.astype(np.float64) ** 2).sum(1).max())
    err = np.abs(got - want)
    assert (err <= 4.0 * d * 2.0 ** -24 * s * s).all()
    print(f"wgmma accumulation, d={d}: largest error {float((err / (2.0 ** -24 * s * s)).max()):.3f} u (|q| + xmax)^2")


@pytest.mark.parametrize("d", [64, 768, 1536])
def test_gemm_accumulation_of_sub_ulp_products(d):
    """What wgmma's f32 accumulation does with products below one ulp of the running sum: q = [256, 1, 1, ..],
    x = [1, 3/4 ulp(256), ...] (all bf16-exact, every product exact), so q.x = 256 + (d - 1) 3/4 ulp(256) exactly and
    the score |x|^2 - 2 q.x ~ -511 keeps q.x to 1/2 ulp(256).  Accumulating one product at a time, round-to-nearest
    keeps ~(d - 1) ulp (each 3/4 rounds up to 1), truncation keeps none; a wider internal sum keeps (d - 1) 3/4.  The
    kept fraction is printed; the assertion is the tc_band term (4 d u (|q| + xmax)^2), which covers all three."""
    q = np.ones((1, d), np.float32)
    q[0, 0] = 256
    x = np.full((1, d), 0.75 * 2.0 ** -15, np.float32)
    x[0, 0] = 1
    got = float(_native.debug_gemm(q, x)[0, 0])
    xn2 = float(np.float32((x.astype(np.float64) ** 2).sum()))
    exact = 256 + (d - 1) * 0.75 * 2.0 ** -15
    acc = (xn2 - got) / 2
    s = np.sqrt(256.0 ** 2 + d - 1) + np.sqrt(1 + (d - 1) * (0.75 * 2.0 ** -15) ** 2)
    assert abs(2 * acc - 2 * exact) <= 4.0 * d * 2.0 ** -24 * s * s
    print(f"wgmma sub-ulp accumulation, d={d}: kept {(acc - 256) / 2.0 ** -15:.2f} ulp(256) of the exact "
          f"{(d - 1) * 0.75:.2f} ({(d - 1):d} with round-to-nearest one at a time, 0 with truncation)")

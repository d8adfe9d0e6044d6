"""Index-build passes through the C ABI (lgpu_ivf_assign / lgpu_pq_encode, csrc/build.cu) against the oracle:
bit-exact partition ids and PQ codes, and an index of every float kind built with them searched against the oracle.
The training kernels (lgpu_kmeans_train / lgpu_pq_train) are compared with an exact Lloyd run in test_gpu_train.py."""
import numpy as np
import pytest

import oracle
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS, train_ivf_pq
from tests import hnsw_sq_oracle, rq_oracle, sq_oracle
from tests.train_oracle import assign_chunk_rows, threaded
from tests.util import queries, random_index

pytestmark = pytest.mark.gpu

# rows per case where the default (1000, or 300 at dim 768) does not cross what the case is for
ASSIGN_ROWS = {
    (32, 8, 3): 65536 + 37,       # past lgpu_pq_encode's 65536-row chunk and lgpu_ivf_assign's at small nlist
    (32, 8, 2000): 40000,         # lgpu_ivf_assign's chunk at nlist 2000 is 33554 rows
}


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dim,m,nlist", [(64, 8, 17), (48, 3, 5), (32, 32, 40), (768, 96, 64),
                                         (64, 32, 17), (64, 16, 17), (64, 2, 17),      # dsub 2, 4, 32
                                         (32, 8, 3), (32, 4, 1), (32, 8, 2000)])
def test_assign_and_encode_match_oracle(metric, dim, m, nlist):
    rng = np.random.default_rng(41)
    ix = random_index(rng, dim=dim, nlist=nlist, m=m, metric=metric, n=200)
    n = ASSIGN_ROWS.get((dim, m, nlist), 1000 if dim < 768 else 300)
    if (dim, m, nlist) in ASSIGN_ROWS:
        assert n > assign_chunk_rows(nlist)
    v = queries(rng, n, dim)
    v[3] = ix.centroids[min(2, nlist - 1)]                      # a row sitting exactly on a centroid
    if nlist > 1:
        ix.centroids[nlist - 1] = ix.centroids[0]               # two identical centroids: the tie goes to the lower
        v[4] = ix.centroids[0]                                  # and a row on both of them
    orc = oracle.OracleIndex.from_data(ix)
    want_parts, want_codes = np.empty(n, np.uint32), np.empty((n, m), np.uint8)

    def run(r0, r1):
        want_parts[r0:r1] = orc.ivf_assign(v[r0:r1])
        want_codes[r0:r1] = orc.pq_encode(v[r0:r1], want_parts[r0:r1])
    threaded(run, n)
    parts = _native.ivf_assign(ix.centroids, v, metric)
    assert np.array_equal(parts, want_parts)
    if nlist > 1:
        assert parts[4] == 0
    codes = _native.pq_encode(ix.centroids, ix.codebook, v, parts, metric)
    assert codes.shape == (n, m) and codes.dtype == np.uint8
    assert np.array_equal(codes, want_codes)
    if metric == "cosine":                  # an all-zero row has no direction: NaN to every centroid, no partition
        v[5] = 0
        with pytest.raises(ValueError, match="no finite centroid distance"):
            _native.ivf_assign(ix.centroids, v[:16], metric)


def test_encode_rejects_bad_input():
    rng = np.random.default_rng(42)
    ix = random_index(rng, dim=32, nlist=4, m=4, n=50)
    v = queries(rng, 5, 32)
    with pytest.raises(ValueError):
        _native.pq_encode(ix.centroids, ix.codebook, v, np.full(5, 9, np.uint32))        # partition out of range
    assert _native.ivf_assign(ix.centroids, v[:0]).shape == (0,)


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_index_built_with_native_passes(metric):
    """train_ivf_pq(native_passes=True): every row's own vector probes its partition first, its codes are the
    oracle's encoding for the trained centroids/codebook, and the index searches bit-identically."""
    rng = np.random.default_rng(43)
    n, dim = 3000, 32
    v = (rng.standard_normal((n, 8)) @ rng.standard_normal((8, dim))).astype(np.float32)
    v += 0.05 * rng.standard_normal((n, dim)).astype(np.float32)
    ix = train_ivf_pq(v, num_partitions=12, num_sub_vectors=4, distance_type=metric, max_iterations=8,
                      keep_vectors=True, device="cuda", native_passes=True)
    orc = oracle.OracleIndex.from_data(ix)
    part_of_row = np.repeat(np.arange(ix.nlist), np.diff(ix.part_offsets.astype(np.int64))).astype(np.uint32)
    assert np.array_equal(orc.ivf_assign(ix.vectors), part_of_row)
    want = orc.pq_encode(ix.vectors, part_of_row)
    for p in range(ix.nlist):
        a, b = int(ix.part_offsets[p]), int(ix.part_offsets[p + 1])
        got = ix.codes_t[a * ix.m:b * ix.m].reshape(ix.m, b - a).T
        assert np.array_equal(got, want[a:b])
    gpu = _native.GpuIvfPq(ix)
    q = v[rng.choice(n, 40, replace=False)]
    gi, gd, gc = gpu.search(q, k=5, nprobes=4)
    oi, od, oc = orc.search(q, k=5, nprobes=4, nthreads=4)
    gpu.close()
    assert np.array_equal(gi, oi) and np.array_equal(gd.view(np.uint32), od.view(np.uint32)) and np.array_equal(gc, oc)


def _same_search(got, want, what):
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2]), f"{what}: ids / counts"
    assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), f"{what}: distances"


_ORACLE_SEARCH = {"IVF_SQ": sq_oracle.search, "IVF_RQ": rq_oracle.search, "IVF_HNSW_SQ": hnsw_sq_oracle.search}


@pytest.mark.parametrize("kind,metric", [(k, mt) for k in _ORACLE_SEARCH for mt in IVF_KINDS[k].metrics])
def test_sq_rq_hnsw_index_built_with_native_passes(kind, metric):
    """IVF_SQ, IVF_RQ and IVF_HNSW_SQ trained with native_passes (lgpu_kmeans_train + lgpu_ivf_assign): every row sits
    in the partition its own raw vector probes first, and the index searches bit-identically to its oracle."""
    rng = np.random.default_rng(44)
    n, dim = 3000, 32
    v = (rng.standard_normal((n, 8)) @ rng.standard_normal((8, dim))).astype(np.float32)
    v += 0.05 * rng.standard_normal((n, dim)).astype(np.float32)
    extra = {"m": 8, "ef_construction": 40} if kind == "IVF_HNSW_SQ" else {}
    data = IVF_KINDS[kind].train(v, num_partitions=12, distance_type=metric, max_iterations=8, keep_vectors=True,
                                 device="cuda", native_passes=True, **extra)
    ivf = getattr(data, "sq", data)
    orc = oracle.OracleIndex(dim=dim, nlist=ivf.nlist, m=1, metric=metric, centroids=ivf.centroids,
                             codebook=np.zeros(0, np.float32), part_offsets=ivf.part_offsets,
                             codes_t=np.zeros(0, np.uint8), row_ids=ivf.row_ids)
    part_of_row = np.repeat(np.arange(ivf.nlist), np.diff(ivf.part_offsets.astype(np.int64))).astype(np.uint32)
    assert np.array_equal(orc.ivf_assign(ivf.vectors), part_of_row)
    assert np.array_equal(ivf.vectors, v[ivf.row_ids.astype(np.int64)])
    gpu = getattr(_native, IVF_KINDS[kind].handle)(data)
    q = v[rng.choice(n, 40, replace=False)]
    try:
        got = gpu.search(q, k=5, nprobes=4)
    finally:
        gpu.close()
    _same_search(got, _ORACLE_SEARCH[kind](data, q, k=5, nprobes=4, nthreads=4), f"{kind} {metric}")


@pytest.mark.parametrize("kind", [k for k, v in IVF_KINDS.items() if "cosine" in v.metrics])
def test_cosine_build_on_the_gpu_refuses_an_all_zero_row(kind):
    """An all-zero row has no direction, so under cosine no partition: create_index(accelerator="cuda") refuses it by
    index before any training, as the default build does (test_train_host.py), instead of failing inside
    lgpu_ivf_assign after training."""
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(45)
    x = rng.standard_normal((2000, 32)).astype(np.float32)
    x[1234] = 0
    t = lancedb.connect("memory://").create_table("v", {"vector": x, "id": np.arange(2000)})
    kw = dict(num_partitions=8, max_iterations=3, index_type=kind, accelerator="cuda", m=8, ef_construction=40,
              num_bits=1 if kind == "IVF_RQ" else 8)
    n0 = _native_launches()
    with pytest.raises(ValueError, match=r"vector 1234 has norm 0"):
        t.create_index(metric="cosine", **kw)
    assert _native_launches() == n0
    t.create_index(metric="l2", **kw)
    assert _native_launches() > n0


def test_create_index_with_accelerator_trains_on_the_gpu_and_matches_the_oracle():
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(63)
    x = rng.standard_normal((8000, 64)).astype(np.float32)
    t = lancedb.connect("memory://").create_table("v", {"vector": x, "id": np.arange(8000)})
    n0 = _native_launches()
    t.create_index(metric="l2", num_partitions=16, num_sub_vectors=8, max_iterations=5, accelerator="cuda")
    assert _native_launches() > n0
    q = rng.standard_normal((4, 64)).astype(np.float32)
    orc = oracle.OracleIndex.from_data(t._index_data["vector"])
    oi, od, oc = orc.search(q, k=10, nprobes=6)
    for i in range(4):
        out = t.search(q[i]).nprobes(6).limit(10).with_row_id(True).to_arrow()
        assert out["_rowid"].to_pylist() == [int(v) for v in oi[i, :10]]


def _native_launches():
    from lancedb_b200 import _native
    return _native.kernel_launch_count()

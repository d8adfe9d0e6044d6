"""Binary IVF_FLAT (hamming) on the GPU: the b1 MMA scan kernel against NumPy integers, GpuIvfBinary against the C
oracle (ids, counts and distance bits) over row widths, list counts, batch sizes, k, ties, empty partitions, prefilter
with maximum_nprobes, distance_range, refine_factor, timeout and the host / filtered / device entry points; nprobes =
nlist against the flat binary search; then the reference's known answer through create_index."""
import numpy as np
import pytest

import lancedb_b200 as lancedb
import pyarrow as pa
from lancedb_b200 import _native
from tests import ivf_binary_oracle as O
from tests.util import assert_same

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,N,nbytes", [(1, 1, 1), (7, 300, 3), (8, 257, 32), (9, 33, 33), (13, 1000, 128),
                                        (5, 1100, 1024), (3, 600, 4099)])
def test_debug_scan_equals_numpy(B, N, nbytes):
    rng = np.random.default_rng(B * 1000 + nbytes)
    q = rng.integers(0, 256, (B, nbytes), dtype=np.uint8)
    x = rng.integers(0, 256, (N, nbytes), dtype=np.uint8)
    x[: min(N, 2)] = 255
    q[0] = 0
    got = _native.debug_ivf_hamming_scan(q, x)
    assert np.array_equal(got, O.hamming_np(q, x).astype(np.uint32))


@pytest.mark.parametrize("n,nbytes,nlist,B,k,nprobes,patterns,empty", [
    (3000, 1, 1, 1, 1, 1, 0, ()),
    (5000, 3, 16, 7, 10, 4, 16, ()),
    (6000, 32, 64, 8, 100, 8, 0, (0, 5, 9)),
    (4000, 33, 100, 9, 2048, 20, 4, ()),
    (2000, 1024, 32, 64, 50, 5, 0, (1,)),
    (20000, 128, 4096, 1024, 10, 20, 0, ()),        # B x nlist large enough for the b1 wgmma coarse step
    (12000, 16, 512, 1024, 7, 3, 64, ()),
])
def test_gpu_ivf_binary_equals_oracle(n, nbytes, nlist, B, k, nprobes, patterns, empty):
    rng = np.random.default_rng(n + nbytes + nlist)
    ix = O.random_index(rng, n, nbytes, nlist, empty=empty, patterns=patterns)
    q = ix.vectors[rng.integers(0, n, B)] ^ (rng.random((B, nbytes)) < 0.1).astype(np.uint8)
    gpu = _native.GpuIvfBinary(ix)
    assert_same(gpu.search(q, k=k, nprobes=nprobes), O.search(ix, q, k=k, nprobes=nprobes), "search")
    gpu.close()


@pytest.mark.parametrize("nlist,nbytes", [(1, 8), (37, 33), (4096, 16)])
def test_all_probes_equal_flat_binary_search(nlist, nbytes):
    rng = np.random.default_rng(nlist)
    ix = O.random_index(rng, 30000, nbytes, nlist, patterns=200, row_ids=rng.permutation(100000)[:30000])
    q = rng.integers(0, 256, (64, nbytes), dtype=np.uint8)
    gpu = _native.GpuIvfBinary(ix)
    got = gpu.search(q, k=20, nprobes=nlist)
    if nlist > 2048:                                     # above the select's k limit nprobes must cover every partition
        assert_same(gpu.search(q, k=20, nprobes=nlist + 5), got, "nprobes > nlist")
        with pytest.raises(ValueError, match="2048"):
            gpu.search(q, k=20, nprobes=3000)
    gpu.close()
    flat = _native.GpuBinary(ix.vectors, row_ids=ix.row_ids)
    want = flat.search(q, k=20)
    flat.close()
    assert_same(got, want, "nprobes = nlist vs flat")


def test_prefilter_range_refine_timeout_and_entry_points():
    import torch
    rng = np.random.default_rng(11)
    n, nbytes, nlist = 40000, 24, 200
    ix = O.random_index(rng, n, nbytes, nlist, empty=(3, 7), patterns=500)
    q = ix.vectors[rng.integers(0, n, 33)]
    gpu = _native.GpuIvfBinary(ix)
    mask = rng.random(n) < 0.004
    bm = _native.mask_bitmap(mask)
    for mx in (0, 50, nlist):
        got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=n, max_nprobes=mx)
        assert_same(got, O.search(ix, q, k=10, nprobes=2, allow=mask, max_nprobes=mx), f"prefilter max_nprobes={mx}")
    d = O.search(ix, q[:1], k=60, nprobes=6)[1][0]
    lo, hi = float(d[5]), float(d[40])
    assert_same(gpu.search(q, k=20, nprobes=6, lower=lo, upper=hi),
                O.search(ix, q, k=20, nprobes=6, lower=lo, upper=hi),
                "distance_range")
    assert_same(gpu.search(q, k=7, nprobes=6, refine_factor=5), O.search(ix, q, k=7, nprobes=6), "refine_factor")
    assert_same(gpu.search(q, k=7, nprobes=6, timeout_ms=60000), O.search(ix, q, k=7, nprobes=6), "generous timeout")
    want = O.search(ix, q, k=9, nprobes=6)
    p = _native.make_params(9, 6)
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    di = torch.empty((33, 9), dtype=torch.int64, device="cuda")
    dd = torch.empty((33, 9), dtype=torch.float32, device="cuda")
    dc = torch.empty(33, dtype=torch.int32, device="cuda")
    gpu.search_device(dq.data_ptr(), 33, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(), 0)
    torch.cuda.synchronize()
    assert_same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want, "device")
    _native.set_profiling(True)
    gpu.search(q, k=9, nprobes=6)
    stages = _native.last_stage_ms()
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    assert scanned > 0 and scanned % 32 == 0 and stages["scan"] >= 0 and stages["total"] > 0
    gpu.close()


def test_multi_sub_batch_and_timeout():
    # one query's distance segments hold all 300000 rows: the default 8 GiB workspace takes ~7000 queries per sub-batch
    rng = np.random.default_rng(12)
    n, nbytes, nlist = 300000, 8, 2
    ix = O.random_index(rng, n, nbytes, nlist, patterns=3000)
    q = rng.integers(0, 256, (9000, nbytes), dtype=np.uint8)
    gpu = _native.GpuIvfBinary(ix)
    assert_same(gpu.search(q, k=5, nprobes=2), O.search(ix, q, k=5, nprobes=2), "two sub-batches")
    with pytest.raises(TimeoutError, match="timeout"):
        gpu.search(q, k=5, nprobes=2, timeout_ms=1)
    gpu.close()


def test_known_answer_through_create_index():
    """python/python/tests/test_index.py:491-512: rows [i] * 128, IvfFlat(hamming, num_partitions=10),
    nearest_to([v] * 128) is row v"""
    x = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 128, axis=1)
    db = lancedb.connect("memory://")
    schema = pa.schema([pa.field("vector", pa.list_(pa.uint8(), 128)), pa.field("id", pa.int64())])
    t = db.create_table("t", pa.table({"vector": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), 128),
                                       "id": np.arange(256)}, schema=schema))
    t.create_index(metric="hamming", num_partitions=10, index_type="IVF_FLAT", accelerator="cuda")   # k-modes on the GPU
    assert t.list_indices()[0]["index_type"] == "IVF_FLAT"
    for v in range(256):
        out = t.search(np.full(128, v)).distance_type("hamming").limit(1).to_arrow()
        assert out["id"].to_pylist() == [v] and out["_distance"].to_pylist() == [0.0]


def test_unused_refine_factor_and_maximum_nprobes_are_not_limited():
    # refine_factor changes nothing, so k * refine_factor may exceed the select's 2048; maximum_nprobes is only read
    # when it widens under a prefilter, so without one any value is accepted
    rng = np.random.default_rng(13)
    n, nbytes, nlist = 30000, 16, 4096
    ix = O.random_index(rng, n, nbytes, nlist, patterns=300)
    q = ix.vectors[rng.integers(0, n, 40)]
    gpu = _native.GpuIvfBinary(ix)
    want = O.search(ix, q, k=300, nprobes=8)
    assert_same(gpu.search(q, k=300, nprobes=8, refine_factor=10), want, "k x refine_factor above 2048")
    assert_same(gpu.search(q, k=300, nprobes=8, max_nprobes=3000), want, "maximum_nprobes without a prefilter")
    mask = rng.random(n) < 0.01
    with pytest.raises(ValueError, match="maximum_nprobes"):
        gpu.search(q, k=20, nprobes=8, allow=_native.mask_bitmap(mask), allow_bits=n, max_nprobes=3000)
    gpu.close()


@pytest.mark.parametrize("nbytes", [40, 128])
def test_trainer_on_the_gpu_equals_the_cpu_and_numpy(nbytes):
    """k-modes on the GPU is exact integer work: rows wider than 256 bits (where a bf16 dot product would round) land in
    the same partitions as on the CPU and in the NumPy mirror"""
    from lancedb_b200.index import kmodes_assign, train_ivf_binary
    rng = np.random.default_rng(nbytes)
    pats = rng.integers(0, 256, (40, nbytes), dtype=np.uint8)
    x = pats[rng.integers(0, 40, 6000)] ^ (rng.random((6000, nbytes)) < 0.2).astype(np.uint8)
    g = train_ivf_binary(x, num_partitions=24, max_iterations=6, sample_rate=64, seed=3, device="cuda")
    c = train_ivf_binary(x, num_partitions=24, max_iterations=6, sample_rate=64, seed=3)
    for f in ("centroids", "part_offsets", "vectors", "row_ids"):
        assert np.array_equal(getattr(g, f), getattr(c, f)), f
    assign = np.repeat(np.arange(24), np.diff(g.part_offsets.astype(np.int64)))
    assert np.array_equal(assign, np.argmin(O.hamming_np(g.vectors, g.centroids), axis=1))   # every row's nearest
    r = np.random.default_rng(3)                         # the trainer's sample and initial rows, then kmodes_np
    samp = x[np.sort(r.choice(6000, 1536, replace=False))]
    init = samp[r.choice(1536, 24, replace=False)]
    cent, _ = O.kmodes_np(samp, init, 6)
    assert np.array_equal(g.centroids, cent)
    # the assignment alone, on 1024-bit rows with dot products far above 256 and tied centroids
    xs = rng.integers(0, 256, (5000, 128), dtype=np.uint8)
    cs = rng.integers(0, 256, (64, 128), dtype=np.uint8)
    cs[7] = cs[3]
    assert np.array_equal(kmodes_assign(xs, cs, "cuda"), np.argmin(O.hamming_np(xs, cs), axis=1))

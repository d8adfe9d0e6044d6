"""IVF_SQ on the GPU: the integer tensor-core scan kernel against NumPy integers, and GpuIvfSq against the C oracle
(ids, counts and distance bits) over metrics, list counts, batch sizes, k, partition shapes, awkward queries, prefilter,
maximum_nprobes, distance_range, refine_factor and every search entry point; then create_index through the builder."""
import ctypes as C
import threading

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests import sq_oracle
from tests.sq_oracle import random_sq_index

pytestmark = pytest.mark.gpu
f32 = np.float32


def _same(got, want, what=""):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ"
    assert np.array_equal(gi, oi), f"{what}: ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distance bits differ"


@pytest.mark.parametrize("B,N,dim", [(1, 1, 1), (7, 300, 7), (8, 257, 31), (9, 5000, 32), (130, 1000, 33),
                                     (33, 2000, 768), (5, 4099, 1000), (130, 5000, 64)])
def test_debug_sq_distances_equal_numpy_integers(B, N, dim):
    rng = np.random.default_rng(B * 1000 + dim)
    q = rng.integers(0, 256, (B, dim), dtype=np.uint8)
    x = rng.integers(0, 256, (N, dim), dtype=np.uint8)
    x[: min(N, 3)] = 255                                 # extreme rows
    got = _native.debug_sq_distances(q, x)
    qi, xi = q.astype(np.int64), x.astype(np.int64)
    want = (xi * xi).sum(1)[None, :] + (qi * qi).sum(1)[:, None] - 2 * (qi @ xi.T)
    assert np.array_equal(got.astype(np.int64), want)


def test_debug_sq_distances_above_2_31_wrap_exactly():
    # 65536 x 255^2 = 4261478400 > 2^31: the s32 accumulator wraps, the u32 result must not
    dim = 65536
    q = np.zeros((3, dim), np.uint8)
    q[1] = 255
    q[2, ::2] = 255
    x = np.full((5, dim), 255, np.uint8)
    x[1] = 0
    got = _native.debug_sq_distances(q, x).astype(np.int64)
    qi, xi = q.astype(np.int64), x.astype(np.int64)
    want = (xi * xi).sum(1)[None, :] + (qi * qi).sum(1)[:, None] - 2 * (qi @ xi.T)
    assert np.array_equal(got, want) and want.max() == 65536 * 65025


def _queries(rng, ix, B):
    q = rng.standard_normal((B, ix.dim)).astype(f32)
    if B > 3:
        q[1] *= 1000.0                                    # far outside the bounds: codes saturate
        q[2, 0] = np.nan                                  # no finite centroid distance: no rows
        q[3] = ix.vectors[7]                              # an exact stored row (and its duplicates)
    return q


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_sq_small_lists_vs_oracle(metric):
    rng = np.random.default_rng(21 if metric == "l2" else 22)
    ix = random_sq_index(rng, n=6000, dim=40, nlist=16, metric=metric, empty=(2, 9))
    gpu = _native.GpuIvfSq(ix)
    for B in (1, 7, 8, 37):
        q = _queries(rng, ix, B)
        for k, nprobes in ((1, 3), (10, 5), (100, 16)):
            got = gpu.search(q, k=k, nprobes=nprobes)
            _same(got, sq_oracle.search(ix, q, k=k, nprobes=nprobes), f"B={B} k={k} nprobes={nprobes}")
            if B > 3:
                assert got[2][2] == 0
    gpu.close()
    # k > N, tiny and empty partitions, every partition probed
    tiny = random_sq_index(rng, n=150, dim=40, nlist=16, metric=metric, empty=(0, 3, 4))
    gpu = _native.GpuIvfSq(tiny)
    q = _queries(rng, tiny, 9)
    got = gpu.search(q, k=200, nprobes=16)
    _same(got, sq_oracle.search(tiny, q, k=200, nprobes=16), "k > N")
    assert got[2][0] == 150
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_sq_tensor_core_coarse_step_vs_oracle(metric):
    rng = np.random.default_rng(23 if metric == "l2" else 24)
    ix = random_sq_index(rng, n=60000, dim=128, nlist=1024, metric=metric, empty=(5, 77))
    gpu = _native.GpuIvfSq(ix)
    q = _queries(rng, ix, 1024)
    for k, nprobes in ((10, 20), (100, 8)):
        _same(gpu.search(q, k=k, nprobes=nprobes), sq_oracle.search(ix, q, k=k, nprobes=nprobes), f"k={k}")
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_sq_prefilter_range_refine_vs_oracle(metric):
    rng = np.random.default_rng(25 if metric == "l2" else 26)
    ix = random_sq_index(rng, n=8000, dim=48, nlist=32, metric=metric)
    gpu = _native.GpuIvfSq(ix)
    q = _queries(rng, ix, 40)
    nbits = ix.nrows * 3 + 7
    mask = rng.random(nbits) < 0.02                           # narrow: many queries need maximum_nprobes
    bm = _native.mask_bitmap(mask)
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits, max_nprobes=32)
    _same(got, sq_oracle.search(ix, q, k=10, nprobes=2, allow=mask, max_nprobes=32), "prefilter + maximum_nprobes")
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits)
    _same(got, sq_oracle.search(ix, q, k=10, nprobes=2, allow=mask), "prefilter")
    d = sq_oracle.search(ix, q[:1], k=50, nprobes=4)[1][0]
    lo, hi = float(d[5]), float(d[30])
    got = gpu.search(q, k=20, nprobes=4, lower=lo, upper=hi)
    _same(got, sq_oracle.search(ix, q, k=20, nprobes=4, lower=lo, upper=hi), "distance_range")
    got = gpu.search(q, k=7, nprobes=4, refine_factor=5)
    _same(got, sq_oracle.search(ix, q, k=7, nprobes=4, refine_factor=5), "refine_factor")
    gpu.close()


def test_ivf_sq_device_async_and_coalesced_entry_points(monkeypatch):
    import torch
    # the coalescing window is read once per process, at the first coalesced call: take the one
    # test_gpu_api.py's batching test needs, whichever of the two runs first
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")
    rng = np.random.default_rng(27)
    ix = random_sq_index(rng, n=5000, dim=32, nlist=24)
    gpu = _native.GpuIvfSq(ix)
    q = _queries(rng, ix, 19)
    want = sq_oracle.search(ix, q, k=9, nprobes=6)
    p = _native.make_params(9, 6)
    dq = torch.from_numpy(q).cuda()
    di = torch.empty((19, 9), dtype=torch.int64, device="cuda")
    dd = torch.empty((19, 9), dtype=torch.float32, device="cuda")
    dc = torch.empty(19, dtype=torch.int32, device="cuda")
    gpu.search_device(dq.data_ptr(), 19, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(), 0)
    torch.cuda.synchronize()
    _same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want, "device")
    ids = np.empty((19, 9), np.uint64); dist = np.empty((19, 9), f32); cnt = np.empty(19, np.uint32)
    _native.ticket_wait(gpu.search_async(q, p, ids, dist, cnt))
    _same((ids, dist, cnt), want, "async")
    res = [None] * 19

    def one(i):
        res[i] = gpu.search_one(q[i], k=9, nprobes=6)

    th = [threading.Thread(target=one, args=(i,)) for i in range(19)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i in range(19):
        gi, gd, gc = res[i]
        assert gc == want[2][i] and np.array_equal(gi, want[0][i])
        assert np.array_equal(gd.view(np.uint32), want[1][i].view(np.uint32))
    assert gpu.device_bytes() >= ix.nrows * (64 + 4 + 8)     # codes padded to 64 bytes, |k|^2, row ids
    _native.set_profiling(True)
    gpu.search(q, k=9, nprobes=6)
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    assert scanned > 0 and scanned % ix.dim == 0
    gpu.close()


def test_ivf_sq_rejections():
    rng = np.random.default_rng(28)
    ix = random_sq_index(rng, n=500, dim=16, nlist=4)
    gpu = _native.GpuIvfSq(ix)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_filter_bounds(ix.vectors[:2], 2, 10)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_partition_distances(ix.vectors[0], 0, 10)
    gpu.close()
    # the C ABI itself rejects dot and dimensions above 65536
    lib = _native.load()
    c = np.zeros((1, 16), f32); off = np.zeros(2, np.uint64)
    for metric, dim in ((2, 16), (0, 65537)):
        desc = _native.SqDesc(_native.ABI_VERSION, dim, 1, metric, 0, 0, 0, 0.0, 1.0, c.ctypes.data, off.ctypes.data,
                              None, None, None)
        h = C.c_void_p()
        with pytest.raises(ValueError):
            _native.check(lib.lgpu_ivf_sq_open(C.byref(desc), C.byref(h)))


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_create_index_ivf_sq_search_to_arrow(metric):
    rng = np.random.default_rng(29)
    x = rng.standard_normal((5000, 64)).astype(f32)
    db = lancedb.connect("memory://")
    t = db.create_table("v", {"vector": x, "id": np.arange(5000)})
    t.create_index(metric=metric, num_partitions=16, index_type="IVF_SQ", max_iterations=4, accelerator="cuda")
    assert t.list_indices()[0]["index_type"] == "IVF_SQ"
    data = t._index_data["vector"]
    q = rng.standard_normal((3, 64)).astype(f32)
    oi, od, oc = sq_oracle.search(data, q, k=12, nprobes=4)
    for i in range(3):
        out = t.search(q[i]).distance_type(metric).nprobes(4).limit(10).offset(2).with_row_id(True).to_arrow()
        assert out["_rowid"].to_pylist() == [int(v) for v in oi[i, 2:12]]
        assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32).view(np.uint32), od[i, 2:12].view(np.uint32))
        assert out["id"].to_pylist() == out["_rowid"].to_pylist()
    out = t.search(q[0]).distance_type(metric).nprobes(4).refine_factor(3).limit(5).to_arrow()
    rd = sq_oracle.search(data, q[:1], k=5, nprobes=4, refine_factor=3)[1]
    assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32), rd[0])
    # recall against the exact flat search: SQ ranks close to f32
    import oracle
    fi = oracle.flat_search(x, q, k=10, metric=metric)[0]
    gi = _native.GpuIvfSq.search(t._index["vector"], q, k=10, nprobes=16)[0]
    assert np.mean([len(set(fi[b]) & set(gi[b])) / 10 for b in range(3)]) >= 0.6

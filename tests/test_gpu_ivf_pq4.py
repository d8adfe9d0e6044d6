"""4-bit IVF_PQ on the GPU: the pair-table scan kernel against NumPy integer sums, and GpuIvfPq(num_bits = 4) against the
C oracle (ids, counts and distance bits) over metrics, list counts, batch sizes, k, partition shapes, ties, awkward
queries, both code layouts, prefilter, maximum_nprobes, distance_range, refine_factor and every search entry point; the
per-partition debug path; the rejections; then create_index through the builder."""
import ctypes as C
import threading

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from lancedb_b200.aio import IvfPq
from lancedb_b200.index import IvfPqIndexData
from tests import pq4_oracle
from tests.pq4_oracle import random_pq4_index, row_major_codes, sums_np

pytestmark = pytest.mark.gpu
f32 = np.float32


def _same(got, want, what=""):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ"
    assert np.array_equal(gi, oi), f"{what}: ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distance bits differ"


@pytest.mark.parametrize("B,N,m", [(1, 1, 2), (7, 300, 8), (8, 2049, 48), (9, 5000, 96), (17, 4099, 16),
                                   (3, 2048, 256), (130, 777, 30), (5, 6000, 2)])
def test_debug_pq4_sums_equal_numpy_integers(B, N, m):
    rng = np.random.default_rng(B * 1000 + m)
    t = rng.integers(0, 256, (B, m, 16), dtype=np.uint8)
    codes = rng.integers(0, 256, (N, m // 2), dtype=np.uint8)
    got = _native.debug_pq4_sums(t, codes)
    assert np.array_equal(got.astype(np.int64), sums_np(t, codes))


def test_debug_pq4_sums_all_255_at_the_largest_m():
    # 255 x 256 = 65280: the largest lane sum, one below 2^16 - 255, must not carry into the neighbouring slot
    m = 256
    t = np.full((9, m, 16), 255, np.uint8)
    t[1] = 0
    codes = np.random.default_rng(3).integers(0, 256, (2500, m // 2), dtype=np.uint8)
    got = _native.debug_pq4_sums(t, codes)
    assert np.array_equal(got.astype(np.int64), sums_np(t, codes))
    assert got.max() == 255 * 256 and (got[1] == 0).all()


def _queries(rng, ix, B):
    q = rng.standard_normal((B, ix.dim)).astype(f32)
    if B > 3:
        q[1] *= 1000.0                                    # far from every codeword
        q[2, 0] = np.nan                                  # no finite centroid distance: no rows
        if ix.vectors is not None:
            q[3] = ix.vectors[7]
    return q


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq4_small_lists_vs_oracle(metric):
    rng = np.random.default_rng({"l2": 31, "cosine": 32, "dot": 33}[metric])
    ix = random_pq4_index(rng, n=6000, dim=48, nlist=16, m=12, metric=metric, empty=(2, 9))
    gpu = _native.GpuIvfPq(ix)
    for B in (1, 7, 8, 37):
        q = _queries(rng, ix, B)
        for k, nprobes in ((1, 3), (10, 5), (100, 16)):
            got = gpu.search(q, k=k, nprobes=nprobes)
            _same(got, pq4_oracle.search(ix, q, k=k, nprobes=nprobes), f"B={B} k={k} nprobes={nprobes}")
            if B > 3:
                assert got[2][2] == 0
    gpu.close()
    # k > N, one-row and empty partitions, every partition probed
    tiny = random_pq4_index(rng, n=150, dim=48, nlist=16, m=12, metric=metric,
                            sizes=[0, 1, 0, 30, 1, 20, 0, 18, 1, 40, 0, 10, 9, 10, 0, 10])
    gpu = _native.GpuIvfPq(tiny)
    q = _queries(rng, tiny, 9)
    got = gpu.search(q, k=200, nprobes=16)
    _same(got, pq4_oracle.search(tiny, q, k=200, nprobes=16), "k > N")
    assert got[2][0] == 150
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq4_tensor_core_coarse_step_vs_oracle(metric):
    rng = np.random.default_rng({"l2": 34, "cosine": 35, "dot": 36}[metric])
    ix = random_pq4_index(rng, n=60000, dim=128, nlist=1024, m=16, metric=metric, empty=(5, 77), with_vectors=False)
    gpu = _native.GpuIvfPq(ix)
    q = _queries(rng, ix, 1024)
    for k, nprobes in ((10, 20), (100, 8)):
        _same(gpu.search(q, k=k, nprobes=nprobes), pq4_oracle.search(ix, q, k=k, nprobes=nprobes), f"k={k}")
    gpu.close()


@pytest.mark.parametrize("m,dim", [(2, 64), (48, 768), (96, 768), (256, 256), (32, 1024)])
def test_ivf_pq4_sub_vector_lengths_and_long_partitions_vs_oracle(m, dim):
    # dsub 32, 16, 8, 1 and 32; partitions longer than one 2048-row tile
    rng = np.random.default_rng(37 + m)
    ix = random_pq4_index(rng, n=9000, dim=dim, nlist=3, m=m, metric="l2", empty=(), with_vectors=False)
    gpu = _native.GpuIvfPq(ix)
    q = _queries(rng, ix, 11)
    _same(gpu.search(q, k=50, nprobes=2), pq4_oracle.search(ix, q, k=50, nprobes=2), f"m={m}")
    gpu.close()


def test_ivf_pq4_ties_at_the_kth_place_and_row_major_layout():
    rng = np.random.default_rng(40)
    ix = random_pq4_index(rng, n=3000, dim=32, nlist=4, m=8, metric="l2", empty=())
    # partition 0: every row the same code bytes -> every distance equal, ordered by row id
    a, b = int(ix.part_offsets[0]), int(ix.part_offsets[1])
    w = ix.code_bytes
    ix.codes_t[a * w:b * w] = np.repeat(rng.integers(0, 256, w, dtype=np.uint8), b - a)
    q = _queries(rng, ix, 16)
    want = pq4_oracle.search(ix, q, k=10, nprobes=4)
    gpu = _native.GpuIvfPq(ix)
    _same(gpu.search(q, k=10, nprobes=4), want, "transposed codes")
    gpu.close()
    # the same index handed over row-major: the open re-lays it out to the same scan
    rm = np.ascontiguousarray(row_major_codes(ix))
    keep = [np.ascontiguousarray(ix.centroids), np.ascontiguousarray(ix.codebook), ix.part_offsets, rm, ix.row_ids,
            ix.vectors]
    desc = _native.IndexDesc(_native.ABI_VERSION, ix.dim, ix.nlist, ix.m, 4, _native.METRICS[ix.metric], 0, 0,
                             ix.nrows, *[a.ctypes.data for a in keep])
    h = C.c_void_p()
    _native.check(_native.load().lgpu_index_open(C.byref(desc), C.byref(h)))
    g2 = _native.GpuIvfPq.__new__(_native.GpuIvfPq)
    g2._h, g2.dim, g2.nlist, g2.m, g2.metric = h, ix.dim, ix.nlist, ix.m, ix.metric
    _same(g2.search(q, k=10, nprobes=4), want, "row-major codes")
    g2.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq4_prefilter_range_refine_vs_oracle(metric):
    rng = np.random.default_rng({"l2": 41, "cosine": 42, "dot": 43}[metric])
    ix = random_pq4_index(rng, n=8000, dim=48, nlist=32, m=24, metric=metric)
    gpu = _native.GpuIvfPq(ix)
    q = _queries(rng, ix, 40)
    nbits = int(ix.row_ids.max()) + 1 - 37
    mask = rng.random(nbits) < 0.02                           # narrow: many queries need maximum_nprobes
    bm = _native.mask_bitmap(mask)
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits, max_nprobes=32)
    _same(got, pq4_oracle.search(ix, q, k=10, nprobes=2, allow=mask, max_nprobes=32), "prefilter + maximum_nprobes")
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits)
    _same(got, pq4_oracle.search(ix, q, k=10, nprobes=2, allow=mask), "prefilter")
    d = pq4_oracle.search(ix, q[:1], k=50, nprobes=4)[1][0]
    lo, hi = float(d[5]), float(d[30])
    got = gpu.search(q, k=20, nprobes=4, lower=lo, upper=hi)
    _same(got, pq4_oracle.search(ix, q, k=20, nprobes=4, lower=lo, upper=hi), "distance_range")
    got = gpu.search(q, k=7, nprobes=4, refine_factor=5)
    _same(got, pq4_oracle.search(ix, q, k=7, nprobes=4, refine_factor=5), "refine_factor")
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq4_debug_partition_distances_vs_oracle(metric):
    rng = np.random.default_rng(44)
    ix = random_pq4_index(rng, n=5000, dim=64, nlist=5, m=16, metric=metric, empty=())
    gpu = _native.GpuIvfPq(ix)
    q = rng.standard_normal(64).astype(f32)
    for p in range(ix.nlist):
        n = int(ix.part_offsets[p + 1] - ix.part_offsets[p])
        got = gpu.debug_partition_distances(q, p, n)
        assert np.array_equal(got.view(np.uint32), pq4_oracle.partition_distances(ix, q, p).view(np.uint32))
    gpu.close()


def test_ivf_pq4_device_async_and_coalesced_entry_points(monkeypatch):
    import torch
    # the coalescing window is read once per process, at the first coalesced call: take the one
    # test_gpu_api.py's batching test needs, whichever of the two runs first
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")
    rng = np.random.default_rng(45)
    ix = random_pq4_index(rng, n=5000, dim=32, nlist=24, m=8)
    gpu = _native.GpuIvfPq(ix)
    q = _queries(rng, ix, 19)
    want = pq4_oracle.search(ix, q, k=9, nprobes=6)
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
    _native.set_profiling(True)
    gpu.search(q, k=9, nprobes=6)
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    assert scanned > 0 and scanned % (ix.m // 2) == 0
    gpu.close()


def test_ivf_pq4_rejections():
    rng = np.random.default_rng(46)
    ix = random_pq4_index(rng, n=500, dim=16, nlist=4, m=4)
    gpu = _native.GpuIvfPq(ix)
    with pytest.raises(ValueError, match="8-bit IVF_PQ"):
        gpu.debug_filter_bounds(ix.vectors[:2], 2, 10)
    gpu.close()
    # the C ABI itself rejects an odd m, m above LGPU_PQ4_MAX_M, an unsupported dsub and nbits other than 4 or 8
    lib = _native.load()
    off = np.zeros(2, np.uint64)
    for dim, m, nbits in ((12, 3, 4), (512, 512, 4), (192, 2, 4), (16, 4, 2), (16, 4, 1), (16, 4, 16)):
        c = np.zeros((1, dim), f32); cb = np.zeros(m * 256 * (dim // m), f32)
        desc = _native.IndexDesc(_native.ABI_VERSION, dim, 1, m, nbits, 0, 1, 0, 0, c.ctypes.data, cb.ctypes.data,
                                 off.ctypes.data, None, None, None)
        h = C.c_void_p()
        with pytest.raises(ValueError):
            _native.check(lib.lgpu_index_open(C.byref(desc), C.byref(h)))
    with pytest.raises(ValueError):
        _native.check(lib.lgpu_debug_pq4_sums(None, 1, None, 1, 3, 0, None))


@pytest.mark.parametrize("metric,accelerator", [("l2", None), ("cosine", "cuda"), ("dot", "cuda")])
def test_create_index_ivf_pq4_search_to_arrow(metric, accelerator):
    rng = np.random.default_rng(47)
    x = rng.standard_normal((5000, 64)).astype(f32)
    db = lancedb.connect("memory://")
    t = db.create_table("v", {"vector": x, "id": np.arange(5000)})
    t.create_index(metric=metric, num_partitions=16, num_bits=4, max_iterations=4, accelerator=accelerator)
    data = t._index_data["vector"]
    assert isinstance(data, IvfPqIndexData) and data.num_bits == 4 and data.m == 4
    assert t.list_indices()[0]["index_type"] == "IVF_PQ"
    q = rng.standard_normal((3, 64)).astype(f32)
    oi, od, oc = pq4_oracle.search(data, q, k=12, nprobes=4)
    for i in range(3):
        out = t.search(q[i]).distance_type(metric).nprobes(4).limit(10).offset(2).with_row_id(True).to_arrow()
        assert out["_rowid"].to_pylist() == [int(v) for v in oi[i, 2:12]]
        assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32).view(np.uint32), od[i, 2:12].view(np.uint32))
    out = t.search(q[0]).distance_type(metric).nprobes(4).refine_factor(3).limit(5).to_arrow()
    rd = pq4_oracle.search(data, q[:1], k=5, nprobes=4, refine_factor=3)[1]
    assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32), rd[0])


def test_async_create_index_ivf_pq4():
    import asyncio
    rng = np.random.default_rng(48)
    x = rng.standard_normal((3000, 32)).astype(f32)

    async def run():
        db = await lancedb.connect_async("memory://")
        t = await db.create_table("v", {"vector": x})
        await t.create_index("vector", config=IvfPq(num_partitions=8, num_bits=4, max_iterations=2))
        return t._table._index_data["vector"]

    data = asyncio.run(run())
    assert data.num_bits == 4 and data.m == 2 and data.codebook.shape == (2, 16, 16)

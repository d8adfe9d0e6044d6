"""4-bit IVF_PQ on the GPU, what only this kind has: the pair-table scan kernel against NumPy integer sums, GpuIvfPq
(num_bits = 4) against the C oracle (ids, counts and distance bits) over sub-vector lengths, long partitions, ties at
the k-th place and both code layouts, the per-partition debug path, the rejections, and create_index through the async
builder.  The search cases 4-bit IVF_PQ shares with IVF_SQ and IVF_RQ are in test_gpu_ivf_kinds.py."""
import ctypes as C

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from lancedb_b200.aio import IvfPq
from tests import pq4_oracle
from tests.pq4_oracle import random_pq4_index, row_major_codes, sums_np
from tests.util import assert_same, ivf_queries

pytestmark = pytest.mark.gpu
f32 = np.float32


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


@pytest.mark.parametrize("m,dim", [(2, 64), (48, 768), (96, 768), (256, 256), (32, 1024)])
def test_ivf_pq4_sub_vector_lengths_and_long_partitions_vs_oracle(m, dim):
    # dsub 32, 16, 8, 1 and 32; partitions longer than one 2048-row tile
    rng = np.random.default_rng(37 + m)
    ix = random_pq4_index(rng, n=9000, dim=dim, nlist=3, m=m, metric="l2", empty=(), with_vectors=False)
    gpu = _native.GpuIvfPq(ix)
    q = ivf_queries(rng, ix, 11, 1000.0)
    assert_same(gpu.search(q, k=50, nprobes=2), pq4_oracle.search(ix, q, k=50, nprobes=2), f"m={m}")
    gpu.close()


def test_ivf_pq4_ties_at_the_kth_place_and_row_major_layout():
    rng = np.random.default_rng(40)
    ix = random_pq4_index(rng, n=3000, dim=32, nlist=4, m=8, metric="l2", empty=())
    # partition 0: every row the same code bytes -> every distance equal, ordered by row id
    a, b = int(ix.part_offsets[0]), int(ix.part_offsets[1])
    w = ix.code_bytes
    ix.codes_t[a * w:b * w] = np.repeat(rng.integers(0, 256, w, dtype=np.uint8), b - a)
    q = ivf_queries(rng, ix, 16, 1000.0)
    want = pq4_oracle.search(ix, q, k=10, nprobes=4)
    gpu = _native.GpuIvfPq(ix)
    assert_same(gpu.search(q, k=10, nprobes=4), want, "transposed codes")
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
    assert_same(g2.search(q, k=10, nprobes=4), want, "row-major codes")
    g2.close()


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

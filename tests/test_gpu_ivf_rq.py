"""IVF_RQ on the GPU: the binary tensor-core scan kernel against NumPy integers and the oracle's estimates, and GpuIvfRq
against the C oracle (ids, counts and distance bits) over metrics, list counts, batch sizes, k, partition shapes,
awkward queries, prefilter, maximum_nprobes, distance_range, refine_factor and every search entry point; then
create_index through the builder."""
import ctypes as C
import threading

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests import rq_oracle
from tests.rq_oracle import random_rq_index, rq_estimates_np, rq_slot_np

pytestmark = pytest.mark.gpu
f32 = np.float32


def _same(got, want, what=""):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ"
    assert np.array_equal(gi, oi), f"{what}: ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distance bits differ"


@pytest.mark.parametrize("B,N,dim,metric", [(1, 1, 1, "l2"), (7, 300, 7, "cosine"), (8, 257, 255, "l2"),
                                            (9, 33, 256, "l2"), (13, 1000, 257, "cosine"), (33, 2000, 768, "l2"),
                                            (5, 4099, 1000, "cosine"), (3, 700, 4096, "l2")])
def test_debug_rq_distances_equal_numpy_and_oracle(B, N, dim, metric):
    rng = np.random.default_rng(B * 1000 + dim)
    q = rng.standard_normal((B, dim)).astype(f32)
    if B > 2:
        q[1] = 0.25                                       # delta = 0: every u is 0
        q[2, 0] = 1e30                                    # one huge component: the other u collapse to 0
    codes = rng.integers(0, 256, (N, (dim + 7) // 8), dtype=np.uint8)   # stray padding bits are cleared at open
    codes[: min(N, 2)] = 255
    add = (rng.random(N) * 10).astype(f32)
    scale = (-rng.random(N) * 3).astype(f32)
    est, ip = _native.debug_rq_distances(q, codes, add, scale, metric)
    zero = np.zeros(dim, f32)
    for b in range(B):
        u, lo, delta, qq, S = rq_slot_np(q[b], zero)
        want_ip = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, ip_only=True)
        assert np.array_equal(ip[b].astype(np.int64), want_ip), b
        want = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, metric)
        assert np.array_equal(est[b].view(np.uint32), want.view(np.uint32)), b
        if b < 2:                                         # the C oracle's own arithmetic on the first rows
            cu, clo, cdelta, cqq, cS = rq_oracle.rq_slot(q[b], zero)
            c = rq_oracle.rq_estimates(codes[:64], add[:64], scale[:64], cu, clo, cdelta, cqq, cS, dim, metric)
            assert np.array_equal(est[b, :64].view(np.uint32), c.view(np.uint32)), b


def test_debug_rq_distances_non_finite_slot_has_no_rows():
    dim, N = 40, 50
    rng = np.random.default_rng(3)
    q = rng.standard_normal((3, dim)).astype(f32)
    q[0, 4] = np.nan
    q[1, 5] = np.inf
    codes = rng.integers(0, 256, (N, 5), dtype=np.uint8)
    est, _ = _native.debug_rq_distances(q, codes, np.ones(N, f32), -np.ones(N, f32))
    assert np.isnan(est[:2]).all() and np.isfinite(est[2]).all()


def _queries(rng, ix, B):
    q = rng.standard_normal((B, ix.dim)).astype(f32)
    if B > 3:
        q[1] *= 1e4                                       # huge magnitude
        q[2, 0] = np.nan                                  # no finite centroid distance: no rows
        q[3] = ix.vectors[7]                              # an exact stored row (and its duplicates)
    return q


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_rq_small_lists_vs_oracle(metric):
    rng = np.random.default_rng(31 if metric == "l2" else 32)
    ix = random_rq_index(rng, n=6000, dim=40, nlist=16, metric=metric, empty=(2, 9))
    gpu = _native.GpuIvfRq(ix)
    for B in (1, 7, 8, 37):
        q = _queries(rng, ix, B)
        for k, nprobes in ((1, 3), (10, 5), (100, 16)):
            got = gpu.search(q, k=k, nprobes=nprobes)
            _same(got, rq_oracle.search(ix, q, k=k, nprobes=nprobes), f"B={B} k={k} nprobes={nprobes}")
            if B > 3:
                assert got[2][2] == 0
    gpu.close()
    # k > N, tiny and empty partitions, every partition probed
    tiny = random_rq_index(rng, n=150, dim=40, nlist=16, metric=metric, empty=(0, 3, 4))
    gpu = _native.GpuIvfRq(tiny)
    q = _queries(rng, tiny, 9)
    got = gpu.search(q, k=200, nprobes=16)
    _same(got, rq_oracle.search(tiny, q, k=200, nprobes=16), "k > N")
    assert got[2][0] == 150
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_rq_tensor_core_coarse_step_vs_oracle(metric):
    rng = np.random.default_rng(33 if metric == "l2" else 34)
    ix = random_rq_index(rng, n=60000, dim=128, nlist=1024, metric=metric, empty=(5, 77))
    gpu = _native.GpuIvfRq(ix)
    q = _queries(rng, ix, 1024)
    for k, nprobes in ((10, 20), (100, 8)):
        _same(gpu.search(q, k=k, nprobes=nprobes), rq_oracle.search(ix, q, k=k, nprobes=nprobes), f"k={k}")
    gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_rq_prefilter_range_refine_vs_oracle(metric):
    rng = np.random.default_rng(35 if metric == "l2" else 36)
    ix = random_rq_index(rng, n=8000, dim=300, nlist=32, metric=metric)
    gpu = _native.GpuIvfRq(ix)
    q = _queries(rng, ix, 40)
    nbits = ix.nrows * 3 + 7
    mask = rng.random(nbits) < 0.02                           # narrow: many queries need maximum_nprobes
    bm = _native.mask_bitmap(mask)
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits, max_nprobes=32)
    _same(got, rq_oracle.search(ix, q, k=10, nprobes=2, allow=mask, max_nprobes=32), "prefilter + maximum_nprobes")
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits)
    _same(got, rq_oracle.search(ix, q, k=10, nprobes=2, allow=mask), "prefilter")
    d = rq_oracle.search(ix, q[:1], k=50, nprobes=4)[1][0]
    lo, hi = float(d[5]), float(d[30])
    got = gpu.search(q, k=20, nprobes=4, lower=lo, upper=hi)
    _same(got, rq_oracle.search(ix, q, k=20, nprobes=4, lower=lo, upper=hi), "distance_range")
    got = gpu.search(q, k=7, nprobes=4, refine_factor=5)
    _same(got, rq_oracle.search(ix, q, k=7, nprobes=4, refine_factor=5), "refine_factor")
    gpu.close()


def test_ivf_rq_device_async_and_coalesced_entry_points(monkeypatch):
    import torch
    # the coalescing window is read once per process, at the first coalesced call: take the one
    # test_gpu_api.py's batching test needs, whichever of the two runs first
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")
    rng = np.random.default_rng(37)
    ix = random_rq_index(rng, n=5000, dim=100, nlist=24)
    gpu = _native.GpuIvfRq(ix)
    q = _queries(rng, ix, 19)
    want = rq_oracle.search(ix, q, k=9, nprobes=6)
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
    # codes padded to 256 bits, add / scale / popc, row ids, the rotation
    assert gpu.device_bytes() >= ix.nrows * (32 + 12 + 8) + 100 * 100 * 4
    _native.set_profiling(True)
    gpu.search(q, k=9, nprobes=6)
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    assert scanned > 0 and scanned % 32 == 0                 # dim 100 -> 256 bits = 32 bytes per row
    gpu.close()


def test_ivf_rq_rejections():
    rng = np.random.default_rng(38)
    ix = random_rq_index(rng, n=500, dim=16, nlist=4)
    gpu = _native.GpuIvfRq(ix)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_filter_bounds(ix.vectors[:2], 2, 10)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_partition_distances(ix.vectors[0], 0, 10)
    gpu.close()
    # the C ABI itself rejects dot, num_bits != 1, dimensions above 4096 and a missing rotation
    lib = _native.load()
    c = np.zeros((1, 16), f32); off = np.zeros(2, np.uint64); P = np.eye(16, dtype=f32)
    for metric, dim, bits, rot in ((2, 16, 1, P), (0, 16, 8, P), (0, 4097, 1, P), (0, 16, 1, None)):
        desc = _native.RqDesc(_native.ABI_VERSION, dim, 1, metric, 0, bits, 0, c.ctypes.data,
                              None if rot is None else rot.ctypes.data, off.ctypes.data, None, None, None, None, None)
        h = C.c_void_p()
        with pytest.raises(ValueError):
            _native.check(lib.lgpu_ivf_rq_open(C.byref(desc), C.byref(h)))


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_create_index_ivf_rq_search_to_arrow(metric):
    rng = np.random.default_rng(39)
    centers = rng.standard_normal((32, 64)).astype(f32) * 3
    x = (centers[rng.integers(0, 32, 5000)] + rng.standard_normal((5000, 64))).astype(f32)
    db = lancedb.connect("memory://")
    t = db.create_table("v", {"vector": x, "id": np.arange(5000)})
    t.create_index(metric=metric, num_partitions=16, index_type="IVF_RQ", num_bits=1, max_iterations=4,
                   accelerator="cuda")
    assert t.list_indices()[0]["index_type"] == "IVF_RQ"
    data = t._index_data["vector"]
    q = (x[:3] + 0.1 * rng.standard_normal((3, 64))).astype(f32)
    oi, od, oc = rq_oracle.search(data, q, k=12, nprobes=4)
    for i in range(3):
        out = t.search(q[i]).distance_type(metric).nprobes(4).limit(10).offset(2).with_row_id(True).to_arrow()
        assert out["_rowid"].to_pylist() == [int(v) for v in oi[i, 2:12]]
        assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32).view(np.uint32), od[i, 2:12].view(np.uint32))
    out = t.search(q[0]).distance_type(metric).nprobes(4).refine_factor(10).limit(5).to_arrow()
    rd = rq_oracle.search(data, q[:1], k=5, nprobes=4, refine_factor=10)[1]
    assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32), rd[0])
    # recall with refine against the exact flat search: loose, RQ is a refine-first index
    import oracle
    fi = oracle.flat_search(x, q, k=10, metric=metric)[0]
    gi = _native.GpuIvfRq.search(t._index["vector"], q, k=10, nprobes=16, refine_factor=10)[0]
    assert np.mean([len(set(fi[b]) & set(gi[b])) / 10 for b in range(3)]) >= 0.6

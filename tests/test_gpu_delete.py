"""Deleted rows on the GPU (lgpu_*_delete): every handle family, bit for bit against the existing oracles run with the
allow mask allow' = allow AND NOT deleted (no call mask: every id not deleted).

- Every IVF kind (8-bit PQ under l2 and cosine, 4-bit PQ, SQ, HNSW_SQ, RQ, binary IVF_FLAT) as deletions grow through
  0.1 %, 30 %, all rows but k and all rows: the host, filtered, device, async and coalesced routes, maximum_nprobes
  widening, and the union with a tail that has deletions of its own.
- Flat float under l2, cosine and dot (sparse row ids, both sides of 262144 rows, k above 2048), flat binary on both
  sides of the list path's sample, multivector.
- n_deleted counts and idempotence, delete / append / delete, a captured CUDA graph replayed after a delete, widening
  caused by deletions alone, deletes racing searches from threads, refusals, sub-batches under a small LGPU_WS_BYTES,
  and a Table end to end.
- The tensor-core paths under a row filter (flat L2 on both sides of 262144 rows, the binary list and dense paths):
  filters that drop the unfiltered top-k, a threshold sample with fewer than k allowed rows, adversarial bf16 rounding;
  each asserts the bits and that the tensor-core route ran."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import lancedb_b200 as lancedb
import oracle
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS
from tests import hamming_oracle, multivec_oracle, unindexed_oracle as U
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
DIM, NBYTES, NLIST, N, NT, B, K = 32, 8, 16, 4000, 600, 48, 10

KINDS = [
    ("IVF_PQ", dict(num_sub_vectors=8), "l2"),
    ("IVF_PQ", dict(num_sub_vectors=8), "cosine"),
    ("IVF_PQ", dict(num_sub_vectors=8, num_bits=4), "l2"),
    ("IVF_SQ", dict(), "l2"),
    ("IVF_HNSW_SQ", dict(m=6, ef_construction=40), "l2"),
    ("IVF_RQ", dict(num_bits=1), "cosine"),
    ("IVF_FLAT", dict(), "hamming"),
]


def _live(nbits, dead, allow=None):
    """allow' as a bool mask over row ids [0, nbits)"""
    m = np.ones(nbits, bool) if allow is None else allow.copy()
    m[np.asarray(sorted(dead), np.int64)] = False
    return m


def _steps(rng, ids, k):
    """cumulative deletion sets: 0.1 %, 30 %, all but k, all"""
    perm = rng.permutation(ids)
    n = len(ids)
    return [perm[:max(1, n // 1000)], perm[:(3 * n) // 10], perm[:n - k], perm]


def _device_search(h, q, p, B, k, binary=False):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((B, k), dtype=torch.int64, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    h.search_device(dq.data_ptr(), B, p, ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _train(kind, params, metric, rng):
    binary = kind == "IVF_FLAT"
    x = rng.integers(0, 256, (N, NBYTES)).astype(np.uint8) if binary else rng.standard_normal((N, DIM)).astype(f32)
    kw = {} if binary else dict(keep_vectors=True)
    d = IVF_KINDS[kind].train(x, num_partitions=NLIST, distance_type=metric, max_iterations=4, **kw, **params)
    h = getattr(_native, IVF_KINDS[kind].handle)(d, device=0)
    if binary:
        q = x[rng.integers(0, N, B)] ^ rng.integers(0, 2, (B, NBYTES)).astype(np.uint8)
        tail = rng.integers(0, 256, (NT, NBYTES)).astype(np.uint8)
        th = _native.GpuBinary(tail, row_ids=np.arange(N, N + NT, dtype=np.uint64))
    else:
        q = rng.standard_normal((B, DIM)).astype(f32)
        tail = rng.standard_normal((NT, DIM)).astype(f32)
        th = _native.GpuFlat(tail, row_ids=np.arange(N, N + NT, dtype=np.uint64))
    return d, h, q, tail, th


@pytest.mark.parametrize("kind,params,metric", KINDS, ids=[f"{k}-{m}-{p.get('num_bits', '')}" for k, p, m in KINDS])
def test_ivf_deletes_on_every_route(kind, params, metric):
    rng = np.random.default_rng(11)
    d, h, q, tail, th = _train(kind, params, metric, rng)
    binary = kind == "IVF_FLAT"
    tail_ids = np.arange(N, N + NT, dtype=np.uint64)
    call = rng.random(N + NT) < 0.6
    call_bm = _native.mask_bitmap(call)
    dead = set()
    for step, (di, dt) in enumerate(zip(_steps(rng, np.arange(N), K), _steps(rng, np.arange(N, N + NT), K))):
        new = set(int(i) for i in di) - dead
        # the call reports the ids it newly deleted: already-deleted and absent ids count for nothing
        assert h.delete(np.concatenate([di, [N + NT + 5, 10 ** 9]])) == len(new)
        assert h.delete(di) == 0
        assert th.delete(dt) == len(set(int(i) for i in dt) - dead)
        dead |= new | set(int(i) for i in dt)
        live = _live(N + NT, dead)
        for nprobes, max_np in ((4, 0), (2, NLIST)):
            what = f"step {step} nprobes {nprobes}/{max_np}"
            assert_same(h.search(q, k=K, nprobes=nprobes, max_nprobes=max_np),
                        U.index_search(d, q, K, nprobes, allow=live[:N], max_nprobes=max_np),
                        what + " host", prefix=True)
            assert_same(h.search(q, k=K, nprobes=nprobes, max_nprobes=max_np, allow=call_bm, allow_bits=N + NT),
                        U.index_search(d, q, K, nprobes, allow=live & call, max_nprobes=max_np),
                        what + " filtered", prefix=True)
            assert_same(h.search_unindexed(th, q, k=K, nprobes=nprobes, max_nprobes=max_np),
                        U.union_search(d, tail, tail_ids, q, K, nprobes, allow=live, max_nprobes=max_np),
                        what + " union", prefix=True)
            assert_same(h.search_unindexed(th, q, k=K, nprobes=nprobes, max_nprobes=max_np, allow=call_bm,
                                           allow_bits=N + NT),
                        U.union_search(d, tail, tail_ids, q, K, nprobes, allow=live & call, max_nprobes=max_np),
                        what + " union filtered", prefix=True)
        p = _native.make_params(K, 4, max_nprobes=NLIST)
        want = U.index_search(d, q, K, 4, allow=live[:N], max_nprobes=NLIST)
        assert_same(_device_search(h, q, p, B, K, binary), want, f"step {step} device", prefix=True)
        if binary:
            continue
        ids, dist, cnt = (np.empty((B, K), np.uint64), np.empty((B, K), f32), np.empty(B, np.uint32))
        _native.ticket_wait(h.search_async(q, p, ids, dist, cnt))
        assert_same((ids, dist, cnt), want, f"step {step} async", prefix=True)
        want = U.index_search(d, q[:3], K, 20, allow=live[:N])
        for i in range(3):
            gi, gd, gc = h.search_one(q[i], k=K, nprobes=20)
            assert_same((gi[None], gd[None], np.array([gc], np.uint32)),
                        (want[0][i:i + 1], want[1][i:i + 1], want[2][i:i + 1]), f"step {step} coalesced", prefix=True)
    assert dead == set(range(N + NT))
    h.close(); th.close()


def test_widening_matches_the_oracle_with_deletions():
    rng = np.random.default_rng(13)
    d, h, q, _, th = _train("IVF_SQ", {}, "l2", rng)
    gone = rng.permutation(N)[:int(N * 0.97)]
    h.delete(gone)
    live = _live(N, set(int(i) for i in gone))
    want = U.index_search(d, q, K, 1, allow=live, max_nprobes=NLIST)
    assert_same(h.search(q, k=K, nprobes=1, max_nprobes=NLIST), want, "widened", prefix=True)
    narrow = U.index_search(d, q, K, 1, allow=live)
    assert (want[2] > narrow[2]).any()
    h.close(); th.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_flat_float_deletes(metric):
    rng = np.random.default_rng(14)
    n, dim = 6000, 64
    x = rng.standard_normal((n, dim)).astype(f32)
    ids = (np.arange(n) * 3 + 7).astype(np.uint64)            # sparse ids: id_bound is above the row count
    q = rng.standard_normal((32, dim)).astype(f32)
    fl = _native.GpuFlat(x, row_ids=ids)
    nbits = int(ids.max()) + 1
    call = rng.random(nbits) < 0.5
    call_bm = _native.mask_bitmap(call)
    dead = set()
    for step, di in enumerate(_steps(rng, ids.astype(np.int64), K)):
        new = set(int(i) for i in di) - dead
        assert fl.delete(np.concatenate([di, di[:3], [8, 9]])) == len(new)     # 8 and 9 fall between the ids
        dead |= new
        live = _live(nbits, dead)
        for k in ((K, 2100) if step == 1 else (K,)):
            want = oracle.flat_search(x, q, k, metric=metric, row_ids=ids, nthreads=0, allow=live)
            assert_same(fl.search(q, k=k, metric=metric), want, f"{metric} step {step} k {k}", prefix=True)
        assert_same(fl.search(q, k=K, metric=metric, allow=call_bm, allow_bits=nbits),
                    oracle.flat_search(x, q, K, metric=metric, row_ids=ids, nthreads=0, allow=live & call),
                    f"{metric} step {step} filtered", prefix=True)
        p = _native.make_params(K, 0)
        import torch
        dq = torch.from_numpy(q).cuda()
        o = [torch.empty((32, K), dtype=t, device="cuda") for t in (torch.int64, torch.float32)]
        c = torch.empty(32, dtype=torch.int32, device="cuda")
        fl.search_device(metric, dq.data_ptr(), 32, p, o[0].data_ptr(), o[1].data_ptr(), c.data_ptr(),
                         torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert_same((o[0].cpu().numpy().view(np.uint64), o[1].cpu().numpy(), c.cpu().numpy().view(np.uint32)),
                    oracle.flat_search(x, q, K, metric=metric, row_ids=ids, nthreads=0, allow=live),
                    f"{metric} device", prefix=True)
    fl.close()


def test_flat_l2_above_the_large_shortlist_threshold():
    rng = np.random.default_rng(15)
    n, dim = 270000, 32
    x = rng.standard_normal((n, dim)).astype(f32)
    q = rng.standard_normal((16, dim)).astype(f32)
    fl = _native.GpuFlat(x)
    unfiltered = oracle.flat_search(x, q, K, nthreads=0)
    gone = np.unique(unfiltered[0][:, :K // 2].astype(np.int64))      # the unfiltered top-k loses half its rows
    gone = np.concatenate([gone, rng.permutation(n)[:n // 3]])
    fl.delete(gone)
    live = _live(n, set(int(i) for i in gone))
    assert_same(fl.search(q, k=K), oracle.flat_search(x, q, K, nthreads=0, allow=live), "large N", prefix=True)
    fl.close()


@pytest.mark.parametrize("n", [5000, 70000])
def test_flat_binary_deletes(n):
    rng = np.random.default_rng(16)
    x = rng.integers(0, 256, (n, 32)).astype(np.uint8)
    q = x[rng.integers(0, n, 24)]
    bx = _native.GpuBinary(x)
    call = rng.random(n) < 0.5
    dead = set()
    for step, di in enumerate(_steps(rng, np.arange(n), K)):
        new = set(int(i) for i in di) - dead
        assert bx.delete(di) == len(new)
        dead |= new
        live = _live(n, dead)
        assert_same(bx.search(q, k=K), hamming_oracle.flat_search_u8(x, q, K, allow=live),
                    f"binary {n} step {step}", prefix=True)
        assert_same(bx.search(q, k=K, allow=_native.mask_bitmap(call), allow_bits=n),
                    hamming_oracle.flat_search_u8(x, q, K, allow=live & call),
                    f"binary {n} step {step} filtered", prefix=True)
        assert_same(_device_search(bx, q, _native.make_params(K, 0), 24, K, True),
                    hamming_oracle.flat_search_u8(x, q, K, allow=live), f"binary {n} step {step} device", prefix=True)
    bx.close()


def test_multivector_deletes():
    rng = np.random.default_rng(17)
    lens = rng.integers(0, 6, 3000)
    off = multivec_oracle.offsets_of(lens)
    x = rng.standard_normal((int(off[-1]), 16)).astype(f32)
    qoff = multivec_oracle.offsets_of([1, 3, 5, 2])
    q = rng.standard_normal((int(qoff[-1]), 16)).astype(f32)
    mv = _native.GpuMultivec(x, off)
    dead = set()
    for step, di in enumerate(_steps(rng, np.arange(3000), K)):
        dead |= set(int(i) for i in di)
        mv.delete(di)
        live = _live(3000, dead)
        assert_same(mv.search(q, k=K, q_offsets=qoff),
                    multivec_oracle.flat_search_mv(x, off, q, qoff, K, allow=live),
                    f"multivector step {step}", prefix=True)
    mv.close()


@pytest.mark.parametrize("binary", [False, True])
def test_delete_append_delete(binary):
    rng = np.random.default_rng(18)
    rows = (lambda n: rng.integers(0, 256, (n, 32)).astype(np.uint8)) if binary else \
        (lambda n: rng.standard_normal((n, 64)).astype(f32))
    x0, x1 = rows(5000), rows(3000)
    h = (_native.GpuBinary if binary else _native.GpuFlat)(x0)
    assert h.delete(np.arange(0, 5000, 3)) == 1667
    assert h.delete([7500]) == 0                       # not held yet: nothing is recorded against it
    h.append(x1, np.arange(5000, 8000, dtype=np.uint64))
    assert h.delete(np.arange(4990, 5010)) == 20 - 3   # 4992, 4995 and 4998 were deleted already
    allx = np.concatenate([x0, x1])
    live = _live(8000, set(range(0, 5000, 3)) | set(range(4990, 5010)))
    q = allx[rng.integers(0, 8000, 16)]
    if binary:
        want = hamming_oracle.flat_search_u8(allx, q, K, allow=live)
    else:
        want = oracle.flat_search(allx, q, K, nthreads=0, allow=live)
    assert live[7500]
    assert_same(h.search(q, k=K), want, "after delete / append / delete", prefix=True)
    h.close()


def test_graph_replay_after_delete():
    rng = np.random.default_rng(19)
    x = rng.standard_normal((5000, 64)).astype(f32)
    q = rng.standard_normal((16, 64)).astype(f32)
    fl = _native.GpuFlat(x)
    for _ in range(3):                                      # eager, capture, replay
        assert_same(fl.search(q, k=K), oracle.flat_search(x, q, K, nthreads=0), "before", prefix=True)
    gone = np.unique(oracle.flat_search(x, q, 3, nthreads=0)[0].astype(np.int64))
    fl.delete(gone)
    live = _live(5000, set(int(i) for i in gone))
    for _ in range(3):                                      # the graph captured without a filter is not replayed
        assert_same(fl.search(q, k=K), oracle.flat_search(x, q, K, nthreads=0, allow=live), "after", prefix=True)
    fl.close()
    d, h, q, _, th = _train("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    for _ in range(3):
        assert_same(h.search(q, k=K, nprobes=4), U.index_search(d, q, K, 4), "ivf before", prefix=True)
    gone = np.unique(h.search(q, k=2, nprobes=4)[0].astype(np.int64))
    h.delete(gone)
    live = _live(N, set(int(i) for i in gone))
    for _ in range(3):
        assert_same(h.search(q, k=K, nprobes=4), U.index_search(d, q, K, 4, allow=live), "ivf after", prefix=True)
    h.close(); th.close()


def test_deletes_racing_searches():
    rng = np.random.default_rng(20)
    d, h, q, _, th = _train("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    gone = rng.permutation(N)[:N // 2]
    before = U.index_search(d, q, K, 4)
    after = U.index_search(d, q, K, 4, allow=_live(N, set(int(i) for i in gone)))
    results, errors = [], []

    def searcher():
        try:
            for _ in range(30):
                results.append(h.search(q, k=K, nprobes=4))
        except Exception as e:              # noqa: BLE001 -- reported below
            errors.append(e)

    ts = [threading.Thread(target=searcher) for _ in range(3)]
    for t in ts:
        t.start()
    h.delete(gone)
    for t in ts:
        t.join()
    assert not errors
    for r in results:
        bits = lambda a: (a[0].tobytes(), a[1].view(np.uint32).tobytes(), np.asarray(a[2], np.uint32).tobytes())
        assert bits(r) in (bits(before), bits(after))
    h.close(); th.close()


def test_delete_refusals():
    lib = _native.load()
    x = np.zeros((10, 8), f32)
    fl = _native.GpuFlat(x, row_ids=np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 1 << 33], np.uint64))
    with pytest.raises(ValueError, match="LGPU_DELETE_ID_BOUND"):
        fl.delete([1])
    bx = _native.GpuBinary(np.zeros((4, 8), np.uint8))
    import ctypes as C
    n = C.c_uint64(0)
    ids = np.array([1], np.uint64)
    assert lib.lgpu_flat_delete(bx._h, _native._ptr(ids), 1, C.byref(n)) == _native.LGPU_INVALID_INPUT
    assert b"flat handle expected, got a binary handle" in lib.lgpu_last_error()
    assert bx.delete([]) == 0 and bx.delete([1]) == 1
    fl.close(); bx.close()


# ---- the tensor-core paths under a row filter: the shortlist, the sample's threshold and the filtering pass work on
# the allowed rows only, so deleted rows and prefilters keep the flat float (L2) and binary searches on the tensor cores.
# Each case asserts the bits and that the tensor-core route ran.
def _tc_flat_case(x, q, gone, call=None, ids=None):
    fl = _native.GpuFlat(x, row_ids=ids)
    nbits = len(x) if ids is None else int(ids.max()) + 1
    fl.delete(gone)
    live = _live(nbits, set(int(i) for i in gone))
    kw = {} if call is None else dict(allow=_native.mask_bitmap(call), allow_bits=nbits)
    _native.set_profiling(True)
    try:
        got = fl.search(q, k=K, **kw)
        st = _native.last_filter_stats()
    finally:
        _native.set_profiling(False)
    fl.close()
    want = oracle.flat_search(x, q, K, row_ids=ids, nthreads=0, allow=live if call is None else live & call)
    assert_same(got, want, "tensor-core flat under a filter", prefix=True)
    # [1]: distances the tensor cores computed, every row for every query on the tensor-core route, none on the exact one
    assert st["rescored"] == len(q) * len(x) and st["queries"] == len(q), f"the exact route ran: {st}"
    return got


@pytest.mark.parametrize("n", [6000, 270000])
def test_tensor_core_flat_l2_under_a_filter(n):
    rng = np.random.default_rng(30)
    x = rng.standard_normal((n, 64)).astype(f32)
    q = rng.standard_normal((32, 64)).astype(f32)
    q[0] = x[11]
    top = oracle.flat_search(x, q, K, nthreads=0)[0].astype(np.int64)
    gone = np.concatenate([np.unique(top.reshape(-1)), rng.permutation(n)[:n // 10]])    # the unfiltered top-k goes
    _tc_flat_case(x, q, gone)
    call = rng.random(n) < 0.5
    _tc_flat_case(x, q, gone[:50], call=call)
    ids = rng.permutation(n).astype(np.uint64) * 2 + 1
    _tc_flat_case(x, q, ids[top[:, :3].reshape(-1)].astype(np.int64), ids=ids)


def test_tensor_core_flat_l2_sample_with_fewer_than_k_allowed_rows():
    """N >= 262144: the threshold sample is the first 65536 rows; with k - 1 of them left, every query's threshold is
    +inf, its list overflows and the exact fix-up answers it"""
    rng = np.random.default_rng(31)
    n = 270000
    x = rng.standard_normal((n, 32)).astype(f32)
    q = rng.standard_normal((16, 32)).astype(f32)
    gone = np.setdiff1d(np.arange(65536), rng.permutation(65536)[:K - 1])
    _tc_flat_case(x, q, gone)


@pytest.mark.parametrize("n", [4096, 262144])
def test_tensor_core_flat_adversarial_rounding_under_a_filter(n):
    """split_support_case (tests/test_gpu_tensorcore.py): the true nearest row is scored too high and k decoys too low;
    deleting some decoys and rows around them must leave the result bit-exact on the tensor-core route"""
    from tests.util import split_support_case
    q, X = split_support_case(64, 1.0, n, 10)
    Q = np.tile(q, (8, 1))
    top = oracle.flat_search(X, Q[:1], 2 * K, nthreads=0)[0][0].astype(np.int64)
    for gone in (top[1:K:2], top[:1], np.arange(0, n, 7)):
        _tc_flat_case(X, Q, gone)


@pytest.mark.parametrize("n,B,with_ids", [(70000, 16, False), (70000, 24, True), (8192, 128, False)])
def test_tensor_core_binary_under_a_filter(n, B, with_ids):
    """N > 65536: the list path (sample rows are every stride-th row: deleting them moves the threshold); N <= 65536
    with B >= 128: the dense wgmma path"""
    rng = np.random.default_rng(32)
    x = rng.integers(0, 256, (n, 32)).astype(np.uint8)
    q = x[rng.integers(0, n, B)] ^ (rng.random((B, 32)) < 0.05).astype(np.uint8)
    ids = (rng.permutation(n).astype(np.uint64) * 3 + 2) if with_ids else None
    bx = _native.GpuBinary(x, row_ids=ids)
    nbits = n if ids is None else int(ids.max()) + 1
    rid = np.arange(n) if ids is None else ids.astype(np.int64)
    top = hamming_oracle.flat_search_u8(x, q, K, row_ids=ids)[0].astype(np.int64)
    sample = rid[::n // 65536][:30000] if n > 65536 else rid[:0]      # most of the list path's threshold sample
    gone = np.unique(np.concatenate([top[:, :3].reshape(-1), sample, rid[rng.permutation(n)[:n // 5]]]))
    bx.delete(gone)
    live = _live(nbits, set(int(i) for i in gone))
    call = rng.random(nbits) < 0.7
    for allow, kw in ((live, {}), (live & call, dict(allow=_native.mask_bitmap(call), allow_bits=nbits))):
        _native.set_profiling(True)
        try:
            got = bx.search(q, k=K, **kw)
            st = _native.last_filter_stats()
        finally:
            _native.set_profiling(False)
        assert_same(got, hamming_oracle.flat_search_u8(x, q, K, row_ids=ids, allow=allow), f"binary {n}", prefix=True)
        assert st["rescored"] > 0, "the binary search did not run on the tensor cores"
    bx.close()


def test_table_end_to_end():
    rng = np.random.default_rng(21)
    x = rng.standard_normal((N, DIM)).astype(f32)
    t = lancedb.connect().create_table("t", {"id": np.arange(N), "grp": np.arange(N) % 3, "vector": x})
    t.create_index(metric="l2", num_partitions=NLIST, num_sub_vectors=8, max_iterations=4)
    t.add({"id": np.arange(N, N + 200), "grp": np.arange(N, N + 200) % 3,
           "vector": rng.standard_normal((200, DIM)).astype(f32)})
    q = x[5]
    assert t.delete("grp = 0").num_deleted_rows == len(range(0, N + 200, 3))
    got = t.search(q).nprobes(4).limit(20).with_row_id(True).to_arrow()
    assert all(r % 3 for r in got["_rowid"].to_pylist()) and got["id"].to_pylist() == got["_rowid"].to_pylist()
    flat = t.search(q).bypass_vector_index().limit(20).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    live = np.arange(N + 200) % 3 != 0
    want = oracle.flat_search(t._data.column("vector").combine_chunks().flatten().to_numpy().reshape(-1, DIM), q, 20,
                              nthreads=0, allow=live)
    assert flat == want[0][0, :want[2][0]].tolist()
    t.optimize()
    assert t.index_stats("vector_idx")["num_indexed_rows"] == int(live.sum())
    again = t.search(q).nprobes(4).limit(20).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert all(r % 3 for r in again)


def test_append_may_not_undelete():
    """An appended row may not take the id of a deleted row the handle holds (its bit would bring that row back); an
    id between the held ones, or above them, is fine.  A refused append changes nothing."""
    rng = np.random.default_rng(23)
    for binary in (False, True):
        rows = (lambda n: rng.integers(0, 256, (n, 32)).astype(np.uint8)) if binary else \
            (lambda n: rng.standard_normal((n, 64)).astype(f32))
        x = rows(5000)
        ids = np.arange(5000, dtype=np.uint64) * 2                     # even ids: odd ones below 9998 name no row
        h = (_native.GpuBinary if binary else _native.GpuFlat)(x, row_ids=ids)
        assert h.delete([10, 12]) == 2
        extra = rows(2)
        with pytest.raises(ValueError, match="undelete"):
            h.append(extra, np.array([20001, 12], np.uint64))
        with pytest.raises(ValueError, match="undelete"):
            h.append(extra[:1], np.array([10], np.uint64))
        assert h.nrows == 5000
        q = x[rng.integers(0, 5000, 16)]
        search = (lambda xx, qq, k, **kw: hamming_oracle.flat_search_u8(xx, qq, k, **kw)) if binary else \
            (lambda xx, qq, k, **kw: oracle.flat_search(xx, qq, k, nthreads=0, **kw))
        assert_same(h.search(q, k=K), search(x, q, K, row_ids=ids), "after a refused append", prefix=True)
        h.append(extra, np.array([11, 20001], np.uint64))               # a gap below id_bound, and a new id above it
        allx, allid = np.concatenate([x, extra]), np.concatenate([ids, [11, 20001]]).astype(np.uint64)
        keep = ~np.isin(allid, [10, 12])
        assert_same(h.search(q, k=K), search(allx[keep], q, K, row_ids=allid[keep]),
                    "after an allowed append", prefix=True)
        h.close()


def _sub_batch_child():
    """Run in a child with a small LGPU_WS_BYTES, which splits these batches into sub-batches: deletions (and their AND
    with a call bitmap, made once per call) against the oracle."""
    rng = np.random.default_rng(22)
    x = rng.standard_normal((6000, 64)).astype(f32)
    q = rng.standard_normal((128, 64)).astype(f32)
    fl = _native.GpuFlat(x)
    gone = rng.permutation(6000)[:2000]
    fl.delete(gone)
    live = _live(6000, set(int(i) for i in gone))
    call = rng.random(6000) < 0.5
    assert_same(fl.search(q, k=K), oracle.flat_search(x, q, K, nthreads=0, allow=live), "flat split", prefix=True)
    assert_same(fl.search(q, k=K, allow=_native.mask_bitmap(call), allow_bits=6000),
                oracle.flat_search(x, q, K, nthreads=0, allow=live & call), "flat split filtered", prefix=True)
    d, h, _, tail, th = _train("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    qi = rng.standard_normal((1024, DIM)).astype(f32)
    gone = np.concatenate([rng.permutation(N)[:N // 2], np.arange(N, N + NT, 2)])
    h.delete(gone[gone < N]); th.delete(gone[gone >= N])
    live = _live(N + NT, set(int(i) for i in gone))
    assert h.debug_sub_batch_size(1024, 4) < 1024
    assert_same(h.search(qi, k=K, nprobes=4, max_nprobes=NLIST),
                U.index_search(d, qi, K, 4, allow=live[:N], max_nprobes=NLIST), "ivf split", prefix=True)
    assert_same(h.search_unindexed(th, qi, k=K, nprobes=4),
                U.union_search(d, tail, np.arange(N, N + NT, dtype=np.uint64),
                                                                            qi, K, 4, allow=live),
                "union split", prefix=True)
    print("ok")


def _charge_child():
    """Run in a child with LGPU_WS_BYTES = 8 MiB: the AND of a call bitmap with the live rows (3.7 MiB here) is charged
    to the budget, so the filtered call splits its batch into more sub-batches than the same search without a call
    bitmap (whose filter is the live bitmap itself, outside the workspace), and both equal the oracle."""
    rng = np.random.default_rng(24)
    n, B = 6000, 512
    x = rng.standard_normal((n, 64)).astype(f32)
    q = rng.standard_normal((B, 64)).astype(f32)
    ids = (np.arange(n) * 5000).astype(np.uint64)         # id_bound ~ 3e7 bits
    fl = _native.GpuFlat(x, row_ids=ids)
    fl.delete(ids[::3])
    nbits = int(ids.max()) + 1
    live = np.zeros(nbits, bool)
    live[ids.astype(np.int64)] = True
    live[ids[::3].astype(np.int64)] = False
    call = np.ones(nbits, bool)
    n0 = _native.kernel_launch_count()
    got = fl.search(q, k=K, timeout_ms=60000)          # (a deadline keeps the call eager: every launch is counted)
    plain = _native.kernel_launch_count() - n0
    assert_same(got, oracle.flat_search(x, q, K, row_ids=ids, nthreads=0, allow=live), "live bitmap only", prefix=True)
    n0 = _native.kernel_launch_count()
    got = fl.search(q, k=K, allow=_native.mask_bitmap(call), allow_bits=nbits)
    filtered = _native.kernel_launch_count() - n0
    assert_same(got, oracle.flat_search(x, q, K, row_ids=ids, nthreads=0, allow=live & call),
                "with a call bitmap", prefix=True)
    # 24 000 bytes per query: 2 sub-batches in 8 MiB, 3 once the 3.7 MiB bitmap is charged (plus the AND launch)
    assert filtered > plain + 1, (plain, filtered)
    print("ok")


def _child(mode, budget):
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(budget))
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_delete", mode], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_sub_batches_under_a_small_workspace():
    _child("split", 1 << 20)


def test_the_and_bitmap_is_charged_to_the_workspace_budget():
    _child("charge", 8 << 20)


if __name__ == "__main__":
    {"split": _sub_batch_child, "charge": _charge_child}[sys.argv[1]]()

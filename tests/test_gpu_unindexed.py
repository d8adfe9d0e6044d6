"""Rows added after an index was built (Table.add), on the GPU: every IVF kind's union search -- the index's result
merged with the exact top-k of the unindexed tail -- bit for bit against the union oracle (tests/unindexed_oracle.py)
as the tail grows across the tensor-core threshold, at k = 10, 2049 and above every row, with refine_factor,
distance_range, prefilters that admit only tail rows or only indexed rows, non-finite tail rows, the device route;
fast_search against the index-only oracle; optimize() against the oracle over the extended index.  Then appended
GpuFlat / GpuBinary handles against the same handles opened on the concatenated rows."""
import sys

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests import hamming_oracle, unindexed_oracle as U
from tests.util import assert_same

pytestmark = pytest.mark.gpu
f32 = np.float32
DIM, NBYTES, NLIST, N0, B = 32, 8, 8, 3000, 64

# kind, create_index arguments, metric
KINDS = [
    ("IVF_PQ", dict(num_sub_vectors=8), "l2"),
    ("IVF_PQ", dict(num_sub_vectors=8), "cosine"),
    ("IVF_PQ", dict(num_sub_vectors=8, num_bits=4), "l2"),
    ("IVF_SQ", dict(), "l2"),
    ("IVF_HNSW_SQ", dict(m=6, ef_construction=40), "l2"),
    ("IVF_RQ", dict(num_bits=1), "cosine"),
    ("IVF_FLAT", dict(), "hamming"),
]


def _rows(rng, kind, n):
    if kind == "IVF_FLAT":
        return rng.integers(0, 256, (n, NBYTES)).astype(np.uint8)
    return rng.standard_normal((n, DIM)).astype(f32)


def _table(kind, params, metric, rng):
    x = _rows(rng, kind, N0)
    db = lancedb.connect()
    if kind == "IVF_FLAT":
        t = db.create_table("t", {"vector": x}, schema=pa.schema([pa.field("vector", pa.list_(pa.uint8(), NBYTES))]))
    else:
        t = db.create_table("t", {"vector": x})
    t.create_index(metric=metric, num_partitions=NLIST, index_type=kind, max_iterations=4, **params)
    return t


def _search(t, q, **kw):
    args = dict(column="vector", k=10, nprobes=3, refine_factor=None, distance_type=None, lower=None, upper=None,
                use_index=True)
    args.update(kw)
    return t._vector_search(q, **args)


def _tail(t):
    n0 = t._tail_from["vector"]
    return t._new_rows("vector", n0), np.arange(n0, t.count_rows(), dtype=np.uint64)


def _check(t, q, what, k=10, nprobes=3, refine_factor=0, lower=None, upper=None, mask=None, max_nprobes=0):
    tail, tid = _tail(t)
    got = _search(t, q, k=k, nprobes=nprobes, refine_factor=refine_factor or None, lower=lower, upper=upper,
                  allow_mask=mask, max_nprobes=max_nprobes)
    want = U.union_search(t._index_data["vector"], tail, tid, q, k, nprobes, refine_factor, lower, upper, mask,
                          max_nprobes if mask is not None else 0)
    assert_same(got, want, what, prefix=True)


@pytest.mark.parametrize("kind,params,metric", KINDS, ids=[f"{k}-{m}-{p.get('num_bits', '')}" for k, p, m in KINDS])
def test_union_search_matches_the_oracle_as_the_tail_grows(kind, params, metric):
    rng = np.random.default_rng(sum(map(ord, kind + metric)) + 7 * len(params))
    t = _table(kind, params, metric, rng)
    q = _rows(rng, kind, B)
    index_only = _search(t, q)
    t.add({"vector": _rows(rng, kind, 0)})                # nothing added: no tail, today's call
    assert "vector" not in t._tail
    assert_same(_search(t, q), index_only, "empty add", prefix=True)
    for n, what in ((1, "1"), (4094, "4095"), (1, "4096"), (15904, "20000")):
        t.add({"vector": _rows(rng, kind, n)})
        _check(t, q, f"tail {what}")
    assert t.index_stats("vector_idx")["num_unindexed_rows"] == 20000
    # fast_search: the index alone, exactly today's call
    data = t._index_data["vector"]
    assert_same(_search(t, q, fast_search=True), U.index_search(data, q, 10, 3), "fast_search", prefix=True)
    big_k = kind != "IVF_HNSW_SQ"                         # IVF_HNSW_SQ keeps k x refine_factor <= 2048
    if big_k:
        _check(t, q, "k 2049", k=2049)
        _check(t, q[:3], "k above every row", k=N0 + 20000 + 5, nprobes=NLIST)
    if kind != "IVF_FLAT":
        _check(t, q, "refine", refine_factor=3)
        d = U.tail_search(data, *_tail(t), q[:1], 50)[1][0]
        _check(t, q, "distance_range", lower=float(d[5]), upper=float(d[40]))
    else:
        _check(t, q, "distance_range", lower=20.0, upper=28.0)
    n = t.count_rows()
    tail_only = np.arange(n) >= N0
    _check(t, q, "prefilter: tail rows only", mask=tail_only & (np.arange(n) % 3 == 0), max_nprobes=NLIST)
    _check(t, q, "prefilter: indexed rows only", mask=~tail_only, max_nprobes=NLIST)
    # the device route, with a device bitmap
    import torch
    mask = np.arange(n) % 2 == 0
    bm = torch.from_numpy(_native.mask_bitmap(mask).view(np.int32).copy()).cuda()
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((B, 10), dtype=torch.int64, device="cuda")
    dist = torch.empty((B, 10), dtype=torch.float32, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    p = _native.make_params(10, 3)
    t._index["vector"].search_unindexed_device(t._tail["vector"], dq.data_ptr(), B, p, bm.data_ptr(), n,
                                               ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = (ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32))
    tail, tid = _tail(t)
    assert_same(got, U.union_search(data, tail, tid, q, 10, 3, allow=mask), "device route", prefix=True)
    # optimize: the tail is folded into the index without retraining
    t.optimize()
    st = t.index_stats("vector_idx")
    assert (st["num_indexed_rows"], st["num_unindexed_rows"]) == (n, 0) and "vector" not in t._tail
    ext = t._index_data["vector"]
    assert np.array_equal(np.sort(ext.row_ids), np.arange(n, dtype=np.uint64))
    assert_same(_search(t, q), U.index_search(ext, q, 10, 3), "after optimize", prefix=True)
    if big_k:
        assert_same(_search(t, q, k=2049, nprobes=5), U.index_search(ext, q, 2049, 5),
                    "after optimize, k 2049", prefix=True)


def test_union_with_non_finite_tail_rows():
    # Table.add refuses such rows (on_bad_vectors="error"); the library's union serves a tail that holds them
    rng = np.random.default_rng(5)
    t = _table("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    tail = _rows(rng, "IVF_PQ", 5000)
    tail[3, 0] = np.nan
    tail[10, 4] = np.inf
    tail[11] = -np.inf
    tail[12, 1] = 3e38
    with pytest.raises(ValueError, match="NaN"):
        t.add({"vector": tail})
    assert t.count_rows() == N0 and "vector" not in t._tail
    ids = np.arange(N0, N0 + 5000, dtype=np.uint64)
    fl = _native.GpuFlat(tail, row_ids=ids)
    q = _rows(rng, "IVF_PQ", B)
    q[0] = tail[12]
    data, ix = t._index_data["vector"], t._index["vector"]
    for k in (10, 2049):
        assert_same(ix.search_unindexed(fl, q, k=k, nprobes=3), U.union_search(data, tail, ids, q, k, 3),
                    f"non-finite tail, k {k}", prefix=True)
    fl.close()


def test_host_union_honours_timeout_ms():
    rng = np.random.default_rng(6)
    t = _table("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    ix = t._index["vector"]
    n = 300_000
    fl = _native.GpuFlat(_rows(rng, "IVF_PQ", n), row_ids=np.arange(N0, N0 + n, dtype=np.uint64))
    bm = _native.mask_bitmap(np.ones(N0 + n, bool))
    q = _rows(rng, "IVF_PQ", 4096)
    want = ix.search_unindexed(fl, q[:256], k=10, nprobes=3, allow=bm, allow_bits=N0 + n)
    assert_same(ix.search_unindexed(fl, q[:256], k=10, nprobes=3, allow=bm, allow_bits=N0 + n, timeout_ms=60000), want,
                "generous timeout", prefix=True)
    with pytest.raises(TimeoutError, match="timeout"):       # 4096 x 300k exact distances cannot finish in 1 ms
        ix.search_unindexed(fl, q, k=10, nprobes=3, allow=bm, allow_bits=N0 + n, timeout_ms=1)
    assert_same(ix.search_unindexed(fl, q[:256], k=10, nprobes=3, allow=bm, allow_bits=N0 + n), want,
                "after the timeout", prefix=True)
    fl.close()


def _sub_batch_child():
    """Run in a process of its own under a 1 MiB LGPU_WS_BYTES: the tail's scan splits the batch into sub-batches."""
    for kind, params, metric in (KINDS[0], KINDS[3], KINDS[6]):
        rng = np.random.default_rng(len(kind))
        t = _table(kind, params, metric, rng)
        t.add({"vector": _rows(rng, kind, 20000)})
        q = _rows(rng, kind, B)         # the tail's scan needs 20000 x 4 bytes a query: at most 13 of them a sub-batch
        for k in (10, 2049):
            _check(t, q, f"{kind} sub-batches, k {k}", k=k)
        _check(t, q, f"{kind} sub-batches, prefilter", mask=np.arange(t.count_rows()) % 2 == 1, max_nprobes=NLIST)
    print("sub-batches ok")


def test_union_when_the_workspace_budget_splits_the_batch():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, LGPU_WS_BYTES=str(1 << 20))
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_unindexed", "sub_batches"], cwd=root, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "sub-batches ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_builder_surface_routes_the_union():
    rng = np.random.default_rng(8)
    t = _table("IVF_PQ", dict(num_sub_vectors=8), "l2", rng)
    extra = _rows(rng, "IVF_PQ", 200)
    t.add({"vector": extra})
    q = extra[17]
    row = t.search(q).limit(1).with_row_id(True).to_arrow()
    assert row["_rowid"][0].as_py() == N0 + 17 and row["_distance"][0].as_py() == 0.0
    fast = t.search(q).limit(1).fast_search().with_row_id(True).to_arrow()
    assert fast["_rowid"][0].as_py() < N0
    flat = t.search(q).limit(1).bypass_vector_index().with_row_id(True).to_arrow()
    assert flat["_rowid"][0].as_py() == N0 + 17


def _flat_case(rng, n, metric_rows=DIM):
    x = rng.standard_normal((n, metric_rows)).astype(f32)
    return x, rng.permutation(np.arange(10, 10 + n, dtype=np.uint64) * 3)


# (cuts, a NaN row at n // 2): all-finite rows keep the tensor-core operand, which the appends then extend
@pytest.mark.parametrize("cuts,nan", [((100, 3996, 904), True), ((4096, 1, 6000), True), ((4096, 1, 6000), False),
                                      ((100, 3996, 904), False), ((1, 1, 1), False)])
def test_appended_flat_equals_flat_opened_on_the_concatenation(cuts, nan):
    import oracle
    rng = np.random.default_rng(sum(cuts))
    n = sum(cuts)
    x, ids = _flat_case(rng, n)
    if nan:
        x[n // 2, 3] = np.nan
    q = rng.standard_normal((16, DIM)).astype(f32)
    whole = _native.GpuFlat(x, row_ids=ids)
    grown = _native.GpuFlat(x[:cuts[0]], row_ids=ids[:cuts[0]])
    for _ in range(3):                                   # eager, captured, replayed: graphs bake the buffers in
        grown.search(q, k=10)
    a = cuts[0]
    for c in cuts[1:]:
        grown.append(x[a:a + c], ids[a:a + c])
        a += c
    mask = np.zeros(int(ids.max()) + 1, bool)
    mask[ids[::3].astype(np.int64)] = True
    bm = _native.mask_bitmap(mask)
    for metric in ("l2", "cosine", "dot"):
        for k in (10, 2049):
            assert_same(grown.search(q, k=k, metric=metric), whole.search(q, k=k, metric=metric),
                        f"{metric} k {k}", prefix=True)
        assert_same(grown.search(q, k=10, metric=metric, allow=bm, allow_bits=mask.size),
                    whole.search(q, k=10, metric=metric, allow=bm, allow_bits=mask.size),
                    f"{metric} filtered", prefix=True)
    assert_same(grown.search(q, k=10), oracle.flat_search(x, q, k=10, row_ids=ids, nthreads=0),
                "l2 oracle", prefix=True)
    # positions continue when no ids are given
    pos = _native.GpuFlat(x[:7])
    pos.append(x[7:n])
    assert_same(pos.search(q, k=10), _native.GpuFlat(x).search(q, k=10), "positions", prefix=True)


@pytest.mark.parametrize("cuts", [(100, 65436, 5000), (70000, 3)])
def test_appended_binary_equals_binary_opened_on_the_concatenation(cuts):
    rng = np.random.default_rng(sum(cuts))
    n = sum(cuts)
    x = rng.integers(0, 256, (n, NBYTES)).astype(np.uint8)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    q = rng.integers(0, 256, (256, NBYTES)).astype(np.uint8)
    whole = _native.GpuBinary(x, row_ids=ids)
    grown = _native.GpuBinary(x[:cuts[0]], row_ids=ids[:cuts[0]])
    for _ in range(3):
        grown.search(q, k=10)
    a = cuts[0]
    for c in cuts[1:]:
        grown.append(x[a:a + c], ids[a:a + c])
        a += c
    for k in (10, 2049):
        got = grown.search(q, k=k)
        assert_same(got, whole.search(q, k=k), f"k {k}", prefix=True)
        assert_same(got, hamming_oracle.flat_search_u8(x, q, k, row_ids=ids), f"oracle k {k}", prefix=True)


if __name__ == "__main__" and sys.argv[1:] == ["sub_batches"]:
    _sub_batch_child()

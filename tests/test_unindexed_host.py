"""Rows added after an index was built, without a GPU: Table.add and its refusals, index_stats as the reference pins it
(100 / 100 -> 200 / 0 after optimize), which native handle each builder state calls (default, fast_search,
bypass_vector_index, no index), the async and remote lowering of fast_search, and IndexData.extend for every kind in
IVF_KINDS (rows land after their partition's rows, in row-id order, encoded with the index's fitted model)."""
import asyncio

import numpy as np
import pyarrow as pa
import pytest
import torch

import lancedb_b200 as lancedb
from lancedb_b200 import _native, aio, remote
from lancedb_b200 import index as I
from lancedb_b200.index import IVF_KINDS

NBYTES = 4


class _FakeHandle:
    """Stands in for a native handle: records each call, answers with k copies of row 0."""
    calls = []

    def __init__(self, data=None, row_ids=None, device=0):
        rows = getattr(data, "nrows", None)
        self.nrows = rows if rows is not None else len(data)
        self.metric = getattr(data, "metric", "l2")
        self.closed = False
        _FakeHandle.calls.append(("open", type(self).__name__, self.nrows))

    def _answer(self, name, q, k):
        _FakeHandle.calls.append((name, type(self).__name__))
        B = np.asarray(q).reshape(-1, np.asarray(q).shape[-1]).shape[0]
        return np.zeros((B, k), np.uint64), np.zeros((B, k), np.float32), np.full(B, 1, np.uint32)

    def search(self, q, k=10, **kw):
        return self._answer("search", q, k)

    def search_unindexed(self, tail, q, k=10, **kw):
        assert isinstance(tail, _FakeHandle)
        return self._answer("search_unindexed", q, k)

    def append(self, rows, row_ids=None):
        _FakeHandle.calls.append(("append", type(self).__name__, len(rows)))
        self.nrows += len(rows)

    def close(self):
        self.closed = True


class FakeIvf(_FakeHandle):
    pass


class FakeFlat(_FakeHandle):
    pass


@pytest.fixture
def fake_native(monkeypatch):
    _FakeHandle.calls = []
    monkeypatch.setattr(_native, "GpuIvfBinary", FakeIvf)
    monkeypatch.setattr(_native, "GpuBinary", FakeFlat)
    monkeypatch.setattr(_native, "GpuFlat", FakeFlat)
    return _FakeHandle.calls


def _binary_table(n=100, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256, (n, NBYTES)).astype(np.uint8)
    schema = pa.schema([pa.field("id", pa.int64()), pa.field("vector", pa.list_(pa.uint8(), NBYTES))])
    t = lancedb.connect().create_table("t", {"id": np.arange(n), "vector": x}, schema=schema)
    return t, rng


def test_add_appends_rows_and_refuses_other_schemas(fake_native):
    t, rng = _binary_table()
    t.add({"id": [100, 101], "vector": rng.integers(0, 256, (2, NBYTES))})
    assert t.count_rows() == 102 and t.to_arrow()["id"].to_pylist()[-2:] == [100, 101]
    with pytest.raises(ValueError, match="schema"):
        t.add({"vector": rng.integers(0, 256, (2, NBYTES))})                       # a column missing
    with pytest.raises(ValueError, match="schema"):
        t.add({"id": [1], "vector": rng.integers(0, 256, (1, NBYTES)), "extra": [1]})
    with pytest.raises(ValueError, match="schema"):
        t.add({"id": [1], "vector": rng.integers(0, 256, (1, NBYTES + 1))})        # another vector width
    with pytest.raises(NotImplementedError):
        t.add({"id": [1], "vector": rng.integers(0, 256, (1, NBYTES))}, mode="overwrite")
    with pytest.raises(ValueError):
        t.add({"id": [1], "vector": rng.integers(0, 256, (1, NBYTES))}, mode="merge")
    assert t.count_rows() == 102


def test_index_stats_count_added_rows_until_optimize(fake_native):
    # python/python/lancedb/table.py:3970 / rust/lancedb/src/table/optimize.rs:490-532: 100 / 100 -> 200 / 0
    t, rng = _binary_table()
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector")
    t.add({"id": np.arange(100, 200), "vector": rng.integers(0, 256, (100, NBYTES))})
    st = t.index_stats("vector_idx")
    assert (st["num_indexed_rows"], st["num_unindexed_rows"]) == (100, 100)
    with pytest.raises(NotImplementedError):
        t.optimize(retrain=True)
    t.optimize()
    st = t.index_stats("vector_idx")
    assert (st["num_indexed_rows"], st["num_unindexed_rows"]) == (200, 0)
    assert "vector" not in t._tail and sorted(t._index_data["vector"].row_ids.tolist()) == list(range(200))


def test_each_builder_state_calls_its_handle(fake_native):
    t, rng = _binary_table()
    q = rng.integers(0, 256, NBYTES)
    t.search(q).to_arrow()                                        # no index: the flat handle
    assert fake_native[-1] == ("search", "FakeFlat")
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector")
    t.search(q).to_arrow()                                        # index, no tail: today's call
    assert fake_native[-1] == ("search", "FakeIvf")
    t.add({"id": [100, 101, 102], "vector": rng.integers(0, 256, (3, NBYTES))})
    assert ("append", "FakeFlat", 3) in fake_native               # the full-column cache grows in place
    assert ("open", "FakeFlat", 3) in fake_native                 # the tail handle
    t.search(q).to_arrow()
    assert fake_native[-1] == ("search_unindexed", "FakeIvf")
    t.search(q).fast_search().to_arrow()
    assert fake_native[-1] == ("search", "FakeIvf")
    t.search(q).bypass_vector_index().to_arrow()
    assert fake_native[-1] == ("search", "FakeFlat")
    t.add({"id": [103], "vector": rng.integers(0, 256, (1, NBYTES))})
    assert fake_native[-1] == ("append", "FakeFlat", 1)           # the tail grows in place too
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector")
    assert "vector" not in t._tail                                # a new index holds every row
    t.search(q).to_arrow()
    assert fake_native[-1] == ("search", "FakeIvf")


def test_async_and_remote_lower_fast_search(fake_native):
    t, rng = _binary_table()
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector")
    at = aio.AsyncTable(t)
    q = rng.integers(0, 256, NBYTES)

    async def run():
        await at.add({"id": [100], "vector": rng.integers(0, 256, (1, NBYTES))})
        await at.vector_search(q).to_arrow()
        default = fake_native[-1]
        await at.vector_search(q).fast_search().to_arrow()
        fast = fake_native[-1]
        await at.optimize()
        return default, fast
    default, fast = asyncio.run(run())
    assert default == ("search_unindexed", "FakeIvf") and fast == ("search", "FakeIvf")
    assert t.index_stats("vector_idx")["num_unindexed_rows"] == 0
    t.add({"id": [101], "vector": rng.integers(0, 256, (1, NBYTES))})
    remote.handle_query(t, remote.build_query_body(q, fast_search=True))
    assert fake_native[-1] == ("search", "FakeIvf")
    remote.handle_query(t, remote.build_query_body(q))
    assert fake_native[-1] == ("search_unindexed", "FakeIvf")


def _stub_assign(monkeypatch):
    """The coarse step's assignment and the 8-bit encoder through the C oracle (the same arithmetic as the kernels)."""
    import oracle

    def assign(centroids, vectors, metric="l2", device=0):
        c = np.asarray(centroids, np.float32)
        ix = oracle.OracleIndex(dim=c.shape[1], nlist=c.shape[0], m=1, metric=metric, centroids=c,
                                codebook=np.zeros((1, 256, c.shape[1]), np.float32),
                                part_offsets=np.zeros(c.shape[0] + 1, np.uint64), codes_t=np.zeros(0, np.uint8),
                                row_ids=np.zeros(0, np.uint64))
        return ix.ivf_assign(vectors)

    def encode(centroids, codebook, vectors, parts, metric="l2", device=0):
        c, cb = np.asarray(centroids, np.float32), np.asarray(codebook, np.float32)
        ix = oracle.OracleIndex(dim=c.shape[1], nlist=c.shape[0], m=cb.shape[0], metric=metric, centroids=c,
                                codebook=cb, part_offsets=np.zeros(c.shape[0] + 1, np.uint64),
                                codes_t=np.zeros(0, np.uint8), row_ids=np.zeros(0, np.uint64))
        return ix.pq_encode(vectors, parts)
    monkeypatch.setattr(_native, "ivf_assign", assign)
    monkeypatch.setattr(_native, "pq_encode", encode)
    return assign


CASES = [("IVF_PQ", "l2", dict(num_sub_vectors=4)), ("IVF_PQ", "cosine", dict(num_sub_vectors=4, num_bits=4)),
         ("IVF_SQ", "cosine", {}), ("IVF_HNSW_SQ", "l2", dict(m=4, ef_construction=20)), ("IVF_RQ", "l2", {}),
         ("IVF_FLAT", "hamming", {})]


@pytest.mark.parametrize("kind,metric,params", CASES, ids=[c[0] + "-" + c[1] for c in CASES])
def test_extend_appends_after_each_partition_with_the_fitted_model(monkeypatch, kind, metric, params):
    assert {c[0] for c in CASES} == set(IVF_KINDS)
    assign = _stub_assign(monkeypatch)
    rng = np.random.default_rng(3)
    binary = kind == "IVF_FLAT"
    n0, n = 300, 57
    x = rng.integers(0, 256, (n0 + n, NBYTES)).astype(np.uint8) if binary else \
        rng.standard_normal((n0 + n, 16)).astype(np.float32)
    kw = {} if binary else dict(keep_vectors=True)
    d = IVF_KINDS[kind].train(x[:n0], num_partitions=5, distance_type=metric, max_iterations=3, **kw, **params)
    new_ids = rng.permutation(np.arange(n0, n0 + n)).astype(np.uint64)
    e = d.extend(x[new_ids.astype(np.int64)], new_ids)
    parts = I.kmodes_assign(x[n0:], d.centroids) if binary else assign(getattr(d, "sq", d).centroids, x[n0:], metric)
    old, off = d.part_offsets.astype(np.int64), e.part_offsets.astype(np.int64)
    assert e.nrows == n0 + n
    for p in range(d.nlist):
        rows = e.row_ids[off[p]:off[p + 1]]
        k = old[p + 1] - old[p]
        assert np.array_equal(rows[:k], d.row_ids[old[p]:old[p + 1]])          # the old rows, in their order
        want = np.arange(n0, n0 + n)[parts == p]
        assert np.array_equal(rows[k:], want.astype(np.uint64))                # then the new ones by row id
    # every new row carries the code its kind's encoder gives it against the fitted model
    pos = np.empty(n0 + n, np.int64)
    pos[e.row_ids.astype(np.int64)] = np.arange(n0 + n)
    at = pos[n0:]
    xs = x[n0:]
    if binary:
        assert np.array_equal(e.vectors[at], xs)
        return
    assert np.array_equal(e.vectors[at], xs)
    xn = I._normalise(torch.as_tensor(xs)).numpy() if metric == "cosine" else xs
    sq = getattr(e, "sq", e)
    if kind == "IVF_HNSW_SQ":
        e.validate()                                   # the rebuilt graphs and the kept ones hold every bound
        assert e.ef_construction == params["ef_construction"]      # rebuilt as the index was built
    if kind == "IVF_PQ":
        codes = e.row_codes()[at]
        if d.num_bits == 8:
            assert np.array_equal(codes, _native.pq_encode(d.centroids, d.codebook, xs, parts, metric))
        else:
            want = I.pq_codes(torch.as_tensor(xn), torch.as_tensor(d.centroids), torch.as_tensor(parts.astype(np.int64)),
                              torch.as_tensor(d.codebook), metric).numpy()
            assert np.array_equal(codes, I.pack_pq4(want))
    elif kind in ("IVF_SQ", "IVF_HNSW_SQ"):
        assert np.array_equal(sq.codes[at], I.sq_encode(xn, sq.lo, sq.hi))
    else:
        codes, add, scale = I.rq_encode(torch.as_tensor(xn), d.centroids, parts.astype(np.int64), d.rotation)
        assert np.array_equal(e.codes[at], codes) and np.array_equal(e.add_factors[at], add)
        assert np.array_equal(e.scale_factors[at], scale)


def test_add_refuses_bad_vectors_and_changes_nothing(fake_native, monkeypatch):
    # on_bad_vectors="error" (python/python/lancedb/table.py:4429-4445): a NaN anywhere in a float vector column is
    # refused; under an index, so is a row optimize() could not assign (an infinite component, a zero cosine vector)
    x = np.random.default_rng(4).standard_normal((100, 8)).astype(np.float32)
    t = lancedb.connect().create_table("f", {"vector": x})
    bad = x[:3].copy()
    bad[1, 2] = np.nan
    with pytest.raises(ValueError, match="NaNs"):
        t.add({"vector": bad})
    with pytest.raises(NotImplementedError):
        t.add({"vector": x[:3]}, on_bad_vectors="drop")
    inf = x[:3].copy()
    inf[2, 0] = np.inf
    other = lancedb.connect().create_table("g", {"vector": x})
    other.add({"vector": inf})                               # no index: nothing to refuse it
    assert other.count_rows() == 103 and t.count_rows() == 100
    _stub_assign(monkeypatch)
    monkeypatch.setattr(_native, "GpuIvfSq", FakeIvf)
    t.create_index(metric="cosine", num_partitions=2, index_type="IVF_SQ", vector_column_name="vector")
    for rows in (inf, np.vstack([x[:2], np.zeros((1, 8), np.float32)])):
        with pytest.raises(ValueError, match="cannot join"):
            t.add({"vector": rows})
    assert t.count_rows() == 100 and "vector" not in t._tail
    t.add({"vector": x[:5]})
    t.optimize()
    assert t.index_stats("vector_idx")["num_unindexed_rows"] == 0


def test_add_that_fails_in_a_tail_leaves_the_table_and_tails_as_they_were(fake_native, monkeypatch):
    rng = np.random.default_rng(2)
    vec = pa.list_(pa.uint8(), NBYTES)
    t = lancedb.connect().create_table("t", {"a": rng.integers(0, 256, (100, NBYTES)),
                                             "b": rng.integers(0, 256, (100, NBYTES))},
                                       schema=pa.schema([pa.field("a", vec), pa.field("b", vec)]))
    for c in ("a", "b"):
        t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name=c)
    more = lambda n: {"a": rng.integers(0, 256, (n, NBYTES)), "b": rng.integers(0, 256, (n, NBYTES))}
    t.add(more(10))
    tail_a, tail_b = t._tail["a"], t._tail["b"]

    def fail(rows, row_ids=None):
        raise MemoryError("device allocation failed")
    monkeypatch.setattr(tail_b, "append", fail)
    with pytest.raises(MemoryError):
        t.add(more(10))                      # a's tail took the rows, b's failed
    assert t.count_rows() == 110 and t._tail_from == {"a": 100, "b": 100}
    assert t._tail["b"] is tail_b and tail_b.nrows == 10
    assert t._tail["a"] is not tail_a and t._tail["a"].nrows == 10     # reopened over the table's rows
    assert ("open", "FakeFlat", 10) == fake_native[-1]

"""IVF_HNSW_SQ without a GPU: the C oracle against its NumPy mirror, the level-0 loop against the two-heap form and
against shuffled offers and a lossy visited set, a complete graph against IVF_SQ's oracle, and the builder's
determinism, bounds and recall."""
import numpy as np
import pytest

from lancedb_b200.index import HNSW_NONE, IvfHnswSqIndexData, build_hnsw_graph
from tests import hnsw_sq_oracle as H
from tests import sq_oracle
from tests.util import assert_same

f32 = np.float32


_IX = {}


def _index(metric):
    if metric not in _IX:
        _IX[metric] = H.random_hnsw_index(np.random.default_rng(3 if metric == "l2" else 4), n=700, dim=24, nlist=6,
                                          metric=metric, m=5, ef_construction=30, empty=(1,))
    return _IX[metric]


CASES = [dict(k=10, nprobes=3), dict(k=10, nprobes=3, ef=3), dict(k=10, nprobes=3, ef=10),
         dict(k=6, nprobes=6, ef=900), dict(k=10, nprobes=40), dict(k=5, nprobes=2, refine_factor=3),
         dict(k=10, nprobes=3, lower=3000.0, upper=150000.0), dict(k=12, nprobes=2, ef=20)]


@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_c_oracle_equals_the_numpy_mirror(metric, case):
    data = _index(metric)
    q = np.random.default_rng(case).standard_normal((9, data.dim)).astype(f32)
    q[1] = data.vectors[5]                                   # a row with duplicates: ties by position, then row id
    kw = CASES[case]
    assert_same(H.search(data, q, nthreads=2, **kw), H.search_np(data, q, **kw), str(kw))


def test_prefilter_with_widening_c_equals_numpy():
    data = _index("l2")
    rng = np.random.default_rng(8)
    q = rng.standard_normal((8, data.dim)).astype(f32)
    mask = rng.random(int(data.row_ids.max()) + 1) < 0.04
    for kw in (dict(k=10, nprobes=1, max_nprobes=6), dict(k=10, nprobes=2, max_nprobes=4, ef=25)):
        assert_same(H.search(data, q, allow=mask, **kw), H.search_np(data, q, allow=mask, **kw), str(kw))


def test_empty_and_single_row_partitions():
    from lancedb_b200.index import IvfSqIndexData
    rng = np.random.default_rng(2)
    codes = rng.integers(0, 256, (5, 8), dtype=np.uint8)
    codes[3] = codes[2]                                      # duplicate rows in one partition
    sq = IvfSqIndexData(dim=8, nlist=4, metric="l2", centroids=rng.standard_normal((4, 8)).astype(f32),
                        part_offsets=np.array([0, 0, 1, 5, 5], np.uint64), codes=codes,
                        row_ids=np.array([9, 4, 8, 2, 30], np.uint64), lo=-2.0, hi=2.0)
    data = IvfHnswSqIndexData(sq, 2, *build_hnsw_graph(codes, sq.part_offsets, 2, 10))
    data.validate()
    q = rng.standard_normal((5, 8)).astype(f32)
    for kw in (dict(k=3, nprobes=4), dict(k=10, nprobes=4, ef=2)):
        assert_same(H.search(data, q, **kw), H.search_np(data, q, **kw), str(kw))


def _random_graph(rng, n, deg):
    adj = np.full((n, deg), HNSW_NONE, np.uint32)
    for r in range(n):
        k = rng.integers(0, deg + 1)
        adj[r, :k] = rng.choice(n, k, replace=False)
    return adj


@pytest.mark.parametrize("seed", range(6))
def test_list_loop_equals_the_two_heap_loop_and_ignores_offer_order_and_lost_visits(seed):
    rng = np.random.default_rng(seed)
    n = 300
    codes = rng.integers(0, 4, (n, 6)).astype(np.int64)      # small codes: many equal distances
    q = rng.integers(0, 4, 6)
    dist = lambda r: f32(int(((codes[r] - q) ** 2).sum()))
    adj = _random_graph(rng, n, 8)
    for efp in (1, 3, 10, 64, 400):
        want = H.level0_np(dist, adj, 0, efp)
        assert H.two_heap_np(dist, adj, 0, efp) == want
        assert H.level0_np(dist, adj, 0, efp, rng=np.random.default_rng(seed + 100)) == want
        lossy = np.random.default_rng(seed + 200)
        assert H.level0_np(dist, adj, 0, efp, forget=lambda v: lossy.random() < 0.3) == want


def test_complete_graph_returns_ivf_sq_results():
    data = _index("l2")
    full = H.complete_graph(data.sq)
    q = np.random.default_rng(6).standard_normal((10, data.dim)).astype(f32)
    big = int(np.diff(data.part_offsets.astype(np.int64)).max())
    for kw in (dict(k=10, nprobes=6), dict(k=5, nprobes=3, refine_factor=2)):
        assert_same(H.search(full, q, ef=big, **kw), sq_oracle.search(data.sq, q, **kw), str(kw))


def test_ef_prime_above_2048_is_refused_by_the_oracle():
    data = _index("l2")
    with pytest.raises(RuntimeError):
        H.search(data, np.zeros((1, data.dim), f32), k=10, nprobes=2, ef=2049)


def test_builder_is_deterministic_and_in_bounds():
    from lancedb_b200.index import train_ivf_hnsw_sq
    x = np.random.default_rng(0).standard_normal((1200, 16)).astype(f32)
    a = train_ivf_hnsw_sq(x, num_partitions=3, m=6, ef_construction=40, max_iterations=5)
    b = train_ivf_hnsw_sq(x, num_partitions=3, m=6, ef_construction=40, max_iterations=5)
    for f in ("levels", "adj0", "upper_index", "upper_adj", "entry", "top_level"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    a.validate()                                             # every index in range, degrees within m / 2m
    assert a.adj0.shape[1] == 12 and a.upper_adj.shape[1] == 6
    off = a.part_offsets.astype(np.int64)
    for p in range(a.nlist):                                 # no self loops, no repeated neighbour
        for r in range(off[p + 1] - off[p]):
            nb = a.adj0[off[p] + r]
            nb = nb[nb != HNSW_NONE]
            assert r not in nb and len(set(nb.tolist())) == len(nb)


# recall@10 of the graph search against IVF_SQ's exact scan of the same probes: 0.974 on the first run (2000 x 32
# clustered rows, 4 partitions, m 8, ef_construction 64, ef 0 = 15, nprobes 2); the floor leaves room for builder
# changes
RECALL_FLOOR = 0.95


def test_recall_against_ivf_sq_over_the_same_probes():
    from lancedb_b200.index import train_ivf_hnsw_sq
    rng = np.random.default_rng(1)
    centres = rng.standard_normal((12, 32)).astype(f32) * 4
    x = (centres[rng.integers(0, 12, 2000)] + rng.standard_normal((2000, 32))).astype(f32)
    data = train_ivf_hnsw_sq(x, num_partitions=4, m=8, ef_construction=64, max_iterations=10)
    q = (centres[rng.integers(0, 12, 50)] + rng.standard_normal((50, 32))).astype(f32)
    gi, _, _ = H.search(data, q, k=10, nprobes=2)
    si, _, _ = sq_oracle.search(data.sq, q, k=10, nprobes=2)
    recall = np.mean([len(set(a) & set(b)) / 10 for a, b in zip(gi.tolist(), si.tolist())])
    print("recall@10", recall)
    assert recall >= RECALL_FLOOR


# ---- the Python surfaces, with the native layer stubbed ----


class _StubHnsw:
    """Stands in for _native.GpuIvfHnswSq: records the arrays it was opened with; its search is GpuIvfPq.search, so
    the SearchParams it would pass to lgpu_search are built for real and recorded by the stubbed _host_search."""
    opened, params = [], []
    search = None

    def __init__(self, data, device=0):
        self.data, self.metric, self.dim, self._h = data, data.metric, data.dim, None
        _StubHnsw.opened.append(data)

    def close(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    from lancedb_b200 import _native
    _StubHnsw.opened, _StubHnsw.params = [], []
    _StubHnsw.search = _native.GpuIvfPq.search

    def host_search(fn, head, B, k, p, allow, allow_bits):
        _StubHnsw.params.append((fn, p.k, p.nprobes, p.refine_factor, p.ef))
        return np.zeros((B, k), np.uint64), np.zeros((B, k), f32), np.zeros(B, np.uint32)
    monkeypatch.setattr(_native, "GpuIvfHnswSq", _StubHnsw)
    monkeypatch.setattr(_native, "_host_search", host_search)
    return _StubHnsw


def _table(n=500, dim=16, seed=6):
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(seed)
    db = lancedb.connect("memory://")
    return db, db.create_table("t", {"vector": rng.standard_normal((n, dim)).astype(f32), "id": np.arange(n)})


def test_create_index_ivf_hnsw_sq_builds_lists_and_reports(stub):
    _, t = _table()
    t.create_index(metric="cosine", num_partitions=3, index_type="IVF_HNSW_SQ", m=5, ef_construction=20,
                   max_iterations=2)
    assert len(stub.opened) == 1 and isinstance(stub.opened[0], IvfHnswSqIndexData)
    d = stub.opened[0]
    assert d.m == 5 and d.adj0.shape == (500, 10) and d.metric == "cosine" and d.vectors is not None
    assert t.list_indices() == [{"name": "vector_idx", "index_type": "IVF_HNSW_SQ", "columns": ["vector"]}]
    st = t.index_stats("vector_idx")
    assert st["index_type"] == "IVF_HNSW_SQ" and st["distance_type"] == "cosine" and st["num_indexed_rows"] == 500


def test_create_index_ivf_hnsw_sq_refusals(stub):
    import pyarrow as pa
    db, t = _table(300, 8, 7)
    with pytest.raises(ValueError, match="l2 and cosine"):
        t.create_index(index_type="IVF_HNSW_SQ", metric="dot")
    with pytest.raises(ValueError, match="num_bits"):
        t.create_index(index_type="IVF_HNSW_SQ", num_bits=4)
    with pytest.raises(ValueError, match="m must be"):
        t.create_index(index_type="IVF_HNSW_SQ", m=65)
    for kind in ("IVF_HNSW_PQ", "IVF_HNSW_FLAT"):
        with pytest.raises(NotImplementedError):
            t.create_index(index_type=kind)
    schema = pa.schema([pa.field("bits", pa.list_(pa.uint8(), 4))])
    tb = db.create_table("b", pa.table({"bits": pa.FixedSizeListArray.from_arrays(
        pa.array(np.arange(40, dtype=np.uint8)), 4)}, schema=schema))
    with pytest.raises(NotImplementedError, match="binary"):
        tb.create_index(index_type="IVF_HNSW_SQ")
    mv = pa.array([[[1.0, 2.0], [3.0, 4.0]], [[5.0, 6.0]]], pa.list_(pa.list_(pa.float32(), 2)))
    tm = db.create_table("m", pa.table({"mv": mv}))
    with pytest.raises(NotImplementedError, match="multivector"):
        tm.create_index(index_type="IVF_HNSW_SQ")
    assert stub.opened == []


def test_ef_reaches_search_params(stub):
    import asyncio
    from lancedb_b200 import aio
    _, t = _table()
    t.create_index(num_partitions=2, index_type="IVF_HNSW_SQ", m=4, ef_construction=16, max_iterations=2)
    q = np.zeros(16, f32)
    t.search(q).limit(7).to_arrow()
    t.search(q).limit(7).ef(64).nprobes(3).to_arrow()
    with pytest.raises(ValueError, match="ef"):
        t.search(q).ef(0)

    async def main():
        at = aio.AsyncTable(t)
        await at.query().nearest_to(q).limit(5).ef(33).to_arrow()
        await at.create_index("vector", config=aio.HnswSq(num_partitions=2, m=3, ef_construction=8, max_iterations=2),
                              accelerator=None)
    asyncio.run(main())
    assert [p[4] for p in stub.params] == [0, 64, 33]
    assert stub.params[1][:3] == ("lgpu_search", 7, 3) and stub.params[2][1] == 5
    assert stub.opened[-1].m == 3

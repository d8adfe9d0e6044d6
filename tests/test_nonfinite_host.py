"""The oracles on NaN and infinite centroids and raw vectors, without a GPU: the C oracles equal their NumPy mirrors, and
the rules of DESIGN.md section 0 hold (a NaN _distance is never returned, a partition whose coarse distance is NaN is never
probed, +-inf distances are ordinary values ordered by (_distance, _rowid)).  The goldens under tests/golden/ are
reproduced by test_oracle_pins.py with the same oracle."""
import numpy as np
import pytest

import oracle
from oracle import oracle_np as onp
from tests import pq4_oracle, rq_oracle, sq_oracle
from tests.util import queries, random_index

INF = float("inf")
pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")      # NaN / inf arithmetic is the point


def _plant(c):
    c[1, 3] = np.nan
    c[2, 0] = INF
    c[4, 5] = -INF
    return c


def _nonfinite_queries(rng, dim):
    q = queries(rng, 8, dim)
    q[1] = 0.0
    q[2, 3] = np.nan
    q[3, 0] = INF
    q[4] = INF
    q[5, 1] = 2e19
    return q


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_find_partitions_never_returns_nan_ahead_of_a_number(metric):
    rng = np.random.default_rng(601)
    ix = random_index(rng, dim=16, nlist=12, m=4, n=600, metric=metric)
    _plant(ix.centroids)
    ix.centroids[7] = ix.centroids[2]                      # an inf tie: the lower partition id first
    orc = oracle.OracleIndex.from_data(ix)
    for q in _nonfinite_queries(rng, 16):
        qn = onp.normalize(q) if metric == "cosine" else q
        parts, dists, alld = orc.find_partitions(qn, 12)
        want = np.lexsort((np.arange(12), alld))           # NumPy: NaN last, ties by id
        assert np.array_equal(parts, want)
        nan = np.isnan(dists)
        assert not np.any(nan[:-1] & ~nan[1:]), dists     # NaN only after every number


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq_oracle_equals_its_mirror_on_nonfinite_centroids(metric):
    rng = np.random.default_rng(602)
    ix = random_index(rng, dim=16, nlist=8, m=4, n=800, metric=metric)
    _plant(ix.centroids)
    ix.codebook[1, 9, 2] = INF
    q = _nonfinite_queries(rng, 16)
    orc = oracle.OracleIndex.from_data(ix)
    for nprobes in (3, 8):
        oi, od, oc = orc.search(q, k=12, nprobes=nprobes)
        assert not np.isnan(od).any()
        for b in range(len(q)):
            mi, md = onp.ivfpq_search_one(ix, q[b], 12, nprobes)
            assert oc[b] == len(mi), (b, oc[b], len(mi))
            assert np.array_equal(oi[b, :oc[b]], mi)
            assert np.array_equal(od[b, :oc[b]].view(np.uint32), md.view(np.uint32))


def test_dot_nan_centroid_is_not_probed():
    """dot distances need no residual, so the rows of the other partitions stay finite: a query with nprobes = nlist
    gets every row but those of the NaN partition"""
    rng = np.random.default_rng(603)
    ix = random_index(rng, dim=16, nlist=6, m=4, n=600, metric="dot")
    ix.centroids[2, 0] = np.nan
    oi, od, oc = oracle.OracleIndex.from_data(ix).search(queries(rng, 1, 16), k=600, nprobes=6)
    a, b = int(ix.part_offsets[2]), int(ix.part_offsets[3])
    assert oc[0] == 600 - (b - a)
    assert not set(ix.row_ids[a:b].tolist()) & set(oi[0, :oc[0]].tolist())


def test_refine_never_returns_nan():
    """refine re-ranks the k * refine_factor candidates by the exact distance on the raw vectors; a NaN one is dropped,
    the others are ordered by (_distance, _rowid), inf included"""
    rng = np.random.default_rng(604)
    ix = random_index(rng, dim=16, nlist=4, m=4, n=400, with_vectors=True)
    ix.vectors[::3, 2] = np.nan
    ix.vectors[1::3, 5] = INF
    orc = oracle.OracleIndex.from_data(ix)
    q = queries(rng, 4, 16)
    ci, cd, cc = orc.search(q, k=40, nprobes=4)            # the candidates refine re-ranks
    ri, rd, rc = orc.search(q, k=10, nprobes=4, refine_factor=4)
    pos = {int(r): i for i, r in enumerate(ix.row_ids)}
    for b in range(4):
        ex = [(onp.l2(q[b], ix.vectors[pos[int(r)]]), int(r)) for r in ci[b, :cc[b]]]
        ex = sorted(e for e in ex if not np.isnan(e[0]))[:10]
        assert rc[b] == len(ex)
        assert ri[b, :rc[b]].tolist() == [e[1] for e in ex]
        assert np.array_equal(rd[b, :rc[b]], np.array([e[0] for e in ex], np.float32))


@pytest.mark.parametrize("kind", ["sq", "rq", "pq4"])
def test_kind_oracles_equal_their_mirrors_on_nonfinite_centroids_and_vectors(kind):
    rng = np.random.default_rng(605)
    if kind == "sq":
        ix = sq_oracle.random_sq_index(rng, n=500, dim=24, nlist=6, empty=())
        c_search, np_search = sq_oracle.search, sq_oracle.sq_search_np
    elif kind == "rq":
        ix = rq_oracle.random_rq_index(rng, n=500, dim=24, nlist=6, empty=())
        c_search, np_search = rq_oracle.search, rq_oracle.rq_search_np
    else:
        ix = pq4_oracle.random_pq4_index(rng, n=500, dim=24, nlist=6, m=6, empty=())
        c_search, np_search = pq4_oracle.search, pq4_oracle.pq4_search_np
    ix.centroids[1, 3] = np.nan
    ix.centroids[2, 0] = INF
    ix.vectors[::4, 1] = np.nan
    ix.vectors[1::4, 2] = INF
    q = _nonfinite_queries(rng, 24)
    for kw in (dict(k=10, nprobes=3), dict(k=10, nprobes=6), dict(k=5, nprobes=4, refine_factor=4)):
        oi, od, oc = c_search(ix, q, **kw)
        mi, md, mc = np_search(ix, q, **kw)
        assert np.array_equal(oc, mc) and np.array_equal(oi, mi), kw
        assert np.array_equal(od.view(np.uint32), md.view(np.uint32)), kw
        assert not np.isnan(od).any()


def test_create_index_refuses_nonfinite_rows_on_the_cpu():
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(606)
    x = rng.standard_normal((2000, 16)).astype(np.float32)
    x[777, 3] = np.nan
    x[1500, 0] = -INF
    t = lancedb.connect("memory://").create_table("t", {"vector": list(x), "id": np.arange(2000)})
    with pytest.raises(ValueError, match="vector 777 "):
        t.create_index(metric="l2", num_partitions=8, num_sub_vectors=4)
    x[777, 3] = 0.0
    from lancedb_b200.index import train_ivf_sq
    with pytest.raises(ValueError, match="vector 1500 "):
        train_ivf_sq(x, num_partitions=8)

"""CPU checks of multivector (late-interaction, MaxSim) search: the C oracle against its NumPy mirror, the reduction to
flat cosine search, the reference's doubling pin, and the Python surface (Table, builder, async, remote) against a
stubbed native layer that answers with the C oracle."""
import asyncio

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200
import oracle
from lancedb_b200 import _native, remote
from lancedb_b200.aio import AsyncTable
from tests.multivec_oracle import (cosine_matrix_np, distances, distances_np, flat_search_mv, flat_search_mv_np,
                                   offsets_of)


def _rows(rng, lens, dim):
    off = offsets_of(lens)
    return rng.standard_normal((int(off[-1]), dim)).astype(np.float32), off


@pytest.mark.parametrize("dim", [2, 15, 16, 33, 64])
def test_c_oracle_matches_the_numpy_mirror(dim):
    rng = np.random.default_rng(dim)
    lens = rng.integers(0, 7, 60)
    lens[[0, 5, 59]] = 0                                   # empty (or null) rows
    x, off = _rows(rng, lens, dim)
    x[2] = 0.0                                             # a zero stored vector: its pairs are NaN and skipped
    x[7] = x[8]                                            # identical vectors
    q = rng.standard_normal((9, dim)).astype(np.float32)
    qo = offsets_of([1, 3, 5])
    a, b = distances(x, off, q, qo, 4), distances_np(x, off, q, qo)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.isnan(a[:, [0, 5, 59]]).all()
    for lower, upper in ((None, None), (0.5, None), (None, 3.0), (1.0, 4.0)):
        for k in (1, 7, 100):
            got, want = flat_search_mv(x, off, q, qo, k, lower=lower, upper=upper, nthreads=3), \
                flat_search_mv_np(x, off, q, qo, k, lower=lower, upper=upper)
            assert all(np.array_equal(g, w) for g, w in zip(got, want))
    allow = rng.random(80) < 0.5                           # ids beyond the mask are excluded
    rid = rng.permutation(100)[:60].astype(np.uint64)
    got = flat_search_mv(x, off, q, qo, 10, row_ids=rid, allow=allow, nthreads=2)
    want = flat_search_mv_np(x, off, q, qo, 10, row_ids=rid, allow=allow)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_mirror_cosine_is_the_float_oracles_cosine():
    rng = np.random.default_rng(3)
    q, x = rng.standard_normal((3, 37)).astype(np.float32), rng.standard_normal((5, 37)).astype(np.float32)
    m = cosine_matrix_np(q, x)
    for i in range(3):
        for j in range(5):
            assert np.float32(oracle.cosine(q[i], x[j])).view(np.uint32) == m[i, j].view(np.uint32)


def test_ties_come_back_in_row_id_order_and_nan_queries_return_nothing():
    rng = np.random.default_rng(4)
    v = rng.standard_normal((1, 8)).astype(np.float32)
    x = np.repeat(v, 12, axis=0)
    off = offsets_of([1, 2, 1, 3, 1, 1, 2, 1])             # every row holds only copies of v: all distances equal
    q = rng.standard_normal((2, 8)).astype(np.float32)
    ids, dist, cnt = flat_search_mv(x, off, q, [0, 2], 5)
    assert list(ids[0]) == [0, 1, 2, 3, 4] and len(set(dist[0].view(np.uint32))) == 1
    bad = np.stack([q[0], np.zeros(8, np.float32), np.full(8, np.nan, np.float32)])
    ids, dist, cnt = flat_search_mv(x, off, bad, [0, 1, 2, 3], 5)
    assert list(cnt) == [5, 0, 0]
    ids, dist, cnt = flat_search_mv(x, off, bad[:2], [0, 2], 5)      # one zero vector spoils the whole query
    assert cnt[0] == 0


def test_one_vector_per_row_and_query_is_flat_cosine_search():
    rng = np.random.default_rng(5)
    for dim in (2, 16, 127):
        x = rng.standard_normal((300, dim)).astype(np.float32)
        x[::50] *= 1e-3
        q = rng.standard_normal((6, dim)).astype(np.float32)
        got = flat_search_mv(x, offsets_of(np.ones(300, int)), q, offsets_of(np.ones(6, int)), 20, nthreads=2)
        want = oracle.flat_search(x, q, k=20, metric="cosine")
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2])
        assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


def test_duplicating_the_query_vector_doubles_every_distance_exactly():
    """test_query.py:809-813 (rs2["_distance"] == rs["_distance"] * 2 for [q] -> [q, q]); fl(0 + m) + m == 2 m."""
    rng = np.random.default_rng(6)
    for dim in (2, 48):
        x, off = _rows(rng, rng.integers(1, 9, 400), dim)
        q = rng.standard_normal((1, dim)).astype(np.float32)
        i1, d1, c1 = flat_search_mv(x, off, q, [0, 1], 50)
        i2, d2, c2 = flat_search_mv(x, off, np.concatenate([q, q]), [0, 2], 50)
        assert np.array_equal(i1, i2) and np.array_equal(c1, c2)
        assert np.array_equal(d2.view(np.uint32), (d1 * np.float32(2)).view(np.uint32))
    x = np.array([[i, i + 1, i + 2, i + 3] for i in range(256)], np.float32).reshape(-1, 2)   # the reference's table
    off = offsets_of(np.full(256, 2))
    _, d1, _ = flat_search_mv(x, off, np.array([[1, 2]], np.float32), [0, 1], 10)
    _, d2, _ = flat_search_mv(x, off, np.array([[1, 2], [1, 2]], np.float32), [0, 2], 10)
    assert np.array_equal(d2, d1 * 2)


# ---- the Python surface against a stubbed native layer ----


_GpuMultivec = _native.GpuMultivec


class _StubMultivec:
    """GpuMultivec stand-in answering with the C oracle; records every call."""
    calls = []

    def __init__(self, values, offsets, row_ids=None, device=0):
        self.values, self.offsets = np.asarray(values, np.float32), np.asarray(offsets, np.uint64)
        self.dim = self.values.shape[1]

    def search(self, queries, k=10, q_offsets=None, lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        q, qo = _GpuMultivec._queries(self, queries, q_offsets)
        mask = None
        if allow is not None:
            bits = np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")[:allow_bits]
            mask = bits.astype(bool)
        _StubMultivec.calls.append((q.copy(), qo.copy()))
        return flat_search_mv(self.values, self.offsets, q, qo, k, lower=lower, upper=upper, allow=mask)


@pytest.fixture
def stub(monkeypatch):
    _StubMultivec.calls = []
    monkeypatch.setattr(_native, "GpuMultivec", _StubMultivec)
    return _StubMultivec


def _reference_table(db, value_type=pa.float32(), large=False, name="test"):
    """test_query.py:179-203: 256 rows of [[i, i+1], [i+2, i+3]]."""
    data = [[[i, i + 1], [i + 2, i + 3]] for i in range(256)]
    lt = pa.large_list if large else pa.list_
    df = pa.table({"vector": pa.array(data, type=lt(pa.list_(value_type, list_size=2))),
                   "id": pa.array(list(range(1, 257))), "float_field": pa.array([float(i) for i in range(1, 257)])})
    return db.create_table(name, df)


@pytest.mark.parametrize("large", [False, True])
@pytest.mark.parametrize("vt", [pa.float16(), pa.float32(), pa.float64()])
def test_multivector_columns_are_vector_columns_and_answer_one_query(stub, vt, large):
    db = lancedb_b200.connect()
    tbl = _reference_table(db, vt, large)
    rs = tbl.search([1, 2]).to_arrow()
    rs2 = tbl.search([[1, 2], [1, 2]]).to_arrow()
    assert "query_index" not in rs2.column_names and len(rs2) == len(rs) == 10
    assert rs2["_distance"].to_pylist() == [d * 2 for d in rs["_distance"].to_pylist()]
    q, qo = stub.calls[-1]
    assert q.shape == (2, 2) and list(qo) == [0, 2]
    with pytest.raises(ValueError):
        tbl.search([1, 2, 3]).to_arrow()
    with pytest.raises(ValueError):
        tbl.search([[1, 2], [1, 2, 3]]).to_arrow()
    with pytest.raises(ValueError):
        tbl.search([[[1, 2]]]).to_arrow()
    with pytest.raises(NotImplementedError):
        tbl.create_index(metric="cosine", vector_column_name="vector", num_partitions=1, num_sub_vectors=2)


def test_metric_builder_and_filters(stub):
    db = lancedb_b200.connect()
    tbl = _reference_table(db)
    for metric in ("l2", "dot", "hamming"):
        with pytest.raises(ValueError):
            tbl.search([[1, 2]]).distance_type(metric).to_arrow()
    assert len(tbl.search([[1, 2]]).distance_type("cosine").to_arrow()) == 10
    full = tbl.search([[3, 1], [1, 5]]).limit(40).with_row_id(True).to_arrow()
    off = tbl.search([[3, 1], [1, 5]]).limit(5).offset(7).with_row_id(True).to_arrow()
    assert off["_rowid"].to_pylist() == full["_rowid"].to_pylist()[7:12]
    pre = tbl.search([[3, 1], [1, 5]]).where("id > 100").limit(20).select(["id"]).to_arrow()
    assert pre.column_names == ["id", "_distance"] and len(pre) == 20 and min(pre["id"].to_pylist()) > 100
    post = tbl.search([[3, 1], [1, 5]]).where("id > 100", prefilter=False).limit(20).to_arrow()
    assert all(i > 100 for i in post["id"].to_pylist()) and len(post) <= 20
    d = full["_distance"].to_pylist()
    rng_ = tbl.search([[3, 1], [1, 5]]).distance_range(d[3], d[9]).limit(40).to_arrow()
    assert all(d[3] <= x < d[9] for x in rng_["_distance"].to_pylist())
    assert tbl.search([[3, 1]]).to_pandas().shape[0] == 10
    assert sum(b.num_rows for b in tbl.search([[3, 1]]).limit(30).to_batches(7)) == 30


def test_null_and_empty_rows_are_never_returned(stub):
    db = lancedb_b200.connect()
    data = [[[1.0, 0.0]], None, [], [[0.0, 1.0], [1.0, 1.0]]]
    tbl = db.create_table("t", pa.table({"vector": pa.array(data, type=pa.list_(pa.list_(pa.float32(), 2)))}))
    out = tbl.search([[1.0, 0.0]]).with_row_id(True).to_arrow()
    assert sorted(out["_rowid"].to_pylist()) == [0, 3]


def test_column_inference_by_dimension_and_ambiguity(stub):
    db = lancedb_b200.connect()
    mv = pa.array([[[1.0, 2.0]], [[3.0, 4.0]]], type=pa.list_(pa.list_(pa.float32(), 2)))
    flat = pa.FixedSizeListArray.from_arrays(pa.array(np.ones(6, np.float32)), 3)
    tbl = db.create_table("a", pa.table({"mv": mv, "flat": flat}))
    assert tbl.search([[1, 2], [3, 4]])._vector_column == "mv"
    assert tbl.search([1, 2, 3])._vector_column == "flat"
    flat2 = pa.FixedSizeListArray.from_arrays(pa.array(np.ones(4, np.float32)), 2)
    tbl2 = db.create_table("b", pa.table({"mv": mv, "flat2": flat2}))
    with pytest.raises(ValueError, match="multiple vector columns"):
        tbl2.search([1, 2])


def test_async_and_remote_lower_to_one_multivector_query(stub):
    db = lancedb_b200.connect()
    tbl = _reference_table(db)
    want = tbl.search([[1, 2], [5, 1]]).limit(7).to_arrow()

    async def run():
        at = AsyncTable(tbl)
        a = await at.query().nearest_to([[1, 2], [5, 1]]).limit(7).to_arrow()
        b = await at.query().nearest_to([1, 2]).add_query_vector([5, 1]).limit(7).to_arrow()
        with pytest.raises(ValueError):
            await at.query().nearest_to([[1, 2], [1, 2, 3]]).to_arrow()
        return a, b

    a, b = asyncio.run(run())
    assert a.equals(want) and b.equals(want) and "query_index" not in a.column_names
    body = remote.build_query_body([[1, 2], [5, 1]], k=7)
    out = remote.read_ipc_file(remote.handle_query(tbl, body))
    assert out.equals(want)
    q, qo = stub.calls[-1]
    assert list(qo) == [0, 2]
    with pytest.raises(ValueError):
        remote.handle_query(tbl, {"vector": [[1, 2], [1, 2, 3]], "k": 3})


def test_gpu_multivec_checks_shapes_before_the_device():
    mv = _native.GpuMultivec.__new__(_native.GpuMultivec)    # the checks need no device
    mv.dim = 4
    q, qo = mv._queries([np.zeros((3, 4)), np.zeros(4)], None)
    assert q.shape == (4, 4) and list(qo) == [0, 3, 4]
    q, qo = mv._queries(np.zeros((5, 4)), None)                   # one array = one query
    assert list(qo) == [0, 5]
    assert list(mv._queries(np.zeros((5, 4)), [0, 2, 5])[1]) == [0, 2, 5]
    for bad, off in ((np.zeros((2, 3)), None), ([np.zeros((1, 1, 4))], None), (np.zeros((4, 4)), [0, 2, 2, 4]),
                     (np.zeros((4, 4)), [0, 5]), (np.zeros((4, 4)), [1, 4]), ([np.zeros((4097, 4))], None)):
        with pytest.raises(ValueError):
            mv._queries(bad, off)
    for vals, off in ((np.zeros((3, 4)), [0, 2]), (np.zeros((3, 4)), [0, 2, 1, 3]), (np.zeros((3, 4)), [1, 3]),
                      (np.zeros(3), [0, 3])):
        with pytest.raises(ValueError):
            _native.GpuMultivec(vals, off)


def test_gpu_multivec_has_no_cpu_fallback():
    try:
        if _native.device_count() > 0:
            pytest.skip("a CUDA device is present")
    except ImportError:
        pytest.skip("library not built")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _native.GpuMultivec(np.zeros((3, 4), np.float32), [0, 1, 3])


# ---- the tensor-core shortlist's band (multivec.cu mv_band) under adversarial fp16 rounding ----

F32 = np.float32
U = 2.0 ** -24


def mv_band(nq, d, one_operand=False):
    """multivec.cu mv_band restated in f32 (one_operand: a band that allows only one operand's fp16 rounding)."""
    e = F32(1.01) * F32(2.0 ** (-11 if one_operand else -10)) + (F32(8) * F32(d) + np.sqrt(F32(d)) + F32(40)) * F32(U)
    return F32((F32(nq) * e + F32(4.04) * F32(nq) * F32(nq) * F32(U)) * F32(1 + 2.0 ** -8))


def _approx_maxsim(q, x, off, qoff):
    """The approximate distances of the tensor-core path restated: fp16 of the normalised vectors (normalised as
    mv_normalize_f16_kernel does), products summed in f64 and rounded to f32 (wgmma's accumulation error is a term of
    the band of its own), max over each row's run, sum of (1 - max) over the query's vectors."""
    from tests.multivec_oracle import lance_dot_np

    def nrm16(v):
        n = np.array([np.sqrt(lance_dot_np(r, r[None, :])[0]) for r in v], F32)
        return (v / n[:, None]).astype(F32).astype(np.float16).astype(np.float64)

    S = (nrm16(q) @ nrm16(x).T).astype(F32)
    B, N = len(qoff) - 1, len(off) - 1
    A = np.full((B, N), np.nan, F32)
    for r in range(N):
        if off[r + 1] == off[r]:
            continue
        m = S[:, int(off[r]):int(off[r + 1])].max(axis=1)
        for b in range(B):
            A[b, r] = np.sum(F32(1) - m[int(qoff[b]):int(qoff[b + 1])], dtype=F32)
    return A


def _unit_at_midpoints(rng, d, up):
    """A vector whose lance norm is exactly 1.0f and whose components sit one f32 ulp above (up) or below an fp16
    rounding midpoint: fp16 rounds each of them by (almost) half an fp16 ulp, all in the direction of `up`."""
    from tests.multivec_oracle import lance_dot_np
    while True:
        c = F32(0.125) * (F32(1) + F32(2.0 ** -11) * (2 * rng.integers(0, 64, d) + 1).astype(F32))   # fp16 midpoints
        c = (c * np.where(rng.random(d) < 0.5, 1, -1)).astype(F32)
        c /= np.sqrt(np.sum(c.astype(np.float64) ** 2))
        h = c.astype(np.float16).astype(np.float64)
        lo = np.abs(h) - (2.0 ** (np.floor(np.log2(np.abs(h))) - 11))               # the midpoint below |h|
        mid = np.where(np.abs(c) >= np.abs(h), np.abs(h) + (2.0 ** (np.floor(np.log2(np.abs(h))) - 11)), lo)
        v = (np.sign(c) * np.nextafter(mid.astype(F32), F32(np.inf) if up else F32(0))).astype(F32)
        for _ in range(64):                                  # make the lance norm exactly 1 by nudging one component
            n2 = lance_dot_np(v, v[None, :])[0]
            if n2 == F32(1):
                return v
            v[-1] = np.nextafter(v[-1], np.sign(v[-1]) * (F32(0) if n2 > 1 else F32(np.inf)))


def test_band_holds_under_adversarial_fp16_rounding_and_one_operand_band_does_not():
    from tests.multivec_oracle import distances
    rng = np.random.default_rng(40)
    d = 64
    q = np.stack([_unit_at_midpoints(rng, d, True) for _ in range(6)])
    base = np.stack([_unit_at_midpoints(rng, d, True) for _ in range(40)])
    # rows: copies of the query vectors (similarity ~1, where the fp16 errors add up) and random midpoint vectors
    x = np.concatenate([q, base, q[::-1]]).astype(F32)
    off = offsets_of([1] * 6 + [2] * 20 + [1] * 6)
    qoff = offsets_of([1, 2, 3])
    D = distances(x, off, q, qoff)
    A = _approx_maxsim(q, x, off, qoff)
    worst_full, worst_one = 0.0, 0.0
    for b in range(3):
        nq = int(qoff[b + 1] - qoff[b])
        err = np.nanmax(np.abs(A[b].astype(np.float64) - D[b]))
        worst_full = max(worst_full, err / mv_band(nq, d))
        worst_one = max(worst_one, err / mv_band(nq, d, one_operand=True))
        # every consumer decision: the k-th approximate distance + 2 E (rounded up) admits the true top-k
        for k in (1, 3, 10):
            tau = np.sort(A[b][~np.isnan(A[b])])[k - 1]
            thr = np.nextafter(F32(tau + F32(2) * mv_band(nq, d)), F32(np.inf))
            admitted = set(np.nonzero(A[b] <= thr)[0])
            order = np.lexsort((np.arange(D.shape[1]), D[b]))
            true_top = [r for r in order if not np.isnan(D[b, r])][:k]
            assert set(true_top) <= admitted
    assert worst_full <= 1.0                                 # the band holds
    assert worst_one > 1.0                                   # one operand's rounding alone does not cover these rows

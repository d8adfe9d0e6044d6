"""IVF_RQ without a GPU: the C oracle against its NumPy mirror (rotation, slot grid, estimates, whole searches), edge
cases of the grid, the estimator's algebra and bias, the trainer's invariants, and the refusals of
create_index(index_type="IVF_RQ") and its aio config against a stubbed native layer.  The build through create_index
is in test_ivf_kinds_host.py."""
import asyncio

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200.index import rq_encode, rq_rotation, train_ivf_rq
from tests import rq_oracle
from tests.rq_oracle import random_rq_index, rq_estimates_np, rq_rotate_np, rq_slot_np
from tests.util import record_opens

f32 = np.float32


def _bits(a):
    return np.asarray(a, f32).view(np.uint32)


def _same_f32(a, b):
    return (np.isnan(a) and np.isnan(b)) or _bits(a) == _bits(b)


def _slot_equal(rq, rc):
    cu, clo, cd, cqq, cS = rq_oracle.rq_slot(rq, rc)
    nu, nlo, nd, nqq, nS = rq_slot_np(rq, rc)
    assert np.array_equal(cu, nu) and cS == nS
    assert _same_f32(clo, nlo) and _same_f32(cd, nd) and _same_f32(cqq, nqq)
    return cu, clo, cd, cqq, cS


@pytest.mark.parametrize("dim", [1, 7, 8, 33, 255, 256, 257, 768])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_rotation_grid_and_estimates_c_equal_numpy(dim, metric):
    rng = np.random.default_rng(dim)
    P = rq_rotation(dim, seed=dim)
    x = rng.standard_normal((3, dim)).astype(f32)
    assert np.array_equal(_bits(rq_oracle.rq_rotate(P, x)), _bits(rq_rotate_np(P, x)))
    rq, rc = rq_rotate_np(P, x[:2])
    u, lo, delta, qq, S = _slot_equal(rq, rc)
    assert u.max() <= 15 and S == int(u.astype(np.int64).sum())
    codes = rng.integers(0, 256, (40, (dim + 7) // 8), dtype=np.uint8)
    if dim % 8:
        codes[:, -1] &= (1 << (dim % 8)) - 1              # padding bits are 0
    add = (rng.random(40) * 5).astype(f32); scale = (-rng.random(40) * 2).astype(f32)
    c = rq_oracle.rq_estimates(codes, add, scale, u, lo, delta, qq, S, dim, metric)
    n = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, metric)
    assert np.array_equal(_bits(c), _bits(n))


@pytest.mark.parametrize("dim", [1, 7, 8, 33, 255, 256, 257, 768])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_c_oracle_search_equals_numpy_mirror(dim, metric):
    rng = np.random.default_rng(100 + dim + (metric == "cosine"))
    n = 400 if dim < 700 else 150
    ix = random_rq_index(rng, n=n, dim=dim, nlist=6, metric=metric)
    q = rng.standard_normal((6, dim)).astype(f32)
    q[1] *= 1e4                                          # huge magnitude
    q[2, 0] = np.nan                                     # no finite centroid distance: no rows
    q[3] = ix.vectors[4]                                 # ties among the duplicate rows
    allow = rng.random(n * 3 + 7) < 0.3
    cases = [dict(k=10, nprobes=2), dict(k=n + 50, nprobes=6), dict(k=5, nprobes=3, refine_factor=4),
             dict(k=12, nprobes=1, allow=allow, max_nprobes=6), dict(k=4, nprobes=2, allow=allow)]
    d = rq_oracle.search(ix, q[:1], k=40, nprobes=3)[1][0]
    cases.append(dict(k=8, nprobes=3, lower=float(d[3]), upper=float(d[30])))
    for kw in cases:
        ci, cd, cc = rq_oracle.search(ix, q, nthreads=3, **kw)
        ni, nd, nc = rq_oracle.rq_search_np(ix, q, **kw)
        assert np.array_equal(cc, nc), kw
        assert np.array_equal(ci, ni), kw
        assert np.array_equal(_bits(cd), _bits(nd)), kw
        assert cc[2] == 0
        for b in range(q.shape[0]):                      # ascending by (_distance, _rowid)
            m = int(cc[b])
            keys = list(zip(cd[b, :m].tolist(), ci[b, :m].tolist()))
            assert keys == sorted(keys)


def test_grid_edge_cases():
    dim = 37
    zero = np.zeros(dim, f32)
    # delta = 0: every u is 0, S = 0, the estimate is add + qq + scale * lo * (2 pc - dim)
    u, lo, delta, qq, S = _slot_equal(np.full(dim, 0.5, f32), zero)
    assert delta == 0 and not u.any() and S == 0
    # a row equal to its centroid (o = 0: add = scale = 0) against a query at the centroid: estimate 0
    u, lo, delta, qq, S = _slot_equal(zero, zero)
    codes = np.zeros((1, 5), np.uint8)
    for fn in (rq_oracle.rq_estimates, rq_estimates_np):
        e = fn(codes, np.zeros(1, f32), np.zeros(1, f32), u, lo, delta, qq, S, dim)
        assert _bits(e)[0] == 0                          # +0, not -0
    # signed zeros: -0 orders below +0 whatever their positions
    v = np.zeros(dim, f32); v[3] = -0.0; v[30] = -0.0
    u, lo, delta, qq, S = _slot_equal(v, zero)
    assert np.signbit(lo) and delta == 0 and not np.signbit(delta)
    # a huge component: the others collapse onto the bottom of the grid
    v = np.ones(dim, f32); v[0] = 1e30
    u, lo, delta, qq, S = _slot_equal(v, zero)
    assert u[0] == 15 and not u[1:].any() and np.isinf(qq)
    # a NaN component, or an infinite range: delta is not finite and the slot has no rows
    for bad in (np.nan, np.inf):
        v = np.ones(dim, f32); v[5] = bad
        u, lo, delta, qq, S = _slot_equal(v, zero)
        assert not np.isfinite(delta) and not u.any()
        e = rq_oracle.rq_estimates(codes, np.ones(1, f32), -np.ones(1, f32), u, lo, delta, qq, S, dim)
        assert np.isnan(e).all() and np.isnan(rq_estimates_np(codes, np.ones(1, f32), -np.ones(1, f32), u, lo, delta,
                                                              qq, S, dim)).all()
    # the top of the grid saturates at 15
    u, *_ = _slot_equal(np.linspace(-1, 1, dim).astype(f32), zero)
    assert u[0] == 0 and u[-1] == 15


def test_duplicate_rows_are_ordered_by_row_id():
    rng = np.random.default_rng(11)
    ix = random_rq_index(rng, n=200, dim=16, nlist=1, empty=())
    ix.codes[:] = ix.codes[0]
    ix.add_factors[:] = ix.add_factors[0]; ix.scale_factors[:] = ix.scale_factors[0]
    q = rng.standard_normal((1, 16)).astype(f32)
    ids, dist, cnt = rq_oracle.search(ix, q, k=150, nprobes=1)
    assert cnt[0] == 150 and np.all(dist[0] == dist[0, 0])
    assert np.array_equal(ids[0], np.sort(ix.row_ids)[:150])


def test_estimator_is_exact_up_to_rounding_on_its_grid():
    # o = alpha (2b - 1) and q' on its 16-level grid: the estimate is |o - q'|^2 within the final roundings
    rng = np.random.default_rng(12)
    dim, alpha = 64, 0.7
    for _ in range(20):
        b = rng.integers(0, 2, dim)
        o = alpha * (2.0 * b - 1.0)
        lo_, delta_ = -1.5, 0.2
        uu = rng.integers(0, 16, dim)
        uu[0], uu[1] = 0, 15                             # the grid's ends are taken
        qp = (lo_ + delta_ * uu).astype(f32)
        u, lo, delta, qq, S = rq_slot_np(qp, np.zeros(dim, f32))
        assert np.array_equal(u, uu)
        codes = np.packbits(b.astype(np.uint8), bitorder="little")[None, :]
        add = f32(np.sum(o * o)); scale = f32(-2 * np.sum(o * o) / np.sum(np.abs(o)))
        est = rq_estimates_np(codes, np.array([add]), np.array([scale]), u, lo, delta, qq, S, dim)[0]
        true = float(np.sum((o - qp.astype(np.float64)) ** 2))
        assert abs(float(est) - true) <= 1e-5 * (float(add) + float(qq) + abs(true)) + 1e-5


def test_estimator_mean_signed_error_is_about_zero():
    rng = np.random.default_rng(13)
    dim, n = 256, 3000
    ix = random_rq_index(rng, n=n, dim=dim, nlist=1, empty=())
    ix.centroids[:] = 0
    codes, add, scale = rq_encode(ix.vectors, ix.centroids, np.zeros(n, np.int64), ix.rotation)
    rc = np.zeros(dim, f32)
    errs = []
    for _ in range(16):
        q = rng.standard_normal(dim).astype(f32)
        u, lo, delta, qq, S = rq_slot_np(rq_rotate_np(ix.rotation, q)[0], rc)
        est = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim).astype(np.float64)
        true = ((ix.vectors.astype(np.float64) - q) ** 2).sum(1)
        errs.append(np.mean((est - true) / true))
    assert abs(np.mean(errs)) < 0.01


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_trainer_invariants(metric):
    rng = np.random.default_rng(14)
    x = rng.standard_normal((600, 20)).astype(f32) * 3
    data = train_ivf_rq(x, num_partitions=4, distance_type=metric, max_iterations=3, sample_rate=64, keep_vectors=True)
    data.validate()
    P = data.rotation.astype(np.float64)
    assert np.allclose(P @ P.T, np.eye(20), atol=1e-6)
    rows = data.vectors / np.linalg.norm(data.vectors, axis=1, keepdims=True) if metric == "cosine" else data.vectors
    part = np.repeat(np.arange(4), np.diff(data.part_offsets.astype(np.int64)))
    o = (rows.astype(np.float32).astype(np.float64) - data.centroids[part].astype(np.float64)) @ P.T
    bits = np.unpackbits(data.codes, axis=1, bitorder="little")[:, :20]
    if metric == "l2":                                   # (cosine: torch's normalisation, not restated here)
        assert np.array_equal(bits, (o > 0).astype(np.uint8))
        assert np.allclose(data.add_factors, (o * o).sum(1), rtol=1e-6, atol=0)
        assert np.allclose(data.scale_factors, -2 * (o * o).sum(1) / np.abs(o).sum(1), rtol=1e-6, atol=0)
    else:
        assert np.mean(bits == (o > 0)) > 0.999
        assert np.allclose(data.add_factors, (o * o).sum(1), rtol=1e-5)
    assert sorted(data.row_ids.tolist()) == list(range(600))
    assert np.array_equal(data.rotation, rq_rotation(20))             # seeded
    with pytest.raises(ValueError, match="l2 and cosine"):
        train_ivf_rq(x, num_partitions=4, distance_type="dot")
    with pytest.raises(ValueError, match="num_bits"):
        train_ivf_rq(x, num_partitions=4, num_bits=2)


def test_create_index_ivf_rq_rejections(monkeypatch):
    opened = record_opens(monkeypatch)
    rng = np.random.default_rng(16)
    db = lancedb.connect("memory://")
    t = db.create_table("t", {"vector": rng.standard_normal((300, 8)).astype(f32)})
    with pytest.raises(ValueError, match="num_bits"):
        t.create_index(index_type="IVF_RQ")               # the legacy default of 8 is refused, not rebuilt as 1
    with pytest.raises(ValueError, match="num_bits"):
        t.create_index(index_type="IVF_RQ", num_bits=4)
    with pytest.raises(ValueError, match="l2 and cosine"):
        t.create_index(index_type="IVF_RQ", num_bits=1, metric="dot")
    with pytest.raises(NotImplementedError):
        t.create_index(index_type="IVF_FLAT")
    wide = db.create_table("w", {"vector": np.zeros((20, 4097), f32)})
    with pytest.raises(ValueError, match="4096"):
        wide.create_index(index_type="IVF_RQ", num_bits=1)
    schema = pa.schema([pa.field("bits", pa.list_(pa.uint8(), 4))])
    tb = db.create_table("b", pa.table({"bits": pa.FixedSizeListArray.from_arrays(
        pa.array(np.arange(40, dtype=np.uint8)), 4)}, schema=schema))
    with pytest.raises(NotImplementedError, match="binary"):
        tb.create_index(index_type="IVF_RQ", num_bits=1)
    mv = pa.array([[[1.0, 2.0], [3.0, 4.0]], [[5.0, 6.0]]], pa.list_(pa.list_(pa.float32(), 2)))
    tm = db.create_table("m", pa.table({"mv": mv}))
    with pytest.raises(NotImplementedError, match="multivector"):
        tm.create_index(index_type="IVF_RQ", num_bits=1)
    assert opened == []


def test_async_create_index_with_ivf_rq_config(monkeypatch):
    opened = record_opens(monkeypatch)
    rng = np.random.default_rng(17)

    async def run():
        db = await lancedb.connect_async("memory://")
        t = await db.create_table("t", {"vector": rng.standard_normal((300, 12)).astype(f32)})
        assert lancedb.IvfRq().num_bits == 1
        await t.create_index("vector", config=lancedb.IvfRq(distance_type="cosine", num_partitions=3, max_iterations=2),
                             accelerator=None)
        with pytest.raises(ValueError, match="num_bits"):
            await t.create_index("vector", config=lancedb.IvfRq(num_bits=2), accelerator=None)
        return await t.list_indices()

    assert asyncio.run(run())[0]["index_type"] == "IVF_RQ"
    assert [name for name, _ in opened] == ["GpuIvfRq"]
    assert opened[0][1].metric == "cosine" and opened[0][1].nlist == 3

"""IVF_SQ without a GPU: the C oracle against its NumPy mirror, the quantiser at and around its code boundaries, the
integer distance above 2^24, ties, the trainer, and the refusals of create_index(index_type="IVF_SQ") against a stubbed
native layer.  The build through create_index is in test_ivf_kinds_host.py."""
import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200.index import sq_encode, train_ivf_sq
from tests import sq_oracle
from tests.sq_oracle import random_sq_index
from tests.util import record_opens

f32 = np.float32


def boundary_values(lo, hi):
    """lo + j (hi - lo) / 255 for every j as f32, one f32 ulp either side, values outside [lo, hi], +-inf and NaN."""
    j = np.arange(256, dtype=np.float64)
    b = (lo + j * (hi - lo) / 255.0).astype(f32)
    vals = np.concatenate([b, np.nextafter(b, f32(-np.inf)), np.nextafter(b, f32(np.inf)),
                           np.array([lo - 1.0, hi + 1.0, lo - 1e30, hi + 1e30, np.inf, -np.inf, np.nan, -0.0, 0.0,
                                     np.finfo(f32).max, -np.finfo(f32).max], f32)])
    return vals


@pytest.mark.parametrize("lo,hi", [(-1.0, 1.0), (-0.37, 0.91), (0.0, 255.0), (3.0, 3.0 + 1e-3), (-1e30, 1e30)])
def test_quantiser_boundaries_c_numpy_and_builder_agree(lo, hi):
    lo, hi = float(f32(lo)), float(f32(hi))
    v = boundary_values(lo, hi)
    c = sq_oracle.sq_encode(v, lo, hi)
    assert np.array_equal(c, sq_oracle.sq_encode_np(v, lo, hi))
    assert np.array_equal(c, sq_encode(v, lo, hi))
    # the formula itself, element by element in Python floats (f64, left to right, truncation, saturation)
    for x, got in zip(v.tolist(), c.tolist()):
        t = (float(x) - lo) * 255.0 / (hi - lo)
        want = 0 if t != t or t <= 0 else (255 if t >= 255 else int(t))
        assert got == want, (x, got, want)
    with np.errstate(invalid="ignore"):
        assert c[np.isnan(v)].tolist() == [0] and c[v == np.inf].tolist() == [255] and c[v == -np.inf].tolist() == [0]


def test_quantiser_degenerate_range_is_all_zero():
    v = boundary_values(2.0, 3.0)
    for enc in (sq_oracle.sq_encode, sq_oracle.sq_encode_np, sq_encode):
        assert not enc(v, 2.5, 2.5).any()


def test_distance_above_2_24_is_rounded_to_nearest():
    # 258 x 255^2 + 25^2 + 12^2 = 2^24 + 3: rounds to 2^24 + 4 (truncation would give 2^24)
    a = np.zeros(300, np.uint8)
    b = np.zeros(300, np.uint8)
    a[:258] = 255
    a[258], a[259] = 25, 12
    assert sq_oracle.sq_distance(a, b) == f32(2 ** 24 + 4)
    assert sq_oracle.sq_distances_np(a[None], b)[0, 0] == f32(2 ** 24 + 4)
    # the largest sum the limit allows: 65536 x 255^2 < 2^32
    big = np.full(65536, 255, np.uint8)
    assert sq_oracle.sq_distance(big, np.zeros_like(big)) == f32(65536 * 65025)
    assert sq_oracle.sq_distances_np(big[None], np.zeros_like(big))[0, 0] == f32(65536 * 65025)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_c_oracle_equals_numpy_mirror(metric):
    rng = np.random.default_rng(3 if metric == "l2" else 4)
    ix = random_sq_index(rng, metric=metric)
    q = rng.standard_normal((9, ix.dim)).astype(f32)
    q[1] *= 50.0                                         # far outside the bounds: every code saturates
    q[2, 3] = np.nan                                     # no finite centroid distance: no rows
    q[3] = ix.vectors[4]                                 # ties among the duplicate rows
    allow = rng.random(ix.nrows * 3 + 7) < 0.3
    cases = [dict(k=10, nprobes=2), dict(k=1, nprobes=6), dict(k=700, nprobes=6), dict(k=5, nprobes=3, refine_factor=4),
             dict(k=8, nprobes=2, lower=50.0, upper=40000.0), dict(k=12, nprobes=1, allow=allow, max_nprobes=6),
             dict(k=4, nprobes=2, allow=allow)]
    for kw in cases:
        ci, cd, cc = sq_oracle.search(ix, q, nthreads=3, **kw)
        ni, nd, nc = sq_oracle.sq_search_np(ix, q, **kw)
        assert np.array_equal(cc, nc), kw
        assert np.array_equal(ci, ni), kw
        assert np.array_equal(cd.view(np.uint32), nd.view(np.uint32)), kw
        assert cc[2] == 0
        for b in range(q.shape[0]):                      # ascending by (_distance, _rowid)
            n = int(cc[b])
            keys = list(zip(cd[b, :n].tolist(), ci[b, :n].tolist()))
            assert keys == sorted(keys)


def test_ties_are_ordered_by_row_id():
    rng = np.random.default_rng(11)
    ix = random_sq_index(rng, n=200, dim=8, nlist=1, empty=())
    ix.codes[:] = 0
    ix.codes[::2, 0] = 3                                  # two distances only, 100 rows each
    q = np.full((1, 8), ix.lo, f32)
    ids, dist, cnt = sq_oracle.search(ix, q, k=150, nprobes=1)
    assert np.array_equal(ids[0, :100], np.sort(ix.row_ids[1::2])) and np.all(dist[0, :100] == 0)
    assert np.array_equal(ids[0, 100:150], np.sort(ix.row_ids[0::2])[:50]) and np.all(dist[0, 100:] == 9)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_trainer_encodes_rows_with_the_sample_bounds(metric):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((700, 20)).astype(f32) * 3
    data = train_ivf_sq(x, num_partitions=4, distance_type=metric, max_iterations=3, sample_rate=64, keep_vectors=True)
    data.validate()
    assert data.metric == metric and data.nlist == 4 and data.codes.shape == (700, 20)
    rows = data.vectors / np.linalg.norm(data.vectors, axis=1, keepdims=True) if metric == "cosine" else data.vectors
    assert data.lo >= float(rows.min()) - 1e-6 and data.hi <= float(rows.max()) + 1e-6
    if metric == "l2":                                   # (cosine: torch's normalisation, not restated here)
        assert np.array_equal(data.codes, sq_encode(rows, data.lo, data.hi))
    assert sorted(data.row_ids.tolist()) == list(range(700))
    with pytest.raises(ValueError, match="l2 and cosine"):
        train_ivf_sq(x, num_partitions=4, distance_type="dot")


def test_create_index_ivf_sq_rejections(monkeypatch):
    opened = record_opens(monkeypatch)
    rng = np.random.default_rng(7)
    db = lancedb.connect("memory://")
    t = db.create_table("t", {"vector": rng.standard_normal((300, 8)).astype(f32)})
    with pytest.raises(ValueError, match="num_bits"):
        t.create_index(index_type="IVF_SQ", num_bits=4)
    with pytest.raises(ValueError, match="l2 and cosine"):
        t.create_index(index_type="IVF_SQ", metric="dot")
    with pytest.raises(NotImplementedError):
        t.create_index(index_type="IVF_FLAT")
    schema = pa.schema([pa.field("bits", pa.list_(pa.uint8(), 4))])
    tb = db.create_table("b", pa.table({"bits": pa.FixedSizeListArray.from_arrays(
        pa.array(np.arange(40, dtype=np.uint8)), 4)}, schema=schema))
    with pytest.raises(NotImplementedError, match="binary"):
        tb.create_index(index_type="IVF_SQ")
    mv = pa.array([[[1.0, 2.0], [3.0, 4.0]], [[5.0, 6.0]]], pa.list_(pa.list_(pa.float32(), 2)))
    tm = db.create_table("m", pa.table({"mv": mv}))
    with pytest.raises(NotImplementedError, match="multivector"):
        tm.create_index(index_type="IVF_SQ")
    assert opened == []

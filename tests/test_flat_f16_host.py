"""Float16 vector columns without a GPU: which row type reaches the flat handles (float16 columns as float16, f32 and
f64 columns as f32, on the flat cache and on the unindexed tails), the refusal of an append whose rows do not have the
handle's type, and a CPU restatement of the fp16 tensor-core band (gemm.cu F16Dist, kernels.cuh tc_band) on adversarial
queries: components at fp16 rounding midpoints, subnormal fp16 components, magnitudes near 65504 and cancellation-heavy
rows.  The band holds on all of them, and a band without the query's rounding term does not."""
import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native

F32, F16 = np.float32, np.float16
DIM = 8


# ---- which rows reach the native handles ----
class _RecordingFlat:
    """Stands in for GpuFlat: records the dtype of every row array it is opened or appended with."""
    seen = []

    def __init__(self, vectors, row_ids=None, device=0):
        _RecordingFlat.seen.append(("open", np.asarray(vectors).dtype))
        self.nrows = len(vectors)

    def search(self, q, k=10, **kw):
        B = np.asarray(q).reshape(-1, DIM).shape[0]
        return np.zeros((B, k), np.uint64), np.zeros((B, k), F32), np.ones(B, np.uint32)

    def search_unindexed(self, tail, q, k=10, **kw):
        return self.search(q, k)

    def append(self, rows, row_ids=None):
        _RecordingFlat.seen.append(("append", np.asarray(rows).dtype))
        self.nrows += len(rows)

    def delete(self, ids):
        return len(ids)

    def close(self):
        pass


@pytest.fixture
def flat_stub(monkeypatch):
    _RecordingFlat.seen = []
    monkeypatch.setattr(_native, "GpuFlat", _RecordingFlat)
    return _RecordingFlat.seen


def _table(value_type, n=64, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, DIM)).astype(F32)
    schema = pa.schema([pa.field("id", pa.int64()), pa.field("vector", pa.list_(value_type, DIM))])
    data = pa.table({"id": np.arange(n), "vector": pa.FixedSizeListArray.from_arrays(
        pa.array(x.reshape(-1)).cast(value_type), DIM)}, schema=schema)
    return lancedb.connect().create_table("t", data), rng


@pytest.mark.parametrize("value_type,want", [(pa.float16(), F16), (pa.float32(), F32), (pa.float64(), F32)])
def test_flat_cache_and_its_appends_get_the_columns_row_type(flat_stub, value_type, want):
    t, rng = _table(value_type)
    t.search(np.zeros(DIM, F32)).limit(3).to_arrow()
    t.add({"id": [64, 65], "vector": rng.standard_normal((2, DIM)).tolist()})
    assert flat_stub == [("open", np.dtype(want)), ("append", np.dtype(want))]
    if want == F16:          # the rows are the column's own float16 values
        assert t._rows_of(t._data, "vector").dtype == F16


class _FakeIndex:
    metric = "l2"

    def __init__(self, *a, **kw):
        pass

    def search(self, q, k=10, **kw):
        return _RecordingFlat.search(self, q, k)

    def search_unindexed(self, tail, q, k=10, **kw):
        assert isinstance(tail, _RecordingFlat)
        return self.search(q, k)

    def close(self):
        pass


@pytest.mark.parametrize("value_type,want", [(pa.float16(), F16), (pa.float32(), F32), (pa.float64(), F32)])
def test_unindexed_tails_get_the_columns_row_type(flat_stub, monkeypatch, value_type, want):
    monkeypatch.setattr(_native, "GpuIvfPq", _FakeIndex)
    t, rng = _table(value_type, n=300)
    t.create_index(metric="l2", num_partitions=2, num_sub_vectors=2)
    t.add({"id": [300, 301], "vector": rng.standard_normal((2, DIM)).tolist()})          # _add opens the tail
    t.add({"id": [302], "vector": rng.standard_normal((1, DIM)).tolist()})               # ... and appends to it
    t.delete("id = 300")                                                                   # no reopen: a delete
    t._open_tail("vector", 300)                                                            # a reopen from the table
    assert flat_stub == [("open", np.dtype(want)), ("append", np.dtype(want)), ("open", np.dtype(want))]
    # the index itself keeps the f32 upcast (its refine vectors, its training rows)
    assert t._index_data["vector"].vectors.dtype == F32


@pytest.mark.parametrize("handle,rows", [(F16, F32), (F16, np.float64), (F32, F16)])
def test_append_of_rows_of_another_type_is_refused_before_the_native_call(monkeypatch, handle, rows):
    fl = _native.GpuFlat.__new__(_native.GpuFlat)
    fl.dtype, fl.dim, fl.nrows, fl._h = np.dtype(handle), DIM, 10, None
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native layer was called"))
    with pytest.raises(ValueError, match="needs rows of that type"):
        fl.append(np.zeros((2, DIM), rows))
    assert fl.nrows == 10


# ---- the fp16 band (kernels.cuh tc_band with gemm.cu F16Dist's r_q and r_X) ----
def f16_scores(q, X16):
    """S[x] = |x|^2 - 2 fp16(q).x over fp16 rows x: the products are exact in f32, the sum is rounded once to f32"""
    dot = (X16.astype(np.float64) @ q.astype(F16).astype(np.float64)).astype(F32)
    xn2 = (X16.astype(np.float64) ** 2).sum(1).astype(F32)
    return (xn2 - F32(2) * dot).astype(F32)


def f16_band(q, X16, query_term=True):
    """E_q for an fp16 handle: r_q = |fp16(q) - q|, r_X = max_x |fp16(x) - x| = 0 (the rows are fp16), xmax = max |x|;
    query_term=False drops r_q (a band that assumes the query is fp16-exact)"""
    q64, X64 = q.astype(np.float64), X16.astype(np.float64)
    qn = float(np.sqrt((q64 ** 2).sum()))
    xmax = float(np.sqrt((X64 ** 2).sum(1).max())) * 1.0001
    rq = float(np.sqrt(((q.astype(F16).astype(np.float64) - q64) ** 2).sum())) if query_term else 0.0
    rx = float(np.sqrt(((X16.astype(F32).astype(F16).astype(np.float64) - X64) ** 2).sum(1).max()))
    assert rx == 0.0
    return 2.0 * ((qn + rq) * rx + rq * xmax) * (1.0 + 2.0 ** -10) + 4.0 * q.shape[0] * 2.0 ** -24 * (qn + xmax) ** 2


def f16_midpoint_neighbours(h):
    """For nonzero fp16 values h (normal or subnormal): the f32 values one f32 ulp either side of the midpoint between
    |h| and the next fp16 magnitude, signed like h; the first rounds to h, the second away from zero"""
    a = np.abs(np.asarray(h, F16))
    nxt = np.nextafter(a, F16(np.inf))
    mid = ((a.astype(np.float64) + nxt.astype(np.float64)) / 2).astype(F32)        # exact in f32
    s = np.sign(np.asarray(h, F32))
    return s * np.nextafter(mid, F32(0)), s * np.nextafter(mid, F32(np.inf))


def adversarial_cases(rng, d=64, n=256):
    """(name, q f32 [d], X16 fp16 [n, d]) with the query's rounding error lined up against the rows"""
    cases = []
    for scale in (1.0, 2.0 ** -20, 6.0e4):            # normal, subnormal fp16, near 65504
        h = (rng.uniform(0.5, 1.0, d) * scale).astype(F16)
        h[h == 0] = F16(2.0 ** -24)
        lo, hi = f16_midpoint_neighbours(h)
        q = np.where(rng.random(d) < 0.5, lo, hi).astype(F32)
        err_sign = np.sign(q.astype(F16).astype(np.float64) - q)       # where fp16(q) lands relative to q
        X = (np.abs(h.astype(F32))[None, :] * err_sign[None, :] * rng.uniform(0.5, 1.0, (n, d))).astype(F16)
        cases.append((f"midpoints x{scale:g}", q, X))
    # cancellation: rows within a few fp16 ulps of the query, so |q - x|^2 is tiny against |q|^2 and |x|^2
    base = rng.uniform(-1, 1, d).astype(F16)
    lo, hi = f16_midpoint_neighbours(np.where(base == 0, F16(1), base))
    q = hi.astype(F32)
    X = (base[None, :].astype(F32) + rng.integers(-3, 4, (n, d)) * np.abs(base).astype(F32) * 2.0 ** -10).astype(F16)
    cases.append(("cancellation", q, X))
    return cases


def test_fp16_band_holds_on_adversarial_queries_and_a_band_without_the_query_term_does_not():
    rng = np.random.default_rng(7)
    worst_full, worst_noq = 0.0, 0.0
    for name, q, X16 in adversarial_cases(rng):
        assert np.isfinite(q.astype(F16)).all(), name
        S = f16_scores(q, X16).astype(np.float64)
        q64, X64 = q.astype(np.float64), X16.astype(np.float64)
        exact = ((q64[None, :] - X64) ** 2).sum(1) - (q64 ** 2).sum()
        err = float(np.abs(S - exact).max())
        full, noq = f16_band(q, X16), f16_band(q, X16, query_term=False)
        assert err <= full, (name, err, full)
        worst_full = max(worst_full, err / full)
        worst_noq = max(worst_noq, err / noq)
    assert worst_full <= 1.0
    assert worst_noq > 1.0                    # the query's fp16 rounding is what the band has to carry


def test_a_query_beyond_fp16_range_has_no_finite_band():
    q = np.full(DIM, 1.0, F32)
    q[3] = 65520.0                            # rounds to inf in fp16: the query goes to the exact kernels
    rq = np.sqrt(((q.astype(F16).astype(np.float64) - q.astype(np.float64)) ** 2).sum())
    assert not np.isfinite(rq)
    q[3] = 65519.0                            # still rounds to 65504: finite
    assert np.isfinite(q.astype(F16)).all()

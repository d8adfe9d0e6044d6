"""GpuMultivec.append and Table.add on multivector columns, without a device: the append's checks run before any native
call, Table.add grows the open multivector cache in place (with the new ids once rows were deleted) instead of
reopening it, and a failed append drops the cache so that the next search reopens it."""
import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200
from lancedb_b200 import _native
from tests.multivec_oracle import flat_search_mv, offsets_of


class _NoNative:
    def __getattr__(self, name):
        raise AssertionError(f"native call {name} before the checks")


def _handle(dtype, dim=4):
    mv = _native.GpuMultivec.__new__(_native.GpuMultivec)    # the checks need no device
    mv.dtype, mv.dim, mv.nrows, mv._h = np.dtype(dtype), dim, 3, None
    return mv


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_append_checks_shapes_offsets_and_row_type_before_the_device(dtype, monkeypatch):
    monkeypatch.setattr(_native, "load", lambda: _NoNative())
    mv = _handle(dtype)
    other = np.float16 if dtype == np.float32 else np.float32
    good = np.zeros((3, 4), dtype)
    cases = [
        (np.zeros((3, 4), other), [0, 1, 3], "needs values of that type"),
        (np.zeros(12, dtype), [0, 12], "\\[vectors, dim\\]"),
        (np.zeros((3, 5), dtype), [0, 1, 3], "dimension 4"),
        (good, [0, 1, 2], "end at the number of vectors"),
        (good, [1, 2, 3], "start at 0"),
        (good, [0, 2, 1, 3], "must not decrease"),
        (good, [[0, 3]], "\\[rows \\+ 1\\]"),
    ]
    for vals, off, msg in cases:
        with pytest.raises(ValueError, match=msg):
            mv.append(vals, off)
    long_row = _handle(dtype, dim=1)
    with pytest.raises(ValueError, match="at most"):
        long_row.append(np.zeros(((1 << 20) + 1, 1), dtype), [0, (1 << 20) + 1])
    with pytest.raises(ValueError, match="one id per appended row"):
        mv.append(good, [0, 1, 3], row_ids=[5])
    assert mv.nrows == 3


class _StubMultivec:
    """GpuMultivec on the C oracle, recording opens and appends; `fail` makes the next append raise."""
    opens, appends, fail = [], [], False

    def __init__(self, values, offsets, row_ids=None, device=0):
        self.values, self.offsets = np.asarray(values, np.float32), np.asarray(offsets, np.uint64)
        self.row_ids = None if row_ids is None else np.asarray(row_ids, np.uint64)
        self.dim, self.nrows, self.closed, self.deleted = self.values.shape[1], self.offsets.size - 1, False, set()
        _StubMultivec.opens.append(self)

    def append(self, values, offsets, row_ids=None):
        _StubMultivec.appends.append((np.asarray(values).copy(), np.asarray(offsets).copy(),
                                      None if row_ids is None else np.asarray(row_ids).copy()))
        if _StubMultivec.fail:
            raise ValueError("append refused")
        if row_ids is not None and self.row_ids is None:
            self.row_ids = np.arange(self.nrows, dtype=np.uint64)
        if self.row_ids is not None:
            self.row_ids = np.concatenate([self.row_ids, np.asarray(row_ids, np.uint64)])
        self.offsets = np.concatenate([self.offsets, self.offsets[-1] + np.asarray(offsets, np.uint64)[1:]])
        self.values = np.concatenate([self.values, np.asarray(values, np.float32)])
        self.nrows = self.offsets.size - 1

    def search(self, queries, k=10, q_offsets=None, lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        q = np.concatenate([np.asarray(a, np.float32).reshape(-1, self.dim) for a in queries])
        ids = np.arange(self.nrows) if self.row_ids is None else self.row_ids
        mask = np.ones(int(ids.max()) + 1 if ids.size else 0, bool)
        if allow is not None:
            bits = np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")[:allow_bits] > 0
            mask = np.zeros(max(mask.size, bits.size), bool)
            mask[:bits.size] = bits
        mask[[i for i in self.deleted if i < mask.size]] = False
        return flat_search_mv(self.values, self.offsets, q, [0, q.shape[0]], k, row_ids=self.row_ids, lower=lower,
                              upper=upper, allow=mask)

    def delete(self, ids):
        self.deleted |= set(int(i) for i in ids)
        return len(ids)

    def close(self):
        self.closed = True


@pytest.fixture
def stub(monkeypatch):
    _StubMultivec.opens, _StubMultivec.appends, _StubMultivec.fail = [], [], False
    monkeypatch.setattr(_native, "GpuMultivec", _StubMultivec)
    return _StubMultivec


def _rows(rng, n, dim=2):
    return [rng.standard_normal((int(m), dim)).tolist() for m in rng.integers(0, 4, n)]


def _table(data, vt=pa.float32()):
    return lancedb_b200.connect().create_table("t", pa.table({
        "id": pa.array(np.arange(len(data))), "vector": pa.array(data, type=pa.list_(pa.list_(vt, 2)))}))


def _add(t, data, start, vt=pa.float32()):
    t.add(pa.table({"id": pa.array(np.arange(start, start + len(data))),
                    "vector": pa.array(data, type=pa.list_(pa.list_(vt, 2)))}))


@pytest.mark.parametrize("vt", [pa.float32(), pa.float16()])
def test_table_add_appends_to_the_open_cache_instead_of_reopening_it(stub, vt):
    rng = np.random.default_rng(1)
    a, b, c = _rows(rng, 40), _rows(rng, 7), _rows(rng, 5)
    t = _table(a, vt)
    _add(t, b, 40, vt)                                          # no cache open yet: nothing to grow
    assert stub.appends == []
    t.search([[1.0, 0.5]]).to_arrow()
    assert len(stub.opens) == 1
    _add(t, c, 47, vt)
    assert len(stub.opens) == 1 and len(stub.appends) == 1
    vals, off, rid = stub.appends[0]
    assert vals.dtype == (np.float16 if vt == pa.float16() else np.float32)
    assert list(off) == list(offsets_of([len(r) for r in c])) and rid is None
    assert np.array_equal(vals.astype(np.float32), np.asarray([v for r in c for v in r], vt.to_pandas_dtype())
                          .astype(np.float32).reshape(-1, 2))
    t.delete("id < 3")                                          # the cache is told, and appends now pass ids
    _add(t, b, 52, vt)
    assert len(stub.opens) == 1 and list(stub.appends[1][2]) == list(range(52, 59))
    got = t.search([[1.0, 0.5]]).limit(100).with_row_id(True).to_arrow()
    fresh = _table(a + b + c + b, vt)
    fresh.delete("id < 3")
    want = fresh.search([[1.0, 0.5]]).limit(100).with_row_id(True).to_arrow()
    assert got["_rowid"].to_pylist() == want["_rowid"].to_pylist()
    assert got["_distance"].to_pylist() == want["_distance"].to_pylist()


def test_a_failed_append_drops_the_cache(stub):
    rng = np.random.default_rng(2)
    t = _table(_rows(rng, 30))
    t.search([[1.0, 0.5]]).to_arrow()
    cache = stub.opens[0]
    stub.fail = True
    with pytest.raises(ValueError, match="append refused"):
        _add(t, _rows(rng, 4), 30)
    assert cache.closed and "vector" not in t._multivec
    stub.fail = False
    t.search([[1.0, 0.5]]).to_arrow()                           # reopened from the table's rows
    assert len(stub.opens) == 2 and stub.opens[1].nrows == t._data.num_rows


def test_a_row_holding_a_null_vector_refuses_the_add_and_changes_nothing(stub):
    rng = np.random.default_rng(3)
    a = _rows(rng, 20)
    t = _table(a)
    before = t.search([[1.0, 0.5]]).limit(50).with_row_id(True).to_arrow()
    cache, version = stub.opens[0], t.version
    bad = pa.table({"id": pa.array([20, 21]),
                    "vector": pa.array([[[1.0, 2.0]], [[3.0, 4.0], None]], type=pa.list_(pa.list_(pa.float32(), 2)))})
    with pytest.raises(ValueError, match="null vector"):
        t.add(bad)
    assert t._data.num_rows == 20 and t.version == version and stub.appends == []
    assert t._multivec["vector"] is cache and not cache.closed and cache.nrows == 20
    after = t.search([[1.0, 0.5]]).limit(50).with_row_id(True).to_arrow()
    assert after.equals(before)
    _add(t, _rows(rng, 3), 20)                                  # a good add still grows the cache
    assert cache.nrows == 23 and t._data.num_rows == 23

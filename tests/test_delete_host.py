"""Deleting rows, without a GPU: Table.delete against the reference's known answers (python/python/tests/
test_table.py:2260-2293 and the docstring of python/python/lancedb/table.py:1672-1720), eight threads deleting at
once, refusals, add / index_stats / create_index after a delete, the rollback of a delete that fails in a handle, the
async surface, and IndexData.compact for every kind in IVF_KINDS against the kind's arrays filtered in NumPy.  The
native handles are replaced by exact NumPy stand-ins that honour their deleted rows as lgpu_*_delete does."""
import asyncio
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS
from lancedb_b200.table import DeleteResult

from tests.test_unindexed_host import CASES, _stub_assign

NBYTES = 4


class _Exact:
    """A native handle stand-in: exact search (L2 over floats, Hamming over bytes) of its rows by (_distance, _rowid),
    leaving out the ids outside `allow` and the ids it was told were deleted."""
    log = []
    fail_delete = None          # a class name whose delete raises

    def __init__(self, data=None, row_ids=None, device=0):
        if hasattr(data, "row_ids"):            # an IndexData: its rows, as lgpu_*_open takes them
            self.x, self.ids = np.asarray(data.vectors), np.asarray(data.row_ids, np.uint64)
            self.metric = data.metric
        else:
            self.x = np.asarray(data)
            self.ids = np.arange(len(self.x), dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
            self.metric = "l2"
        self.dead = set()
        _Exact.log.append(("open", type(self).__name__, len(self.ids)))

    def delete(self, ids):
        _Exact.log.append(("delete", type(self).__name__, sorted(int(i) for i in ids)))
        if _Exact.fail_delete == type(self).__name__:
            raise RuntimeError("injected delete failure")
        held = set(int(i) for i in self.ids)
        new = {int(i) for i in ids if int(i) in held} - self.dead
        self.dead |= new
        return len(new)

    def append(self, rows, row_ids=None):
        n = len(rows)
        ids = np.arange(len(self.ids), len(self.ids) + n, dtype=np.uint64) if row_ids is None else row_ids
        self.x = np.concatenate([self.x, np.asarray(rows, self.x.dtype)])
        self.ids = np.concatenate([self.ids, np.asarray(ids, np.uint64)])

    def search(self, q, k=10, allow=None, allow_bits=0, max_nprobes=0, **kw):
        _Exact.log.append(("search", type(self).__name__, max_nprobes))
        q = np.asarray(q).reshape(-1, self.x.shape[1])
        if self.x.dtype == np.uint8:
            d = np.unpackbits(q[:, None, :] ^ self.x[None], axis=2).sum(axis=2).astype(np.float32)
        else:
            d = ((q[:, None, :].astype(np.float64) - self.x[None]) ** 2).sum(axis=2).astype(np.float32)
        ok = np.array([int(i) not in self.dead for i in self.ids], bool)
        if allow is not None:
            bm = np.asarray(allow, np.uint32)
            ok &= np.array([i < allow_bits and (int(bm[i >> 5]) >> (i & 31)) & 1 for i in self.ids.astype(np.int64)],
                           bool)
        B = q.shape[0]
        ids, dist, cnt = np.zeros((B, k), np.uint64), np.zeros((B, k), np.float32), np.zeros(B, np.uint32)
        for b in range(B):
            rows = np.nonzero(ok)[0]
            rows = rows[np.lexsort((self.ids[rows], d[b, rows]))][:k]
            cnt[b] = rows.size
            ids[b, :rows.size], dist[b, :rows.size] = self.ids[rows], d[b, rows]
        return ids, dist, cnt

    def search_unindexed(self, tail, q, k=10, **kw):
        a, b = self.search(q, k, **kw), tail.search(q, k, **kw)
        ids, dist = np.concatenate([a[0], b[0]], 1), np.concatenate([a[1], b[1]], 1)
        out = [np.zeros((len(a[2]), k), np.uint64), np.zeros((len(a[2]), k), np.float32), np.zeros(len(a[2]), np.uint32)]
        for r in range(len(a[2])):
            cols = [c for c in range(2 * k) if c % k < (a[2][r] if c < k else b[2][r])]
            cols = sorted(cols, key=lambda c: (dist[r, c], ids[r, c]))[:k]
            out[2][r] = len(cols)
            out[0][r, :len(cols)], out[1][r, :len(cols)] = ids[r, cols], dist[r, cols]
        return tuple(out)

    def close(self):
        pass


class ExactIvf(_Exact):
    pass


class ExactFlat(_Exact):
    pass


class ExactBinary(_Exact):
    pass


@pytest.fixture
def exact_native(monkeypatch):
    _Exact.log, _Exact.fail_delete = [], None
    monkeypatch.setattr(_native, "GpuIvfBinary", ExactIvf)
    monkeypatch.setattr(_native, "GpuBinary", ExactBinary)
    monkeypatch.setattr(_native, "GpuFlat", ExactFlat)
    return _Exact.log


def _binary_table(n=60, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256, (n, NBYTES)).astype(np.uint8)
    schema = pa.schema([pa.field("id", pa.int64()), pa.field("vector", pa.list_(pa.uint8(), NBYTES))])
    return lancedb.connect().create_table("t", {"id": np.arange(n), "vector": x}, schema=schema), x


def test_delete_known_answers():
    # python/python/tests/test_table.py:2260-2272
    t = lancedb.connect().create_table("my_table", data=[{"vector": [1.1, 0.9], "id": 0},
                                                         {"vector": [1.2, 1.9], "id": 1}])
    assert len(t) == 2 and t.version == 1
    res = t.delete("id=0")
    assert res.version == 2 and t.version == 2
    assert len(t) == 1 and t.count_rows() == 1
    assert t.to_arrow()["id"].to_pylist() == [1]
    # the docstring of python/python/lancedb/table.py:1672-1720
    t = lancedb.connect().create_table("my_table", [{"x": 1, "vector": [1.0, 2]}, {"x": 2, "vector": [3.0, 4]},
                                                    {"x": 3, "vector": [5.0, 6]}])
    res = t.delete("x = 2")
    assert res == DeleteResult(num_deleted_rows=1, version=2)
    assert repr(res) == "DeleteResult(num_deleted_rows=1, version=2)"
    assert t.to_pandas()["x"].tolist() == [1, 3]
    to_remove = ", ".join(str(v) for v in [1, 5])
    assert t.delete(f"x IN ({to_remove})") == DeleteResult(num_deleted_rows=1, version=3)
    assert t.to_pandas()["x"].tolist() == [3]
    assert t.delete("x = 2") == DeleteResult(num_deleted_rows=0, version=3)     # nothing matched: same version


def test_concurrent_deletes_are_thread_safe():
    # python/python/tests/test_table.py:2275-2293
    num_workers = 8
    t = lancedb.connect().create_table("my_table", data=[{"id": r} for r in range(num_workers)])
    barrier = threading.Barrier(num_workers)

    def delete(row_id):
        barrier.wait()
        return t.delete(f"id = {row_id}")

    with ThreadPoolExecutor(max_workers=num_workers) as pool:
        results = list(pool.map(delete, range(num_workers)))
    assert all(r.num_deleted_rows == 1 for r in results)
    assert sorted(r.version for r in results) == list(range(2, num_workers + 2))
    assert t.count_rows() == 0


def test_delete_refuses_empty_and_unparsable_predicates():
    t = lancedb.connect().create_table("t", data=[{"id": r} for r in range(4)])
    for bad in ("", "   ", None):
        with pytest.raises(ValueError):
            t.delete(bad)
    with pytest.raises(ValueError):
        t.delete("id = = 2")
    assert t.count_rows() == 4 and t.version == 1


def test_search_leaves_deleted_rows_out(exact_native):
    t, x = _binary_table()
    q = x[7]
    before = t.search(q).limit(5).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert before[0] == 7
    assert t.delete("id = 7 OR id = 3").num_deleted_rows == 2
    assert ("delete", "ExactBinary", [3, 7]) in exact_native       # the flat cache was told
    got = t.search(q).limit(5).with_row_id(True).to_arrow()
    assert 7 not in got["_rowid"].to_pylist() and 3 not in got["_rowid"].to_pylist()
    assert got["id"].to_pylist() == got["_rowid"].to_pylist()       # ids stay positions
    # a where clause is ANDed with the live rows; the plain query shows live rows with their _rowid
    got = t.search(q).where("id < 10").limit(20).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert sorted(got) == [0, 1, 2, 4, 5, 6, 8, 9]
    assert t.to_arrow()["id"].to_pylist() == [i for i in range(60) if i not in (3, 7)]
    # everything deleted: a search returns no rows
    t.delete("true")
    assert t.count_rows() == 0 and t.search(q).limit(5).to_arrow().num_rows == 0


def test_add_stats_and_create_index_after_delete(exact_native, monkeypatch):
    t, x = _binary_table()
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector",
                   max_iterations=2)
    t.delete("id >= 50")
    assert ("delete", "ExactIvf", list(range(50, 60))) in exact_native
    st = t.index_stats("vector_idx")
    assert st["num_indexed_rows"] == 50 and st["num_unindexed_rows"] == 0
    # every request on a table with deletions is prefiltered: maximum_nprobes reaches the handle
    exact_native.clear()
    t.search(x[0]).maximum_nprobes(29).to_arrow()
    assert ("search", "ExactIvf", 29) in exact_native
    rng = np.random.default_rng(1)
    t.add({"id": [60, 61], "vector": rng.integers(0, 256, (2, NBYTES))})
    assert t.version == 3 and t.count_rows() == 52
    assert t.index_stats("vector_idx")["num_unindexed_rows"] == 2
    assert t.to_arrow()["id"].to_pylist()[-2:] == [60, 61]
    t.delete("id = 61 OR id = 2")                   # one row in the tail, one in the index
    assert ("delete", "ExactBinary", [61]) in exact_native and ("delete", "ExactIvf", [2]) in exact_native
    st = t.index_stats("vector_idx")
    assert st["num_indexed_rows"] == 49 and st["num_unindexed_rows"] == 1
    # a new index trains on the live rows, which keep their positions as row ids
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector",
                   max_iterations=2)
    live = [i for i in range(62) if not (50 <= i < 60 or i in (2, 61))]
    assert sorted(t._index_data["vector"].row_ids.tolist()) == live
    got = t.search(x[3]).limit(60).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert sorted(got) == live


@pytest.mark.parametrize("indexed", [False, True])
@pytest.mark.parametrize("cache_first", [False, True])
def test_rows_added_after_a_delete_take_the_next_positions(exact_native, indexed, cache_first):
    """Row ids are positions, tombstones included: rows added after a delete follow the last row, in the tail and in
    the flat caches (opened before the delete, or over the live rows after it), and a later delete reaches them."""
    t, x = _binary_table()
    if indexed:
        t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector",
                       max_iterations=2)
    if cache_first:
        t.search(x[0]).bypass_vector_index().to_arrow()            # the flat cache, opened before the delete
    t.delete("id >= 50")
    if not cache_first:
        t.search(x[0]).bypass_vector_index().to_arrow()            # ... or after it, over the live rows
    new = np.array([[255, 255, 255, 255], [0, 255, 0, 255]], np.uint8)
    t.add({"id": [60, 61], "vector": new})
    assert t.to_arrow()["id"].to_pylist()[-2:] == [60, 61]
    if indexed:
        assert t._tail_from["vector"] == 60 and t._tail["vector"].ids.tolist() == [60, 61]
    for bypass in (False, True):
        for want, q in zip((60, 61), new):
            b = t.search(q).limit(3).with_row_id(True)
            got = (b.bypass_vector_index() if bypass else b).to_arrow()
            assert got["_rowid"].to_pylist()[0] == want and got["id"].to_pylist()[0] == want
            assert got["_distance"].to_pylist()[0] == 0
            assert not set(got["_rowid"].to_pylist()) & set(range(50, 60))    # deleted rows stay deleted
    assert t.delete("id = 61").num_deleted_rows == 1
    for bypass in (False, True):
        b = t.search(new[1]).limit(70).with_row_id(True)
        got = (b.bypass_vector_index() if bypass else b).to_arrow()["_rowid"].to_pylist()
        assert sorted(got) == list(range(50)) + [60]
    if indexed:
        assert t._tail["vector"].dead == {61}


def test_optimize_drops_deleted_rows_from_every_handle(exact_native):
    t, x = _binary_table()
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector",
                   max_iterations=2)
    t.add({"id": [60, 61, 62], "vector": x[:3]})
    t.delete("id = 1 OR id = 61")
    t.optimize()
    d = t._index_data["vector"]
    live = [i for i in range(63) if i not in (1, 61)]
    assert sorted(d.row_ids.tolist()) == live and not t._tail
    assert t._index["vector"].dead == set()          # nothing left to filter out
    st = t.index_stats("vector_idx")
    assert st["num_indexed_rows"] == 61 and st["num_unindexed_rows"] == 0
    assert t.to_arrow()["id"].to_pylist() == live    # host rows are not rewritten: ids are stable
    # the flat cache reopens over the live rows, with their positions as ids
    got = t.search(x[5]).bypass_vector_index().limit(70).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert sorted(got) == live


def test_failed_delete_leaves_table_and_handles_as_they_were(exact_native):
    t, x = _binary_table()
    t.create_index(metric="hamming", num_partitions=4, index_type="IVF_FLAT", vector_column_name="vector",
                   max_iterations=2)
    t.add({"id": [60, 61], "vector": x[:2]})
    t.delete("id = 4")                                # an earlier tombstone the reopened handle must get back
    ix, tail = t._index["vector"], t._tail["vector"]
    _Exact.fail_delete = "ExactBinary"                # the index takes the delete, then the tail fails
    with pytest.raises(RuntimeError, match="injected"):
        t.delete("id = 5 OR id = 60")
    _Exact.fail_delete = None
    assert t.version == 3 and t.count_rows() == 61
    assert t._index["vector"] is not ix and t._index["vector"].dead == {4}          # reopened, tombstones reapplied
    assert t._tail["vector"].dead == set() and t._tail_from["vector"] == 60
    got = t.search(x[5]).limit(70).with_row_id(True).to_arrow()["_rowid"].to_pylist()
    assert sorted(got) == [i for i in range(62) if i != 4]
    assert t.delete("id = 5 OR id = 60").num_deleted_rows == 2


def test_async_delete(exact_native):
    async def run():
        db = await lancedb.connect_async()
        t = await db.create_table("a", data=[{"id": r, "vector": [float(r), 0.0]} for r in range(6)])
        res = await t.delete("id > 3")
        assert res == DeleteResult(2, 2)
        assert await t.count_rows() == 4 and await t.count_rows("id >= 2") == 2
        rows = await t.query().with_row_id().to_arrow()
        assert rows["_rowid"].to_pylist() == [0, 1, 2, 3]
        got = await t.vector_search([5.0, 0.0]).limit(10).to_arrow()
        assert sorted(got["id"].to_pylist()) == [0, 1, 2, 3]
    asyncio.run(run())


@pytest.mark.parametrize("kind,metric,params", CASES, ids=[c[0] + "-" + c[1] for c in CASES])
def test_compact_drops_rows_and_keeps_the_rest(monkeypatch, kind, metric, params):
    _stub_assign(monkeypatch)
    rng = np.random.default_rng(5)
    binary = kind == "IVF_FLAT"
    n = 300
    x = rng.integers(0, 256, (n, NBYTES)).astype(np.uint8) if binary else rng.standard_normal((n, 16)).astype(np.float32)
    kw = {} if binary else dict(keep_vectors=True)
    d = IVF_KINDS[kind].train(x, num_partitions=5, distance_type=metric, max_iterations=3, **kw, **params)
    keep = rng.random(n) > 0.3
    keep[d.part_offsets[1]:d.part_offsets[2]] = False            # one partition loses every row
    c = d.compact(keep)
    c.validate()
    off, new = d.part_offsets.astype(np.int64), c.part_offsets.astype(np.int64)
    part = np.repeat(np.arange(d.nlist), np.diff(off))
    assert np.array_equal(np.diff(new), np.bincount(part[keep], minlength=d.nlist))
    assert np.array_equal(c.row_ids, d.row_ids[keep])
    if kind == "IVF_PQ":
        assert np.array_equal(c.row_codes(), d.row_codes()[keep])
        for p in range(d.nlist):                                  # the transposed [w][n_p] layout of each partition
            assert np.array_equal(c.partition_codes(p), d.row_codes()[keep][new[p]:new[p + 1]].T)
        assert np.array_equal(c.vectors, d.vectors[keep])
    elif kind in ("IVF_SQ", "IVF_HNSW_SQ"):
        sq, dsq = getattr(c, "sq", c), getattr(d, "sq", d)
        assert np.array_equal(sq.codes, dsq.codes[keep]) and np.array_equal(sq.vectors, dsq.vectors[keep])
        assert (sq.lo, sq.hi) == (dsq.lo, dsq.hi)
        if kind == "IVF_HNSW_SQ":                                 # graphs rebuilt where rows left, kept elsewhere
            for p in range(d.nlist):
                if np.diff(new)[p] == np.diff(off)[p]:
                    assert np.array_equal(c.adj0[new[p]:new[p + 1]], d.adj0[off[p]:off[p + 1]])
    elif kind == "IVF_RQ":
        for f in ("codes", "add_factors", "scale_factors", "vectors"):
            assert np.array_equal(getattr(c, f), getattr(d, f)[keep])
    else:
        assert np.array_equal(c.vectors, d.vectors[keep])
    with pytest.raises(ValueError, match="one flag per row"):
        d.compact(keep[:-1])

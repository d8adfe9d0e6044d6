"""Binary IVF_FLAT (hamming) on the CPU: the C oracle against its NumPy mirror, the k-modes trainer, and the Python
surface (create_index / list_indices / index_stats / rejections / aio.IvfFlat) against a stubbed native layer."""
import asyncio

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from lancedb_b200.index import IvfBinaryIndexData, kmodes_assign, kmodes_update, train_ivf_binary
from tests import ivf_binary_oracle as O
from tests.hamming_oracle import flat_search_u8_np


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("nbytes", [1, 3, 32, 33, 128])
@pytest.mark.parametrize("patterns", [0, 16])
def test_oracle_matches_numpy(nbytes, patterns):
    rng = np.random.default_rng(100 + nbytes + patterns)
    data = O.random_index(rng, 700, nbytes, 9, empty=(0, 4), patterns=patterns)
    q = rng.integers(0, 256, (11, nbytes), dtype=np.uint8)
    allow = rng.random(700) < 0.03
    cases = [dict(k=10, nprobes=2), dict(k=1, nprobes=1), dict(k=900, nprobes=4),       # k > N probed
             dict(k=10, nprobes=50),                                                   # nprobes > nlist
             dict(k=8, nprobes=2, lower=2, upper=4 * nbytes),
             dict(k=20, nprobes=1, allow=allow), dict(k=20, nprobes=1, allow=allow, max_nprobes=6)]
    for kw in cases:
        assert _same(O.search(data, q, nthreads=3, **kw), O.search_np(data, q, **kw)), kw


def test_oracle_all_equal_rows_and_empty_index():
    rng = np.random.default_rng(1)
    x = np.full((300, 16), 0x5a, np.uint8)
    data = O.index_from_assignment(x, rng.integers(0, 256, (4, 16), dtype=np.uint8), rng.integers(0, 4, 300))
    q = rng.integers(0, 256, (5, 16), dtype=np.uint8)
    ids, dist, cnt = O.search(data, q, k=30, nprobes=4)
    assert _same((ids, dist, cnt), O.search_np(data, q, k=30, nprobes=4))
    assert np.array_equal(ids, np.tile(np.arange(30, dtype=np.uint64), (5, 1)))       # every row ties: ids decide
    empty = O.index_from_assignment(np.zeros((0, 16), np.uint8), x[:3], np.zeros(0, np.int64))
    ids, dist, cnt = O.search(empty, q, k=3, nprobes=2)
    assert np.all(cnt == 0) and np.all(ids == O.U64_MAX) and np.all(np.isinf(dist))


@pytest.mark.parametrize("nbytes", [1, 33])
def test_all_probes_equal_flat_search(nbytes):
    rng = np.random.default_rng(2)
    data = O.random_index(rng, 400, nbytes, 6, patterns=8, row_ids=rng.permutation(1000)[:400])
    q = rng.integers(0, 256, (7, nbytes), dtype=np.uint8)
    flat = flat_search_u8_np(data.vectors, q, 25, row_ids=data.row_ids)
    assert _same(O.search(data, q, k=25, nprobes=6), flat)


def test_kmodes_majority_and_tie_rules():
    # 4-bit rows as one byte each; cluster 0 = {0b0011, 0b0001, 0b0111}: bit 0 in 3/3, bit 1 in 2/3, bit 2 in 1/3 -> 0b0011
    # cluster 1 = {0b1000, 0b1100}: bit 3 in 2/2, bit 2 in 1/2 (an exact half keeps 0) -> 0b1000; cluster 2 is empty
    x = np.array([[0b0011], [0b0001], [0b0111], [0b1000], [0b1100]], np.uint8)
    c = np.array([[0b0000], [0b1111], [0b11110000]], np.uint8)
    new = kmodes_update(x, np.array([0, 0, 0, 1, 1]), c)
    assert new.tolist() == [[0b0011], [0b1000], [0b11110000]]
    # ties go to the lowest centroid index: 0b0011 is 1 bit from both 0b0001 and 0b0111
    assert kmodes_assign(np.array([[0b0011]], np.uint8), np.array([[0b0111], [0b0001]], np.uint8)).tolist() == [0]
    assert kmodes_assign(np.array([[0b0011]], np.uint8), np.array([[0b0001], [0b0111]], np.uint8)).tolist() == [0]
    # one full round (assign, then update) against the NumPy mirror
    ref_c, _ = O.kmodes_np(x, c, 1)
    assert np.array_equal(ref_c, kmodes_update(x, kmodes_assign(x, c), c))


def test_trainer_matches_numpy_mirror_and_is_seeded():
    rng = np.random.default_rng(3)
    pats = rng.integers(0, 256, (12, 8), dtype=np.uint8)
    x = pats[rng.integers(0, 12, 2000)] ^ (rng.random((2000, 8)) < 0.05).astype(np.uint8)
    a = train_ivf_binary(x, num_partitions=6, max_iterations=7, sample_rate=64, seed=5)
    b = train_ivf_binary(x, num_partitions=6, max_iterations=7, sample_rate=64, seed=5)
    c = train_ivf_binary(x, num_partitions=6, max_iterations=7, sample_rate=64, seed=6)
    assert all(np.array_equal(getattr(a, f), getattr(b, f)) for f in ("centroids", "part_offsets", "vectors", "row_ids"))
    assert not np.array_equal(a.centroids, c.centroids)
    # restate the trainer: the same sample and initial rows, then kmodes_np
    g = np.random.default_rng(5)
    samp = x[np.sort(g.choice(2000, 384, replace=False))]
    init = samp[g.choice(384, 6, replace=False)]
    cent, _ = O.kmodes_np(samp, init, 7)
    assert np.array_equal(a.centroids, cent)
    assign = np.argmin(O.hamming_np(x, cent), axis=1)
    ref = O.index_from_assignment(x, cent, assign)
    assert np.array_equal(a.part_offsets, ref.part_offsets) and np.array_equal(a.row_ids, ref.row_ids)
    assert np.array_equal(a.vectors, x[a.row_ids.astype(np.int64)])
    with pytest.raises(ValueError, match="hamming"):
        train_ivf_binary(x, num_partitions=2, distance_type="l2")
    with pytest.raises(ValueError, match="num_partitions"):
        train_ivf_binary(x[:3], num_partitions=4)


def _known_answer_data():
    """the reference's test_create_index_with_binary_vectors: rows [i] * 128 for i < 256, IvfFlat(hamming, 10)"""
    return np.repeat(np.arange(256, dtype=np.uint8)[:, None], 128, axis=1)


def test_known_answer_on_oracle():
    x = _known_answer_data()
    data = train_ivf_binary(x, num_partitions=10)
    q = x.copy()                                           # nearest_to([v] * 128) for every v
    ids, dist, cnt = O.search(data, q, k=1, nprobes=20)
    assert ids[:, 0].tolist() == list(range(256)) and np.all(dist[:, 0] == 0)


class _StubIvfBinary:
    """Stands in for _native.GpuIvfBinary: records the index it was opened with and answers from the C oracle."""
    opened = []

    def __init__(self, data, device=0):
        self.data, self.metric = data, data.metric
        _StubIvfBinary.opened.append(data)

    def search(self, queries, k=10, nprobes=20, refine_factor=0, lower=None, upper=None, allow=None, allow_bits=0,
               max_nprobes=0, timeout_ms=0):
        mask = None
        if allow is not None:
            mask = np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")[:allow_bits].astype(bool)
        return O.search(self.data, queries, k=k, nprobes=nprobes, lower=lower, upper=upper, allow=mask,
                        max_nprobes=max_nprobes)

    def close(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    _StubIvfBinary.opened = []
    monkeypatch.setattr(_native, "GpuIvfBinary", _StubIvfBinary)
    return _StubIvfBinary


def _binary_table(db, name, x):
    schema = pa.schema([pa.field("bits", pa.list_(pa.uint8(), x.shape[1])), pa.field("id", pa.int64())])
    return db.create_table(name, pa.table({"bits": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), x.shape[1]),
                                           "id": np.arange(x.shape[0])}, schema=schema))


def test_create_index_ivf_flat_builds_lists_and_searches(stub):
    db = lancedb.connect("memory://")
    t = _binary_table(db, "t", _known_answer_data())
    t.create_index(metric="hamming", num_partitions=10, index_type="IVF_FLAT")
    assert len(stub.opened) == 1 and isinstance(stub.opened[0], IvfBinaryIndexData) and stub.opened[0].nlist == 10
    assert t.list_indices() == [{"name": "bits_idx", "index_type": "IVF_FLAT", "columns": ["bits"]}]
    st = t.index_stats("bits_idx")
    assert st["index_type"] == "IVF_FLAT" and st["distance_type"] == "hamming" and st["num_indexed_rows"] == 256
    for v in (0, 1, 77, 255):
        out = t.search(np.full(128, v), vector_column_name="bits").distance_type("hamming").limit(1).to_arrow()
        assert out["id"].to_pylist() == [v] and out["_distance"].to_pylist() == [0.0]
    with pytest.raises(NotImplementedError, match="IVF_PQ"):
        t.save_lance_index("/nonexistent")


def test_create_index_ivf_flat_rejections(stub):
    rng = np.random.default_rng(8)
    db = lancedb.connect("memory://")
    tf = db.create_table("f", {"vector": rng.standard_normal((300, 8)).astype(np.float32)})
    with pytest.raises(NotImplementedError):
        tf.create_index(index_type="IVF_FLAT")
    with pytest.raises(NotImplementedError):
        tf.create_index(index_type="IVF_FLAT", metric="hamming")
    tb = _binary_table(db, "b", rng.integers(0, 256, (300, 4), dtype=np.uint8))
    with pytest.raises(ValueError, match="hamming"):
        tb.create_index(index_type="IVF_FLAT")                 # the builder's default l2 is refused, not rebuilt
    with pytest.raises(ValueError, match="hamming"):
        tb.create_index(index_type="IVF_FLAT", metric="cosine")
    for kind in ("IVF_PQ", "IVF_SQ", "IVF_RQ"):
        with pytest.raises(NotImplementedError, match="binary"):
            tb.create_index(index_type=kind, num_bits=1 if kind == "IVF_RQ" else 8)
    mv = pa.array([[[1.0, 2.0], [3.0, 4.0]], [[5.0, 6.0]]], pa.list_(pa.list_(pa.float32(), 2)))
    tm = db.create_table("m", pa.table({"mv": mv}))
    with pytest.raises(NotImplementedError, match="multivector"):
        tm.create_index(index_type="IVF_FLAT", metric="hamming")
    with pytest.raises(ValueError, match="2\\^24"):
        train_ivf_binary(np.zeros((4, (1 << 21) + 1), np.uint8), num_partitions=1)
    assert stub.opened == []
    tb.create_index(index_type="IVF_FLAT", metric="hamming", num_partitions=3)
    with pytest.raises(RuntimeError, match="already exists"):
        tb.create_index(index_type="IVF_FLAT", metric="hamming", num_partitions=3, replace=False)


def test_search_uses_index_until_bypassed(stub, monkeypatch):
    rng = np.random.default_rng(9)
    x = rng.integers(0, 256, (500, 8), dtype=np.uint8)
    db = lancedb.connect("memory://")
    t = _binary_table(db, "t", x)
    t.create_index(metric="hamming", num_partitions=5, index_type="IVF_FLAT")
    q = x[17]
    got = t.search(q).distance_type("hamming").nprobes(1).limit(5).to_arrow()
    ref = O.search(stub.opened[0], q[None], k=5, nprobes=1)
    assert got["_rowid" if "_rowid" in got.column_names else "id"].to_pylist()[:5] == ref[0][0].astype(int).tolist()

    calls = []

    class _Flat:
        def __init__(self, vectors, device=0):
            pass

        def search(self, q, **kw):
            calls.append(kw)
            return flat_search_u8_np(x, q, kw["k"])

    monkeypatch.setattr(_native, "GpuBinary", _Flat)
    t.search(q).distance_type("hamming").bypass_vector_index().limit(5).to_arrow()
    assert len(calls) == 1


def test_async_create_index_with_ivf_flat_config(stub):
    x = _known_answer_data()

    async def run():
        db = await lancedb.connect_async("memory://")
        schema = pa.schema([pa.field("bits", pa.list_(pa.uint8(), 128))])
        t = await db.create_table("t", pa.table({"bits": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), 128)},
                                                schema=schema))
        assert lancedb.IvfFlat().distance_type == "l2"
        with pytest.raises(ValueError, match="hamming"):
            await t.create_index("bits", config=lancedb.IvfFlat(), accelerator=None)
        await t.create_index("bits", config=lancedb.IvfFlat(distance_type="hamming", num_partitions=10, max_iterations=3),
                             accelerator=None)
        return await t.list_indices()

    assert asyncio.run(run())[0]["index_type"] == "IVF_FLAT"
    assert len(stub.opened) == 1 and stub.opened[0].nlist == 10

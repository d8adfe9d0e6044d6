"""Binary vectors (fixed_size_list<uint8>, Hamming distance) without a GPU: the oracle, the reference's pins, the
Python surface's typing and validation."""
import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200
from lancedb_b200 import _native
from tests.hamming_oracle import (flat_search_u8, flat_search_u8_np, hamming_u8, hamming_u8_np,
                                  hamming_unpackbits)


def _pairwise_slow(q, x):
    return np.array([[hamming_unpackbits(a, b) for b in x] for a in q], np.uint32)


def _data(nbytes, seed):
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 256, (5, nbytes), dtype=np.uint8)
    x = rng.integers(0, 256, (37, nbytes), dtype=np.uint8)
    x[3] = x[4] = x[5]                                   # duplicates
    x[6] = 0
    x[7] = 255
    q[0] = 0
    q[1] = 255
    return rng, q, x


@pytest.mark.parametrize("nbytes", [1, 3, 8, 33, 160])
def test_c_oracle_matches_the_numpy_mirror(nbytes):
    rng, q, x = _data(nbytes, nbytes)
    slow = _pairwise_slow(q, x)
    assert np.array_equal(hamming_u8(q, x), slow)
    assert np.array_equal(hamming_u8(q, x, nthreads=3), slow)
    assert np.array_equal(hamming_u8_np(q, x, nthreads=4), slow)
    assert hamming_u8(q[:1], x[6:8]).tolist() == [[0, 8 * nbytes]]
    assert hamming_u8(np.zeros((1, nbytes), np.uint8), np.full((1, nbytes), 255, np.uint8)).tolist() == [[8 * nbytes]]
    rid = rng.permutation(37).astype(np.uint64) * 5 + 2
    mask = rng.random(200) < 0.6
    for kw in (dict(k=5), dict(k=50), dict(k=7, row_ids=rid), dict(k=7, row_ids=rid, allow=mask),
               dict(k=9, lower=2 * nbytes, upper=6 * nbytes), dict(k=3, allow=np.zeros(4, bool))):
        got = flat_search_u8(x, q, nthreads=2, **kw)
        want = flat_search_u8_np(x, q, **kw)
        for g, w in zip(got, want):
            assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), kw
    ties = np.tile(x[:1], (37, 1))                      # all rows equal: the top-k is by row id alone
    for g, w in zip(flat_search_u8(ties, q, k=10, row_ids=rid), flat_search_u8_np(ties, q, k=10, row_ids=rid)):
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8))


def test_oracle_order_range_allow_and_short_results():
    x = np.array([[1], [0], [3], [0], [255]], np.uint8)
    ids, dist, cnt = flat_search_u8(x, np.zeros((1, 1), np.uint8), k=4, row_ids=[9, 7, 5, 3, 1])
    # (distance, id): ids 3 and 7 tie at 0 and come back by id
    assert ids[0].tolist() == [3, 7, 9, 5] and dist[0].tolist() == [0, 0, 1, 2] and cnt[0] == 4
    ids, dist, cnt = flat_search_u8(x, np.zeros((1, 1), np.uint8), k=10, lower=1, upper=8)
    assert ids[0, :2].tolist() == [0, 2] and cnt[0] == 2
    assert ids[0, 2] == np.iinfo(np.uint64).max and np.isinf(dist[0, 2])
    allow = np.zeros(4, bool)
    allow[[1, 2]] = True                                  # id 4 lies beyond the mask: excluded
    ids, dist, cnt = flat_search_u8(x, np.zeros((1, 1), np.uint8), k=10, allow=allow)
    assert ids[0, :cnt[0]].tolist() == [1, 2]


def test_reference_pin_i_times_128_table():
    """python/python/tests/test_index.py:67-84, 509-512: rows [i]*128 (i < 256), nearest_to([v]*128) -> id v."""
    x = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 128, axis=1)
    for v in (0, 1, 77, 128, 255):
        ids, dist, _ = flat_search_u8(x, np.full((1, 128), v, np.uint8), k=3)
        assert ids[0, 0] == v and dist[0, 0] == 0
        assert dist[0, 1] == 128                          # one bit flipped in each of the 128 bytes


def _docs_table(db, n=64):
    """The reference docs example (python/python/tests/docs/test_binary_vector.py:16-46)."""
    schema = pa.schema([pa.field("id", pa.int64()), pa.field("vector", pa.list_(pa.uint8(), 32))])
    rng = np.random.default_rng(0)
    data = [{"id": i, "vector": np.packbits(rng.integers(0, 2, 256))} for i in range(n)]
    return db.create_table("bin", data, schema=schema), data


def test_create_table_builds_data_against_the_schema():
    db = lancedb_b200.connect()
    tbl, data = _docs_table(db)
    assert tbl.schema.field("vector").type == pa.list_(pa.uint8(), 32)
    assert tbl.schema.field("id").type == pa.int64()
    got = np.asarray(tbl.to_arrow().column("vector").combine_chunks().flatten().to_numpy(), np.uint8).reshape(-1, 32)
    assert np.array_equal(got, np.stack([d["vector"] for d in data]))
    # without a schema, lists of numbers stay float vectors (unchanged behaviour)
    t2 = db.create_table("f", [{"vector": [1.0, 2.0]}])
    assert t2.schema.field("vector").type == pa.list_(pa.float32(), 2)
    # the schema alone: an empty binary table
    t3 = db.create_table("e", schema=pa.schema([pa.field("vector", pa.list_(pa.uint8(), 4))]))
    assert t3.count_rows() == 0 and t3.search([1, 2, 3, 4]).distance_type("hamming").to_arrow().num_rows == 0


def test_binary_columns_are_vector_columns():
    db = lancedb_b200.connect()
    tbl, _ = _docs_table(db)
    q = tbl.search(np.packbits(np.ones(256, np.uint8)))
    assert q._vector_column == "vector" and q._query.shape == (1, 32)


@pytest.mark.parametrize("bad", [[-1] + [0] * 31, [256] + [0] * 31, [1.5] + [0] * 31, [float("nan")] + [0] * 31,
                                 ["a"] * 32])
def test_bad_query_components_raise_value_error(bad):
    db = lancedb_b200.connect()
    tbl, _ = _docs_table(db)
    with pytest.raises(ValueError):
        tbl.search(bad, vector_column_name="vector").to_arrow()


def test_wrong_query_length_and_metric_pairings_raise_value_error():
    db = lancedb_b200.connect()
    tbl, _ = _docs_table(db)
    with pytest.raises(ValueError):
        tbl.search(np.zeros(31, np.uint8), vector_column_name="vector").to_arrow()
    for metric in ("l2", "cosine", "dot"):
        with pytest.raises(ValueError):
            tbl.search(np.zeros(32, np.uint8)).distance_type(metric).to_arrow()
    ft = db.create_table("floats", {"vector": np.ones((8, 4), np.float32)})
    with pytest.raises(ValueError):
        ft.search(np.ones(4, np.float32)).distance_type("hamming").to_arrow()


def test_no_binary_index():
    db = lancedb_b200.connect()
    tbl, _ = _docs_table(db)
    with pytest.raises(NotImplementedError):
        tbl.create_index(vector_column_name="vector")


def test_gpu_binary_has_no_cpu_fallback():
    try:
        if _native.device_count() > 0:
            pytest.skip("a CUDA device is present")
    except ImportError:
        pytest.skip("library not built")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _native.GpuBinary(np.zeros((4, 32), np.uint8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _native.debug_hamming_gemm(np.zeros((1, 4), np.uint8), np.zeros((2, 4), np.uint8))
    db = lancedb_b200.connect()
    tbl, _ = _docs_table(db)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tbl.search(np.zeros(32, np.uint8)).distance_type("hamming").to_arrow()


def test_gpu_binary_validates_query_shape_and_components_before_the_device():
    bx = _native.GpuBinary.__new__(_native.GpuBinary)    # the checks need no device
    bx.nbytes = 4
    assert bx._queries([1, 2, 3, 4]).shape == (1, 4)
    assert bx._queries(np.zeros((3, 4), np.float32)).dtype == np.uint8
    for bad in (np.zeros(8, np.uint8), np.zeros((2, 3), np.uint8), np.zeros((1, 1, 4), np.uint8), [256, 0, 0, 0],
                [-1, 0, 0, 0], [0.5, 0, 0, 0], ["a"] * 4):
        with pytest.raises(ValueError):
            bx._queries(bad)

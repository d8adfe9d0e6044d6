"""4-bit IVF_PQ without a GPU: the C oracle against its NumPy mirror (the quantiser's rounding and saturation, the folds,
degenerate and NaN tables, m = 2, the nibble order, whole searches), the default num_sub_vectors of create_index.rs, the
trainer, and the Python surface of create_index(num_bits=4) against a stubbed native layer."""
import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from oracle import oracle_np as onp
from lancedb_b200.index import (IvfPqIndexData, get_num_sub_vectors, pack_pq4, suggested_num_sub_vectors,
                                train_ivf_pq, unpack_pq4)
from tests import pq4_oracle
from tests.pq4_oracle import random_pq4_index

f32 = np.float32


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, f32).view(np.uint32), np.asarray(b, f32).view(np.uint32))


def test_quantiser_rounds_half_away_from_zero_and_saturates():
    # qmax - qmin = 510: the scaled value is t / 2 exactly, so odd t land on .5
    t = np.arange(-8, 530, dtype=f32)
    c = pq4_oracle.quant(t, 0.0, 510.0)
    assert np.array_equal(c, pq4_oracle.quant_np(t, 0.0, 510.0))
    want = np.clip(np.floor(t.astype(np.float64) / 2 + 0.5), 0, 255).astype(np.uint8)
    assert np.array_equal(c, want)
    assert c[t == 5].tolist() == [3] and c[t == 1].tolist() == [1]      # 2.5 -> 3, 0.5 -> 1 (not to even)
    # one f32 ulp either side of each .5, NaN, +-inf, a degenerate range (0 / 0 -> 0)
    b = (np.arange(256, dtype=f32) + f32(0.5)) * f32(2)
    v = np.concatenate([b, np.nextafter(b, f32(-np.inf)), np.nextafter(b, f32(np.inf)),
                        np.array([np.nan, np.inf, -np.inf, -0.0, 1e30, -1e30], f32)])
    for lo, hi in ((0.0, 510.0), (-3.0, 7.0), (1.5, 1.5), (2.0, -1.0), (np.inf, -np.inf)):
        assert np.array_equal(pq4_oracle.quant(v, lo, hi), pq4_oracle.quant_np(v, lo, hi)), (lo, hi)
    # qmax == qmin: an entry equal to both is 0 / 0 -> 0; others are +-inf -> 255 / 0
    deg = np.array([1.5, 1.75, 1.25], f32)
    assert pq4_oracle.quant(deg, 1.5, 1.5).tolist() == [0, 255, 0] == pq4_oracle.quant_np(deg, 1.5, 1.5).tolist()


def test_distance_c_and_numpy_agree():
    S = np.concatenate([np.arange(0, 65281, 97), [0, 1, 65280]]).astype(np.uint32)
    for qmin, qmax in ((0.0, 1.0), (-3.25, 11.0), (2.0, 2.0), (1e-30, 1e30), (np.inf, -np.inf)):
        for m in (2, 48, 256):
            for metric in ("l2", "cosine", "dot"):
                assert _bits_equal(pq4_oracle.distance(S, qmin, qmax, m, metric),
                                   pq4_oracle.distance_np(S, qmin, qmax, m, metric))
    # the formula in Python floats rounded to f32 after every step
    s, lo, hi, m = 12345, f32(-0.7), f32(3.9), 48
    d = f32(f32(f32(f32(s) * f32(hi - lo)) / f32(255)) + f32(lo * f32(m)))
    assert pq4_oracle.distance([s], lo, hi, m, "l2")[0] == d
    assert pq4_oracle.distance([s], lo, hi, m, "dot")[0] == f32(d - f32(m - 1))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("m,dim", [(2, 2), (2, 64), (8, 32), (12, 48), (16, 256), (4, 128)])
def test_tables_c_and_numpy_agree(metric, m, dim):
    rng = np.random.default_rng(m * 31 + dim)
    ix = random_pq4_index(rng, n=200, dim=dim, nlist=3, m=m, metric=metric, empty=())
    for p in range(3):
        qn = rng.standard_normal(dim).astype(f32)
        Q, lo, hi = pq4_oracle.tables(ix, qn, p)
        Qn, lon, hin = pq4_oracle.tables_np(ix, qn, p)
        assert np.array_equal(Q, Qn) and _bits_equal(lo, lon) and _bits_equal(hi, hin)
        # partition_distances takes the raw query and normalises it for cosine itself
        qm = onp.normalize(qn) if metric == "cosine" else qn
        assert _bits_equal(pq4_oracle.partition_distances(ix, qn, p), pq4_oracle.partition_distances_np(ix, qm, p))


def test_qmax_is_the_largest_adjacent_pair_of_row_maxima():
    T = np.full((4, 16), 1.0, f32)
    T[0, 3], T[1, 9], T[2, 0], T[3, 15] = 10.0, 1.0, 7.0, 2.0
    T[1, 2] = np.nan
    lo, hi = pq4_oracle.fold_np(T)
    assert lo == 1.0 and hi == f32(11.0)                # row maxima 10, 1, 7, 2: windows 11, 8, 9


def test_dot_tables_with_negative_row_maxima_saturate_at_255():
    # every T = 1 - x.c lies in [-10, -1], so qmax (a sum of two negative row maxima) lies below the entries near -1
    rng = np.random.default_rng(3)
    ix = random_pq4_index(rng, n=100, dim=16, nlist=2, m=4, metric="dot", empty=())
    ix.codebook[:] = rng.uniform(0.5, 2.75, ix.codebook.shape).astype(f32)
    qn = np.ones(16, f32)
    Q, lo, hi = pq4_oracle.tables(ix, qn, 0)
    Qn, lon, hin = pq4_oracle.tables_np(ix, qn, 0)
    assert np.array_equal(Q, Qn) and lo == lon and hi == hin
    assert hi < 0 and (Q == 255).sum() > 16


def test_all_equal_tables_give_zero_codes_and_zero_distance():
    rng = np.random.default_rng(4)
    ix = random_pq4_index(rng, n=50, dim=16, nlist=1, m=4, metric="l2", empty=())
    ix.codebook[:] = 0.0
    qn = ix.centroids[0].copy()                           # residual 0: every T is +0, qmax == qmin == 0
    Q, lo, hi = pq4_oracle.tables(ix, qn, 0)
    assert not Q.any() and lo == 0.0 and hi == 0.0
    assert np.array_equal(Q, pq4_oracle.tables_np(ix, qn, 0)[0])
    d = pq4_oracle.partition_distances(ix, qn, 0)
    assert _bits_equal(d, pq4_oracle.partition_distances_np(ix, qn, 0)) and not d.any()


def test_nan_query_components():
    rng = np.random.default_rng(5)
    ix = random_pq4_index(rng, n=300, dim=32, nlist=4, m=8, metric="l2", empty=())
    qn = rng.standard_normal(32).astype(f32)
    qn[3] = np.nan                                        # one sub-space of NaN entries: skipped by both folds
    Q, lo, hi = pq4_oracle.tables(ix, qn, 1)
    Qn, lon, hin = pq4_oracle.tables_np(ix, qn, 1)
    assert np.array_equal(Q, Qn) and lo == lon and hi == hin and np.isfinite(lo) and np.isfinite(hi)
    assert not Q[0].any()                                 # NaN entries quantise to 0
    qn[:] = np.nan                                        # every entry NaN: +inf / -inf, every distance NaN
    Q, lo, hi = pq4_oracle.tables(ix, qn, 1)
    assert not Q.any() and lo == np.inf and hi == -np.inf
    assert np.isnan(pq4_oracle.partition_distances(ix, qn, 1)).all()
    q = rng.standard_normal((3, 32)).astype(f32)
    q[1, 0] = np.nan
    got = pq4_oracle.search(ix, q, k=5, nprobes=4)
    assert got[2][1] == 0 and np.array_equal(got[0], pq4_oracle.pq4_search_np(ix, q, k=5, nprobes=4)[0])


def test_nibble_order_and_code_layouts():
    c = np.array([[1, 2, 3, 4], [15, 0, 0, 15]], np.uint8)
    p = pack_pq4(c)
    assert p.tolist() == [[0x21, 0x43], [0x0F, 0xF0]]      # byte j: code 2j in bits 0-3, code 2j+1 in bits 4-7
    assert np.array_equal(unpack_pq4(p), c)
    with pytest.raises(ValueError):
        pack_pq4(np.array([[16, 0]], np.uint8))
    with pytest.raises(ValueError):
        pack_pq4(np.zeros((1, 3), np.uint8))
    # the oracle reads sub-vector 2j from the low nibble: swapping the nibbles changes the sums
    rng = np.random.default_rng(6)
    ix = random_pq4_index(rng, n=400, dim=32, nlist=2, m=8, metric="l2", empty=())
    qn = rng.standard_normal(32).astype(f32)
    Q, lo, hi = pq4_oracle.tables(ix, qn, 0)
    n0 = int(ix.part_offsets[1])
    rm = pq4_oracle.row_major_codes(ix)                   # [n][m/2] row-major == the transposed codes, per partition
    assert np.array_equal(rm[:n0].T.reshape(-1), ix.codes_t[:n0 * 4])
    codes = unpack_pq4(rm[:n0]).astype(np.int64)
    S = Q.astype(np.int64)[np.arange(8)[None, :], codes].sum(1)
    assert _bits_equal(pq4_oracle.partition_distances(ix, qn, 0), pq4_oracle.distance_np(S, lo, hi, 8, "l2"))
    swapped = unpack_pq4(((rm[:n0] >> 4) | (rm[:n0] << 4)).astype(np.uint8)).astype(np.int64)
    assert not np.array_equal(Q.astype(np.int64)[np.arange(8)[None, :], swapped].sum(1), S)


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_search_c_oracle_equals_numpy_mirror(metric):
    rng = np.random.default_rng({"l2": 7, "cosine": 8, "dot": 9}[metric])
    ix = random_pq4_index(rng, n=500, dim=16, nlist=6, m=4, metric=metric, empty=(1, 4))
    q = rng.standard_normal((6, 16)).astype(f32)
    q[2] = ix.vectors[5]
    mask = rng.random(int(ix.row_ids.max()) + 1) < 0.05
    d0 = pq4_oracle.search(ix, q[:1], k=40, nprobes=3)[1][0]
    cases = [dict(k=10, nprobes=2), dict(k=1, nprobes=6), dict(k=700, nprobes=6),           # k > N
             dict(k=10, nprobes=1, allow=mask, max_nprobes=6), dict(k=10, nprobes=2, allow=mask),
             dict(k=15, nprobes=3, lower=float(d0[3]), upper=float(d0[30])),
             dict(k=5, nprobes=3, refine_factor=4)]
    for kw in cases:
        a = pq4_oracle.search(ix, q, **kw)
        b = pq4_oracle.pq4_search_np(ix, q, **kw)
        assert np.array_equal(a[2], b[2]) and np.array_equal(a[0], b[0]) and _bits_equal(a[1], b[1]), kw
    # duplicates (rows 5..8 share row 4's codes) tie and come back by row id
    ids, dist, _ = pq4_oracle.search(ix, q, k=700, nprobes=6)
    for i in range(q.shape[0]):
        d = dist[i][np.isfinite(dist[i])]
        assert np.all(np.diff(d) >= 0)
        same = np.nonzero(d[1:] == d[:-1])[0]
        assert len(same) > 0 and np.all(ids[i][same] < ids[i][same + 1])


def test_default_num_sub_vectors_follows_create_index_rs():
    # get_num_sub_vectors (create_index.rs:86-102): the explicit value, else the suggestion, made even for 4 bits
    for dim in (768, 1536, 128, 24, 40, 8, 7, 1):
        s = suggested_num_sub_vectors(dim)
        assert get_num_sub_vectors(None, dim, 8) == s
        assert get_num_sub_vectors(None, dim, None) == s
        assert get_num_sub_vectors(None, dim, 4) == (s + 1 if s % 2 else s)
        assert get_num_sub_vectors(3, dim, 4) == 3
    assert get_num_sub_vectors(None, 768, 4) == 48 and get_num_sub_vectors(None, 24, 4) == 4


def test_trainer_num_bits_4_codes_and_rejections():
    rng = np.random.default_rng(10)
    x = rng.standard_normal((900, 24)).astype(f32)
    data = train_ivf_pq(x, num_partitions=4, num_bits=4, max_iterations=2, sample_rate=32, keep_vectors=True)
    data.validate()
    assert data.num_bits == 4 and data.m == 4 and data.codebook.shape == (4, 16, 6)
    assert data.code_bytes == 2 and data.codes_t.size == 900 * 2 and sorted(data.row_ids.tolist()) == list(range(900))
    # each code is the argmin of |c|^2 - 2 r.c over the 16 codewords (ties to the lowest)
    import torch
    xs = torch.as_tensor(data.vectors)
    part = np.repeat(np.arange(4), np.diff(data.part_offsets.astype(np.int64)))
    r = (xs - torch.as_tensor(data.centroids)[part]).reshape(-1, 4, 6).transpose(0, 1)
    cb = torch.as_tensor(data.codebook)
    want = ((cb * cb).sum(2)[:, None, :] - 2.0 * torch.bmm(r, cb.transpose(1, 2))).argmin(2).T.numpy()
    assert np.array_equal(unpack_pq4(pq4_oracle.row_major_codes(data)), want.astype(np.uint8))
    with pytest.raises(ValueError, match="even"):
        train_ivf_pq(x, num_partitions=4, num_bits=4, num_sub_vectors=3)
    for nb in (1, 2, 16):
        with pytest.raises(ValueError, match="num_bits"):
            train_ivf_pq(x, num_partitions=4, num_bits=nb)
    # the 8-bit trainer is unchanged by the new argument
    a = train_ivf_pq(x, num_partitions=4, max_iterations=2, sample_rate=32)
    b = train_ivf_pq(x, num_partitions=4, max_iterations=2, sample_rate=32, num_bits=8)
    assert a.num_bits == 8 and np.array_equal(a.codes_t, b.codes_t) and np.array_equal(a.codebook, b.codebook)


def test_shard_and_partition_codes_use_the_row_byte_width():
    rng = np.random.default_rng(11)
    ix = random_pq4_index(rng, n=300, dim=16, nlist=5, m=4, empty=(2,))
    for p in range(5):
        n = int(ix.part_offsets[p + 1] - ix.part_offsets[p])
        assert ix.partition_codes(p).shape == (2, n)
    parts = [ix.shard(r, 2) for r in range(2)]
    for s in parts:
        s.validate()
        assert s.num_bits == 4
    assert sum(s.nrows for s in parts) == 300


class _StubPq:
    """Stands in for _native.GpuIvfPq: records the arrays it was opened with."""
    opened = []

    def __init__(self, data, device=0):
        self.data, self.metric = data, data.metric
        _StubPq.opened.append(data)

    def close(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    _StubPq.opened = []
    monkeypatch.setattr(_native, "GpuIvfPq", _StubPq)
    return _StubPq


def test_create_index_num_bits_4_builds_and_rejections(stub):
    rng = np.random.default_rng(12)
    db = lancedb.connect("memory://")
    t = db.create_table("t", {"vector": rng.standard_normal((400, 24)).astype(f32), "id": np.arange(400)})
    t.create_index(metric="l2", num_partitions=4, num_bits=4, max_iterations=2)
    assert len(stub.opened) == 1 and isinstance(stub.opened[0], IvfPqIndexData)
    assert stub.opened[0].num_bits == 4 and stub.opened[0].m == 4 and stub.opened[0].vectors is not None
    assert t.list_indices() == [{"name": "vector_idx", "index_type": "IVF_PQ", "columns": ["vector"]}]
    with pytest.raises(NotImplementedError, match="8-bit"):
        t.save_lance_index("/nonexistent")
    for nb in (1, 2, 16):
        with pytest.raises(ValueError, match="num_bits"):
            t.create_index(num_bits=nb)
    with pytest.raises(ValueError, match="even"):
        t.create_index(num_bits=4, num_sub_vectors=3, num_partitions=4)
    assert len(stub.opened) == 1

"""Float16 multivector columns without a GPU: which row type reaches GpuMultivec (float16 columns as float16, f32 and f64
columns as f32, through Table, the async surface and remote.handle_query), which native opener a float16 array selects,
the shape checks that come before the device, and a CPU restatement of the fp16 handle's tensor-core band
(multivec.cu mv_band_f16, gemm.cu F16RowMaxSim) on adversarial inputs: query components one f32 ulp beside fp16
rounding midpoints, and stored fp16 vectors across the whole fp16 range (subnormals, +-65504, mixed magnitudes).  The
band holds on all of them, and a band without the query's rounding term does not."""
import asyncio

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200
from lancedb_b200 import _native, remote
from lancedb_b200.aio import AsyncTable
from tests.multivec_oracle import distances, flat_search_mv, lance_dot_np, offsets_of
from tests.test_multivec_host import _unit_at_midpoints

F16, F32 = np.float16, np.float32
U = 2.0 ** -24


# ---- which rows reach the native handle ----
_GpuMultivec = _native.GpuMultivec


class _RecordingMultivec:
    """Stands in for GpuMultivec: records the dtype of the values it is opened with and answers with the C oracle on
    their f32 upcast."""
    seen = []

    def __init__(self, values, offsets, row_ids=None, device=0):
        _RecordingMultivec.seen.append(np.asarray(values).dtype)
        self.values, self.offsets = np.asarray(values).astype(F32), np.asarray(offsets, np.uint64)
        self.dim = self.values.shape[1]

    def search(self, queries, k=10, q_offsets=None, lower=None, upper=None, allow=None, allow_bits=0, timeout_ms=0):
        q, qo = _GpuMultivec._queries(self, queries, q_offsets)
        mask = None
        if allow is not None:
            mask = np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")[:allow_bits].astype(bool)
        return flat_search_mv(self.values, self.offsets, q, qo, k, lower=lower, upper=upper, allow=mask)

    def close(self):
        pass


@pytest.fixture
def mv_stub(monkeypatch):
    _RecordingMultivec.seen = []
    monkeypatch.setattr(_native, "GpuMultivec", _RecordingMultivec)
    return _RecordingMultivec.seen


def _table(db, value_type, name):
    """The reference's 256 rows of [[i, i+1], [i+2, i+3]], plus a null and an empty row."""
    data = [[[i, i + 1], [i + 2, i + 3]] for i in range(256)] + [None, []]
    return db.create_table(name, pa.table({"vector": pa.array(data, type=pa.list_(pa.list_(value_type, 2))),
                                           "id": pa.array(list(range(1, 259)))}))


@pytest.mark.parametrize("value_type,want", [(pa.float16(), F16), (pa.float32(), F32), (pa.float64(), F32)])
def test_every_surface_opens_the_handle_on_the_columns_row_type(mv_stub, value_type, want):
    db = lancedb_b200.connect()
    tbl = _table(db, value_type, "t")
    vals, off = tbl._multivec_rows("vector")
    assert vals.dtype == want and vals.shape == (512, 2) and list(off[-3:]) == [512, 512, 512]
    got = tbl.search([[1, 2], [5, 1]]).limit(7).with_row_id(True).to_arrow()
    x = np.array([[[i, i + 1], [i + 2, i + 3]] for i in range(256)], want).reshape(-1, 2).astype(F32)
    ids, dist, cnt = flat_search_mv(x, offsets_of([2] * 256 + [0, 0]), np.array([[1, 2], [5, 1]], F32), [0, 2], 7)
    assert got["_rowid"].to_pylist() == [int(i) for i in ids[0][:cnt[0]]]
    assert np.array_equal(np.array(got["_distance"].to_pylist(), F32).view(np.uint32), dist[0][:cnt[0]].view(np.uint32))

    async def run():
        return await AsyncTable(tbl).query().nearest_to([[1, 2], [5, 1]]).limit(7).to_arrow()

    want_tbl = tbl.search([[1, 2], [5, 1]]).limit(7).to_arrow()
    assert asyncio.run(run()).equals(want_tbl)
    out = remote.read_ipc_file(remote.handle_query(tbl, remote.build_query_body([[1, 2], [5, 1]], k=7)))
    assert out.equals(want_tbl)
    assert mv_stub == [np.dtype(want)]              # one handle, cached for every surface
    # a second table on the same connection opens its own handle, with its own row type
    _table(db, value_type, "u").search([[1, 2]]).to_arrow()
    assert mv_stub == [np.dtype(want)] * 2


class _FakeLib:
    """Records which opener GpuMultivec calls; every call succeeds."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 0
        return fn


@pytest.mark.parametrize("dtype,opener", [(F16, "lgpu_multivec_open_f16"), (F32, "lgpu_multivec_open"),
                                          (np.float64, "lgpu_multivec_open"), (np.int32, "lgpu_multivec_open")])
def test_a_float16_array_opens_an_fp16_handle_and_anything_else_an_f32_one(monkeypatch, dtype, opener):
    lib = _FakeLib()
    monkeypatch.setattr(_native, "load", lambda: lib)
    mv = _native.GpuMultivec(np.ones((5, 8), dtype), [0, 2, 2, 5])
    assert lib.calls == [opener]
    assert mv.dtype == (np.dtype(F16) if dtype == F16 else np.dtype(F32))
    mv._h = None                                     # nothing to close: the fake opener made no handle


def test_gpu_multivec_checks_float16_shapes_before_the_device(monkeypatch):
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native layer was called"))
    for vals, off in ((np.zeros((3, 4), F16), [0, 2]), (np.zeros((3, 4), F16), [0, 2, 1, 3]),
                      (np.zeros((3, 4), F16), [1, 3]), (np.zeros(3, F16), [0, 3]),
                      (np.zeros((2, 0), F16), [0, 2])):
        with pytest.raises(ValueError):
            _native.GpuMultivec(vals, off)
    with pytest.raises(ValueError):
        _native.GpuMultivec(np.zeros((3, 4), F16), [0, 3], row_ids=[1, 2])
    with pytest.raises(ValueError):
        _native.debug_maxsim_gemm(np.zeros((2, 8), F32), np.zeros((3, 4), F16), [0, 3])


# ---- the fp16 handle's tensor-core band (multivec.cu mv_band_f16) under adversarial inputs ----
def mv_band_f16(nq, d, query_term=True):
    """multivec.cu mv_band_f16 restated in f32 (query_term False: the same band without the query's fp16 rounding)."""
    e = (F32(1.01) * F32(2.0 ** -11) if query_term else F32(0)) + (F32(8) * F32(d) + np.sqrt(F32(d)) + F32(42)) * F32(U)
    return F32((F32(nq) * e + F32(4.04) * F32(nq) * F32(nq) * F32(U)) * F32(1 + 2.0 ** -8))


def _norms(v):
    """|v| as lance's f32 dot (row_norms_kernel, mv_normalize_f16_kernel)."""
    return np.array([np.sqrt(lance_dot_np(r, r[None, :])[0]) for r in v], F32)


def _approx_maxsim_f16(q, x16, off, qoff):
    """The F16RowMaxSim approximate distances restated: fp16(q / |q|) . x summed in f64 and rounded to f32 (wgmma's
    accumulation error is a term of the band of its own), scaled by 1/|x| in f32 as the epilogue does (the f32
    reciprocal of |x|, then an f32 product), max over each row's run, sum of (1 - max) over the query's vectors in f32."""
    a = (q / _norms(q)[:, None]).astype(F32).astype(F16).astype(np.float64)
    x32 = x16.astype(F32)
    S = (a @ x32.astype(np.float64).T).astype(F32) * (F32(1) / _norms(x32))[None, :]
    B, N = len(qoff) - 1, len(off) - 1
    A = np.full((B, N), np.nan, F32)
    for r in range(N):
        if off[r + 1] == off[r]:
            continue
        m = S[:, int(off[r]):int(off[r + 1])].max(axis=1)
        for b in range(B):
            s = F32(0)
            for i in range(int(qoff[b]), int(qoff[b + 1])):
                s = F32(s + (F32(1) - m[i]))
            A[b, r] = s
    return A


def adversarial_f16_column(rng, q):
    """Stored fp16 vectors across the fp16 range: copies of the query vectors at magnitudes from subnormal to 65504
    (similarity ~1, where the query's rounding errors add up), vectors holding +-65504 beside subnormal components, and
    random vectors of mixed magnitudes (1e-7 .. 6e4), one to three per row."""
    d = q.shape[1]
    rows = []
    for scale in (2.0 ** -20, 2.0 ** -16, 2.0 ** -14, 2.0 ** -6, 1.0, 2.0 ** 9, None):
        s = 65504 / np.abs(q).max(axis=1, keepdims=True) if scale is None else scale
        rows += list((q * s).astype(F16))                              # one vector per row
    ext = np.where(rng.random((12, d)) < 0.2, F16(65504), F16(2.0 ** -24)).astype(F16)
    ext *= np.where(rng.random((12, d)) < 0.5, F16(1), F16(-1))
    rows += list(ext)
    mixed = (10.0 ** rng.uniform(-7, 4.8, (60, d)) * np.where(rng.random((60, d)) < 0.5, 1, -1)).astype(F16)
    rows += list(mixed)
    x = np.stack(rows).astype(F16)
    lens = [1] * (len(q) * 7)                                          # the scaled copies: one per row
    while sum(lens) < len(x):
        lens.append(min(int(rng.integers(1, 4)), len(x) - sum(lens)))
    assert np.isfinite(x.astype(F32)).all() and (np.abs(x.astype(F32)).max(axis=1) > 0).all()
    return x, offsets_of(lens)


def test_fp16_band_holds_on_adversarial_inputs_and_a_band_without_the_query_term_does_not():
    rng = np.random.default_rng(41)
    d = 64
    q = np.stack([_unit_at_midpoints(rng, d, up) for up in (True, False, True, True, False, True)])
    x16, off = adversarial_f16_column(rng, q)
    # subnormal fp16 components and +-65504 are present
    ax = np.abs(x16.astype(F32))
    assert ((ax > 0) & (ax < 2.0 ** -14)).any() and (ax == 65504).any()
    qoff = offsets_of([1, 2, 3])
    D = distances(x16.astype(F32), off, q, qoff)
    A = _approx_maxsim_f16(q, x16, off, qoff)
    worst_full, worst_noq = 0.0, 0.0
    for b in range(3):
        nq = int(qoff[b + 1] - qoff[b])
        err = np.nanmax(np.abs(A[b].astype(np.float64) - D[b]))
        worst_full = max(worst_full, err / mv_band_f16(nq, d))
        worst_noq = max(worst_noq, err / mv_band_f16(nq, d, query_term=False))
        # every consumer decision: the k-th approximate distance + 2 E (rounded up) admits the true top-k
        for k in (1, 3, 10):
            tau = np.sort(A[b][~np.isnan(A[b])])[k - 1]
            thr = np.nextafter(F32(tau + F32(2) * mv_band_f16(nq, d)), F32(np.inf))
            admitted = set(np.nonzero(A[b] <= thr)[0])
            order = np.lexsort((np.arange(D.shape[1]), D[b]))
            true_top = [r for r in order if not np.isnan(D[b, r])][:k]
            assert set(true_top) <= admitted
    assert worst_full <= 1.0                                 # the band holds
    assert worst_noq > 1.0                                   # without the query's rounding term it does not


def test_fp16_band_is_narrower_than_the_f32_handles():
    from tests.test_multivec_host import mv_band
    for nq in (1, 32, 1030, 4096):
        for d in (8, 128, 4096):
            assert mv_band_f16(nq, d) < mv_band(nq, d)

"""Float16 multivector handles (lgpu_multivec_open_f16): the vectors stay float16, 2 bytes per element.

Every fp16 handle must return what an f32 handle opened on the same rows converted to f32 returns -- same ids, counts
and distance bits -- and both the C oracle's (tests/multivec_oracle.c) on the upcast rows.  Covered: the exact route
(T < 65536, and dim not a multiple of 8 at T >= 65536) and the tensor-core route (T >= 65536, dim a multiple of 8),
confirmed by the profiling counters; variable, empty and null rows; query vector counts from 1 to 300; B 1, 64 and
300; k 10, 100 and 2049; row ids, prefilter, distance_range and deleted rows; both placements (HBM, and pinned host
memory with LGPU_MULTIVEC_HBM_BYTES=0), and many chunks and passes under a small LGPU_WS_BYTES; stored subnormals,
+-65504, inf components, zero vectors and NaN; the fix-up on near-duplicate rows and bad query vectors; the device
entry point and timeout_ms; byte accounting; the tensor-core score's band on adversarial inputs
(lgpu_debug_maxsim_gemm_f16); and a float16 column through Table, the async surface and remote.handle_query."""
import asyncio
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native, remote
from lancedb_b200.aio import AsyncTable
from tests.multivec_oracle import distances, flat_search_mv, offsets_of
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAR = "LGPU_MULTIVEC_HBM_BYTES"
F16, F32 = np.float16, np.float32


def _latent16(rng, n, dim):
    A = rng.standard_normal((8, dim)).astype(F32)
    return (rng.standard_normal((n, 8)).astype(F32) @ A + 0.3 * rng.standard_normal((n, dim))).astype(F16)


def _stats(fn):
    _native.set_profiling(True)
    try:
        return fn(), _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _open(x16, off, monkeypatch, **kw):
    """(fp16 HBM handle, fp16 host handle, f32 HBM handle on the upcast rows)"""
    monkeypatch.delenv(VAR, raising=False)
    h16 = _native.GpuMultivec(x16, off, **kw)
    f32 = _native.GpuMultivec(x16.astype(F32), off, **kw)
    monkeypatch.setenv(VAR, "0")
    host16 = _native.GpuMultivec(x16, off, **kw)
    monkeypatch.delenv(VAR)
    assert h16.dtype == F16 and host16.dtype == F16 and f32.dtype == F32
    assert host16.rows_on_host and not h16.rows_on_host and not f32.rows_on_host
    return h16, host16, f32


def _all(handles, q, qoff, k, what, **kw):
    """every handle's result equal to the f32 handle's (the last), and the same route; returns (result, stats)"""
    ref, sref = _stats(lambda: handles[-1].search(q, k=k, q_offsets=qoff, **kw))
    for h in handles[:-1]:
        got, st = _stats(lambda: h.search(q, k=k, q_offsets=qoff, **kw))
        assert_same(got, ref, f"{what}: fp16 ({'host' if h.rows_on_host else 'HBM'}) against f32")
        assert st["queries"] == sref["queries"], (what, st, sref)
        assert (st["rescored"] < st["queries"] * handles[-1].nrows) == (sref["rescored"] < sref["queries"] *
                                                                         handles[-1].nrows), (what, st, sref)
    return ref, sref


def _prefix(res, k):
    ids, dist, cnt = res
    return ids[:, :k], dist[:, :k], np.minimum(cnt, k).astype(cnt.dtype)


# (name, row lengths, dim, tensor-core route)
COLUMNS = [("exact", (0, 12, 3000), 36, False), ("tensor-core", (0, 9, 20000), 32, True),
           ("dim30", (1, 9, 16000), 30, False)]


@pytest.fixture(scope="module", params=COLUMNS, ids=[c[0] for c in COLUMNS])
def column(request):
    name, (lo, hi, n), dim, tc = request.param
    rng = np.random.default_rng(dim + n + 1)
    lens = rng.integers(lo, hi, n)
    lens[n // 2] = lens[3]
    off = offsets_of(lens)
    x = _latent16(rng, int(off[-1]), dim)
    x[off[n // 2]:off[n // 2 + 1]] = x[off[3]:off[4]]             # a duplicate row: a tie broken by id
    mp = pytest.MonkeyPatch()
    hs = _open(x, off, mp)
    mp.undo()
    yield name, x, off, hs, tc, rng
    for h in hs:
        h.close()


def test_fp16_handles_equal_the_f32_handle_and_the_oracle(column):
    name, x, off, hs, tc, rng = column
    N, dim = off.size - 1, x.shape[1]
    x32 = x.astype(F32)
    lens = rng.integers(1, 9, 300)
    lens[[0, 7]] = [300, 1]                                        # a query of 300 vectors, and one of 1
    qoff_all = offsets_of(lens)
    q_all = _latent16(rng, int(qoff_all[-1]), dim).astype(F32)
    q_all[:int(off[4] - off[3])] = x32[off[3]:off[4]]              # the duplicated row's vectors open query 0
    for B in (1, 64, 300):
        qoff = qoff_all[:B + 1]
        q = q_all[:int(qoff[-1])]
        want = flat_search_mv(x32, off, q, qoff, 2049, nthreads=16)
        for k in (10, 100, 2049):
            got, st = _all(hs, q, qoff, k, (name, B, k))
            assert_same(got, _prefix(want, k), (name, B, k, "against the oracle"))
            assert (st["rescored"] < B * N) == (tc and k <= 2048), (name, B, k, st)


def test_row_ids_prefilter_range_and_deletes(column, monkeypatch):
    name, x, off, _, tc, rng = column
    N = off.size - 1
    x32 = x.astype(F32)
    rid = (np.arange(N, dtype=np.uint64) * 3 + 5)[::-1].copy()
    hs = _open(x, off, monkeypatch, row_ids=rid)
    qoff = offsets_of(rng.integers(1, 17, 64))
    q = _latent16(rng, int(qoff[-1]), x.shape[1]).astype(F32)
    got, st = _all(hs, q, qoff, 20, (name, "row ids"))
    assert_same(got, flat_search_mv(x32, off, q, qoff, 20, row_ids=rid, nthreads=16), (name, "row ids: oracle"))
    assert (st["rescored"] < 64 * N) == tc
    allow = rng.random(int(rid.max()) + 1) < 0.3
    bm = _native.mask_bitmap(allow)
    got, _ = _all(hs, q, qoff, 20, (name, "prefilter"), allow=bm, allow_bits=allow.size)
    assert_same(got, flat_search_mv(x32, off, q, qoff, 20, row_ids=rid, allow=allow, nthreads=16), (name, "prefilter"))
    lo, hi = float(got[1][0, 3]), float(got[1][0, 15])
    got, _ = _all(hs, q, qoff, 20, (name, "range"), lower=lo, upper=hi)
    assert_same(got, flat_search_mv(x32, off, q, qoff, 20, row_ids=rid, lower=lo, upper=hi, nthreads=16),
                (name, "range"))
    gone = rid[rng.choice(N, N // 5, replace=False)]
    for h in hs:
        assert h.delete(gone) == gone.size
    live = np.ones(int(rid.max()) + 1, bool)
    live[gone.astype(np.int64)] = False
    got, _ = _all(hs, q, qoff, 20, (name, "deleted"))
    assert_same(got, flat_search_mv(x32, off, q, qoff, 20, row_ids=rid, allow=live, nthreads=16), (name, "deleted"))
    for h in hs:
        h.close()


def test_special_stored_values(monkeypatch):
    """Subnormals and +-65504 keep the tensor-core route; an inf component, a zero vector or a NaN sends the column to
    the exact route.  Results equal the f32 handle's and the oracle's either way."""
    rng = np.random.default_rng(61)
    off = offsets_of(rng.integers(1, 6, 25_000))
    T = int(off[-1])
    base = _latent16(rng, T, 16)
    ext = base.copy()
    ext[::5] = (ext[::5].astype(F32) * F32(2.0 ** -20)).astype(F16)            # subnormal vectors
    ext[1::5, 0] = F16(65504); ext[2::5, 3] = F16(-65504)                        # +-65504 beside ordinary components
    ext[3::97] = F16(2.0 ** -24)                                                 # the smallest subnormal everywhere
    qoff = offsets_of([4, 1, 9, 2])
    q = _latent16(rng, int(qoff[-1]), 16).astype(F32)
    q[4] = ext[1].astype(F32)                                                    # a query vector at 65504
    cases = [("subnormal and 65504", ext, True)]
    for what, spoil in (("inf", lambda v: v.__setitem__((100, 3), np.inf)), ("zero", lambda v: v.__setitem__(200, 0)),
                        ("NaN", lambda v: v.__setitem__((300, 5), np.nan))):
        v = ext.copy()
        spoil(v)
        cases.append((what, v, False))
    for what, x, tc in cases:
        hs = _open(x, off, monkeypatch)
        got, st = _all(hs, q, qoff, 10, what)
        assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 10, nthreads=16), (what, "oracle"))
        assert (st["rescored"] < 4 * (off.size - 1)) == tc, (what, st)
        for h in hs:
            h.close()


def test_the_fix_up_and_bad_query_vectors(monkeypatch):
    """Near-duplicate rows overflow every shortlist (the fix-up streams the fp16 rows for the flagged queries); a zero
    and a NaN query vector flag their queries; the next call on the same handle is unflagged."""
    rng = np.random.default_rng(62)
    v = rng.standard_normal((1, 16)).astype(F16)
    off = offsets_of(np.full(70_000, 1))
    x = np.repeat(v, 70_000, axis=0)
    x[::7, 0] = np.nextafter(x[0, 0], F16(np.inf))
    hs = _open(x, off, monkeypatch)
    q = rng.standard_normal((5, 16)).astype(F32)
    qoff = offsets_of([2, 3])
    got, st = _all(hs, q, qoff, 40, "near duplicates")
    assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 40, nthreads=16))
    for h in hs[:2]:
        _, st = _stats(lambda: h.search(q, k=40, q_offsets=qoff))
        assert st["flagged_queries"] == 2 and st["candidates"] > 2 * 1024, st
    for h in hs:
        h.close()

    off = offsets_of(rng.integers(0, 6, 30_000))
    x = _latent16(rng, int(off[-1]), 24)
    hs = _open(x, off, monkeypatch)
    qoff = offsets_of([3, 2, 4, 2])
    q = _latent16(rng, int(qoff[-1]), 24).astype(F32)
    q[3] = 0.0
    q[7] = np.nan
    got, st = _all(hs, q, qoff, 12, "bad query vectors")
    assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 12, nthreads=16))
    assert st["flagged_queries"] == 2 and got[2][1] == 0 and got[2][2] == 0
    for h in hs[:2]:
        _, st = _stats(lambda: h.search(q[:3], k=12, q_offsets=[0, 3]))
        assert st["flagged_queries"] == 0
    for h in hs:
        h.close()


def test_device_route_timeout_and_byte_accounting(monkeypatch):
    import torch
    rng = np.random.default_rng(63)
    off = offsets_of(rng.integers(1, 8, 20_000))
    T, dim = int(off[-1]), 64
    x = _latent16(rng, T, dim)
    assert T >= 65536
    h16, host16, f32 = _open(x, off, monkeypatch)
    monkeypatch.setenv(VAR, "0")
    host32 = _native.GpuMultivec(x.astype(F32), off)
    monkeypatch.delenv(VAR)
    assert f32.device_bytes - h16.device_bytes == T * dim * 4                   # f32 vectors + fp16 operand vs fp16
    assert h16.host_bytes() == 0 and host16.host_bytes() == T * dim * 2 and host32.host_bytes() == T * dim * 6
    assert host16.device_bytes == h16.device_bytes - host16.host_bytes() == host32.device_bytes
    qoff = offsets_of([5, 1, 17])
    q = _latent16(rng, int(qoff[-1]), dim).astype(F32)
    want = flat_search_mv(x.astype(F32), off, q, qoff, 16, nthreads=16)
    for h in (h16, host16):
        dq = torch.from_numpy(q).cuda()
        di = torch.empty((3, 16), dtype=torch.int64, device="cuda")
        dd = torch.empty((3, 16), dtype=torch.float32, device="cuda")
        dc = torch.empty(3, dtype=torch.int32, device="cuda")
        h.search_device(dq.data_ptr(), qoff, _native.make_params(16), di.data_ptr(), dd.data_ptr(), dc.data_ptr(),
                        torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert_same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want)
    bq = offsets_of([64] * 16)
    qq = rng.standard_normal((int(bq[-1]), dim)).astype(F32)
    with pytest.raises(TimeoutError):
        host16.search(qq, k=10, q_offsets=bq, timeout_ms=1, allow=_native.mask_bitmap(np.ones(20_000, bool)),
                      allow_bits=20_000)
    assert_same(host16.search(q, k=16, q_offsets=qoff), want)                    # the handle still works
    for h in (h16, host16, f32, host32):
        h.close()
    # below the tensor-core shape: no operand for either row type
    off = offsets_of(np.full(100, 3))
    x = _latent16(rng, 300, 12)
    h16, host16, f32 = _open(x, off, monkeypatch)
    assert f32.device_bytes - h16.device_bytes == 300 * 12 * 2 and host16.host_bytes() == 300 * 12 * 2
    assert host16.device_bytes == h16.device_bytes - host16.host_bytes()
    for h in (h16, host16, f32):
        h.close()


def test_tensor_core_score_stays_within_its_band_on_adversarial_inputs():
    from tests.test_multivec_f16_host import adversarial_f16_column, mv_band_f16
    from tests.test_multivec_host import _unit_at_midpoints
    rng = np.random.default_rng(41)
    d = 64
    q = np.stack([_unit_at_midpoints(rng, d, up) for up in (True, False, True, True, False, True)])
    x16, off = adversarial_f16_column(rng, q)
    S = _native.debug_maxsim_gemm(q, x16, off)
    E = mv_band_f16(1, d)
    worst = 0.0
    for i in range(len(q)):
        D = distances(x16.astype(F32), off, q[i:i + 1], [0, 1])[0]
        A = (F32(1) - S[i]).astype(F32)
        assert np.array_equal(np.isnan(A), np.isnan(D))
        worst = max(worst, float(np.nanmax(np.abs(A.astype(np.float64) - D))) / float(E))
    assert worst <= 1.0, worst
    assert worst > 0.05, worst                  # the inputs do exercise the band (a zero error would prove nothing)


CHILD = r"""
import os
import numpy as np
from lancedb_b200 import _native
from tests.multivec_oracle import flat_search_mv, offsets_of
from tests.util import assert_same

rng = np.random.default_rng(7)
small = int(os.environ["LGPU_WS_BYTES"]) < (4 << 20)
# rows of 4 at dim 64 (70000 vectors): at 8 MiB the tensor-core route over several 2-byte chunks per pass, at 1 MiB the
# exact route over many chunks; then variable rows with empty ones (the exact route, dim 20)
for lens, dim in ((np.full(17_500, 4), 64), (rng.integers(0, 7, 6000), 20)):
    off = offsets_of(lens)
    A = rng.standard_normal((8, dim)).astype(np.float32)
    x = (rng.standard_normal((int(off[-1]), 8)).astype(np.float32) @ A
         + 0.3 * rng.standard_normal((int(off[-1]), dim))).astype(np.float16)
    n = off.size - 1
    os.environ["LGPU_MULTIVEC_HBM_BYTES"] = "0"
    host16 = _native.GpuMultivec(x, off)
    del os.environ["LGPU_MULTIVEC_HBM_BYTES"]
    h16 = _native.GpuMultivec(x, off)
    f32 = _native.GpuMultivec(x.astype(np.float32), off)
    assert host16.rows_on_host
    qoff = offsets_of(rng.integers(1, 17, 64))
    q = rng.standard_normal((int(qoff[-1]), dim)).astype(np.float32)
    for B in (1, 64):
        for k in (10, 100):
            qo = qoff[:B + 1]
            qq = q[:int(qo[-1])]
            _native.set_profiling(True)
            want = f32.search(qq, k=k, q_offsets=qo); sw = _native.last_filter_stats()
            _native.set_profiling(False)
            for h in (h16, host16):
                assert_same(h.search(qq, k=k, q_offsets=qo), want, (dim, B, k, h.rows_on_host))
            assert (sw["rescored"] < B * n) == (dim == 64 and not small), (dim, B, k, sw)
            assert_same(want, flat_search_mv(x.astype(np.float32), off, qq, qo, k, nthreads=16), (dim, B, k, "oracle"))
    for h in (h16, host16, f32):
        h.close()
print("ok")
"""


@pytest.mark.parametrize("ws_bytes", [1 << 20, 8 << 20])
def test_many_chunks_and_passes_under_a_small_workspace_budget(ws_bytes):
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(ws_bytes))
    env.pop(VAR, None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


def test_a_float16_column_through_every_surface_opens_an_fp16_handle():
    rng = np.random.default_rng(64)
    n, dim = 3000, 16
    rows = [_latent16(rng, int(m), dim) for m in rng.integers(1, 6, n)]
    rows[5], rows[9] = None, np.zeros((0, dim), F16)                            # a null and an empty row
    data = pa.array([None if r is None else r.astype(F32).tolist() for r in rows],
                    type=pa.list_(pa.list_(pa.float16(), list_size=dim)))
    db = lancedb.connect()
    tbl = db.create_table("t", pa.table({"vector": data, "id": pa.array(np.arange(n))}))
    qv = rows[7].astype(F32) + F32(0.01)
    got = tbl.search(qv).limit(12).offset(3).with_row_id(True).to_arrow()
    mv = tbl._multivec["vector"]
    lens = [0 if r is None else len(r) for r in rows]
    off = offsets_of(lens)
    x16 = np.concatenate([r for r in rows if r is not None]).astype(F16)
    assert mv.dtype == F16 and int(off[-1]) == x16.shape[0]
    f32 = _native.GpuMultivec(x16.astype(F32), off)
    assert f32.device_bytes - mv.device_bytes == x16.size * 2                   # 2 bytes per element, not 4
    f32.close()
    ids, dist, cnt = flat_search_mv(x16.astype(F32), off, qv, [0, qv.shape[0]], 15)
    assert got["_rowid"].to_pylist() == [int(i) for i in ids[0][3:cnt[0]]]
    assert np.array_equal(np.asarray(got["_distance"].to_pylist(), F32).view(np.uint32), dist[0][3:cnt[0]].view(np.uint32))
    want = tbl.search(qv).limit(12).to_arrow()

    async def run():
        return await AsyncTable(tbl).query().nearest_to(qv).limit(12).to_arrow()

    assert asyncio.run(run()).equals(want)
    out = remote.read_ipc_file(remote.handle_query(tbl, remote.build_query_body(qv.tolist(), k=12)))
    assert out.equals(want)
    assert tbl._multivec["vector"] is mv                                       # one fp16 handle served every surface

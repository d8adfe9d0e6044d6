"""Multivector columns on the GPU: late-interaction (MaxSim) flat search (lgpu_multivec_*), ids, counts and distance
bits against the C oracle (tests/multivec_oracle.c) across row lengths, query sizes, dims, N and B, and through the
Table, async and remote surfaces."""
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
from tests.multivec_oracle import flat_search_mv, offsets_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(got, want):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc)
    assert np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


def _data(rng, lens, dim, qlens):
    off = offsets_of(lens)
    qoff = offsets_of(qlens)
    x = rng.standard_normal((int(off[-1]), dim)).astype(np.float32)
    q = rng.standard_normal((int(qoff[-1]), dim)).astype(np.float32)
    return x, off, q, qoff


def _check(x, off, q, qoff, k, row_ids=None, allow=None, **kw):
    mv = _native.GpuMultivec(x, off, row_ids=row_ids)
    bm, bits = (None, 0) if allow is None else (_native.mask_bitmap(allow), len(allow))
    got = mv.search(q, k=k, q_offsets=qoff, allow=bm, allow_bits=bits, **kw)
    mv.close()
    want = flat_search_mv(x, off, q, qoff, k, row_ids=row_ids, allow=allow, nthreads=8, **kw)
    _same(got, want)
    return got


@pytest.mark.parametrize("dim", [2, 64, 127, 128, 768])
def test_dims_and_variable_rows(dim):
    rng = np.random.default_rng(dim)
    n = 600 if dim < 768 else 150
    lens = rng.integers(1, 301 if dim < 768 else 40, n)
    _check(*_data(rng, lens, dim, [1, 2, 32, 7]), k=10)


@pytest.mark.parametrize("nq", [1, 2, 32, 256, 4096])
def test_query_sizes(nq):
    rng = np.random.default_rng(nq)
    _check(*_data(rng, np.full(200, 4), 16, [nq, 1]), k=7)


@pytest.mark.parametrize("B", [1, 8, 64])
def test_batches_fixed_rows(B):
    rng = np.random.default_rng(B)
    _check(*_data(rng, np.full(3000, 8), 32, rng.integers(1, 40, B)), k=20)


def _stats(fn):
    _native.set_profiling(True)
    try:
        return fn(), _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _latent(rng, n, dim):
    A = rng.standard_normal((8, dim)).astype(np.float32)
    return (rng.standard_normal((n, 8)).astype(np.float32) @ A + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)


@pytest.mark.parametrize("B", [1, 8, 64])
def test_many_rows_take_the_tensor_core_path(B):
    """>= 100 000 rows, variable lengths 1..8: the fp16 MaxSim GEMM + shortlist + exact re-score, bit for bit."""
    rng = np.random.default_rng(7 + B)
    off = offsets_of(rng.integers(1, 9, 100_000))
    x = _latent(rng, int(off[-1]), 32)
    qoff = offsets_of(rng.integers(1, 33, B))
    q = _latent(rng, int(qoff[-1]), 32)
    mv = _native.GpuMultivec(x, off)
    got, st = _stats(lambda: mv.search(q, k=25, q_offsets=qoff))
    mv.close()
    _same(got, flat_search_mv(x, off, q, qoff, 25, nthreads=8))
    assert st["queries"] == B and st["rescored"] < B * 100_000          # a shortlist, not every row
    assert st["candidates"] >= 25 * B and st["flagged_queries"] < B


def test_tensor_core_path_colbert_shape():
    rng = np.random.default_rng(21)
    off = offsets_of(np.full(2000, 128))
    x = _latent(rng, int(off[-1]), 128)
    qoff = offsets_of([32, 32, 7])
    q = _latent(rng, int(qoff[-1]), 128)
    mv = _native.GpuMultivec(x, off)
    got, st = _stats(lambda: mv.search(q, k=10, q_offsets=qoff))
    mv.close()
    _same(got, flat_search_mv(x, off, q, qoff, 10, nthreads=8))
    assert st["rescored"] < 3 * 2000 and st["flagged_queries"] == 0


def test_near_duplicate_rows_take_the_fix_up():
    """All-equal rows: every row lies inside the band, the shortlists overflow, every query is redone exactly (and
    says so in lgpu_last_filter_stats); ties come back in row-id order."""
    rng = np.random.default_rng(22)
    v = rng.standard_normal((1, 16)).astype(np.float32)
    off = offsets_of(np.full(70_000, 1))
    x = np.repeat(v, 70_000, axis=0)
    x[::7] += np.float32(1e-7)                               # near duplicates
    q = rng.standard_normal((5, 16)).astype(np.float32)
    qoff = offsets_of([2, 3])
    mv = _native.GpuMultivec(x, off)
    got, st = _stats(lambda: mv.search(q, k=40, q_offsets=qoff))
    mv.close()
    _same(got, flat_search_mv(x, off, q, qoff, 40, nthreads=8))
    assert st["flagged_queries"] == 2 and st["candidates"] > 2 * 1024


def test_tensor_core_path_with_bad_query_vectors_and_next_call():
    rng = np.random.default_rng(23)
    off = offsets_of(rng.integers(0, 6, 30_000))
    x = _latent(rng, int(off[-1]), 24)
    qoff = offsets_of([3, 2, 4])
    q = _latent(rng, int(qoff[-1]), 24)
    q[3] = 0.0                                               # query 1: a zero vector -> no rows, via the fix-up
    mv = _native.GpuMultivec(x, off)
    got, st = _stats(lambda: mv.search(q, k=12, q_offsets=qoff))
    _same(got, flat_search_mv(x, off, q, qoff, 12, nthreads=8))
    assert got[2][1] == 0 and st["flagged_queries"] == 1
    q2 = q[:3]
    _same(mv.search(q2, k=12), flat_search_mv(x, off, q2, [0, 3], 12, nthreads=8))
    mv.close()


def test_debug_maxsim_gemm_is_within_the_band_of_the_exact_similarity():
    from tests.multivec_oracle import cosine_matrix_np
    rng = np.random.default_rng(24)
    off = offsets_of(rng.integers(0, 5, 300))
    x = rng.standard_normal((int(off[-1]), 64)).astype(np.float32)
    q = rng.standard_normal((20, 64)).astype(np.float32)
    got = _native.debug_maxsim_gemm(q, x, off)
    cos = cosine_matrix_np(q, x)
    e = float(_mv_band(1, 64))
    for r in range(300):
        seg = cos[:, int(off[r]):int(off[r + 1])]
        if seg.shape[1] == 0:
            assert np.isnan(got[:, r]).all()
            continue
        exact = 1.0 - seg.min(axis=1).astype(np.float64)                  # the exact max similarity
        assert np.all(np.abs(got[:, r].astype(np.float64) - exact) <= e)


def _mv_band(nq, d):
    from tests.test_multivec_host import mv_band
    return mv_band(nq, d)


def test_timeout_is_reported_and_the_handle_still_works():
    rng = np.random.default_rng(25)
    x, off, q, qoff = _data(rng, np.full(20_000, 64), 128, [64] * 16)
    mv = _native.GpuMultivec(x, off)
    with pytest.raises(TimeoutError):
        mv.search(q, k=10, q_offsets=qoff, timeout_ms=1, allow=_native.mask_bitmap(np.ones(20_000, bool)),
                  allow_bits=20_000)
    small = q[:2]
    _same(mv.search(small, k=5), flat_search_mv(x, off, small, [0, 2], 5, nthreads=8))
    mv.close()


def test_small_and_empty_columns():
    rng = np.random.default_rng(8)
    for lens in ([], [3], [2, 0, 5]):
        x, off, q, qoff = _data(rng, lens, 12, [2, 1])
        got = _check(x, off, q, qoff, k=10)
        assert list(got[2]) == [sum(1 for n in lens if n > 0)] * 2
    mv = _native.GpuMultivec(*_data(rng, [2, 2], 12, [1])[:2])
    ids, dist, cnt = mv.search([], k=5)                      # B = 0
    assert ids.shape == (0, 5) and cnt.shape == (0,)
    mv.close()


def test_empty_null_zero_and_nan_behave_as_the_contract_says():
    rng = np.random.default_rng(9)
    lens = rng.integers(0, 5, 500)
    x, off, q, qoff = _data(rng, lens, 24, [1, 3, 2, 2])
    x[5] = 0.0                                               # a zero stored vector: its pairs are skipped
    q[2] = 0.0                                               # query 1 holds a zero vector: no rows
    q[7, 3] = np.nan                                         # query 3 holds a NaN component: no rows
    mv = _native.GpuMultivec(x, off)
    got = mv.search(q, k=30, q_offsets=qoff)
    _same(got, flat_search_mv(x, off, q, qoff, 30))
    assert got[2][1] == 0 and got[2][3] == 0 and got[2][0] == 30
    assert not np.isin(got[0][0], np.nonzero(lens == 0)[0]).any()
    nxt = mv.search(q[:1], k=30)                             # the next call still works
    _same(nxt, flat_search_mv(x, off, q[:1], [0, 1], 30))
    mv.close()


def test_ties_in_row_id_order_range_prefilter_offset_and_row_ids():
    rng = np.random.default_rng(10)
    v = rng.standard_normal((1, 16)).astype(np.float32)
    x = np.repeat(v, 400, axis=0)
    off = offsets_of(np.full(200, 2))
    q = rng.standard_normal((3, 16)).astype(np.float32)
    got = _check(x, off, q, [0, 1, 3], k=50)
    assert list(got[0][0]) == list(range(50))
    x, off, q, qoff = _data(rng, rng.integers(1, 12, 5000), 40, [4, 1, 9])
    allow = rng.random(6000) < 0.1
    _check(x, off, q, qoff, k=64, allow=allow)
    _check(x, off, q, qoff, k=2048)                          # SELECT_KMAX
    full = _check(x, off, q, qoff, k=100)
    lo, hi = float(full[1][0, 10]), float(full[1][0, 60])
    _check(x, off, q, qoff, k=100, lower=lo, upper=hi)
    rid = rng.permutation(10_000)[:5000].astype(np.uint64)
    _check(x, off, q, qoff, k=30, row_ids=rid, allow=rng.random(10_000) < 0.5)


def test_device_entry_point_consecutive_shapes_and_closed_handle():
    import torch
    rng = np.random.default_rng(11)
    x, off, q, qoff = _data(rng, rng.integers(0, 20, 3000), 64, [5, 1, 17])
    mv = _native.GpuMultivec(x, off)
    want = flat_search_mv(x, off, q, qoff, 16, nthreads=8)
    dq = torch.from_numpy(q).cuda()
    di = torch.empty((3, 16), dtype=torch.int64, device="cuda")
    dd = torch.empty((3, 16), dtype=torch.float32, device="cuda")
    dc = torch.empty(3, dtype=torch.int32, device="cuda")
    mv.search_device(dq.data_ptr(), qoff, _native.make_params(16), di.data_ptr(), dd.data_ptr(), dc.data_ptr(),
                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want)
    # same B, different per-query vector counts, back to back (host calls are never replayed from a graph)
    for lens in ([5, 1, 17], [1, 17, 5], [5, 1, 17], [2, 2, 2], [5, 1, 17]):
        qo = offsets_of(lens)
        qq = q[:int(qo[-1])]
        _same(mv.search(qq, k=16, q_offsets=qo), flat_search_mv(x, off, qq, qo, 16, nthreads=8))
    h = mv._h
    mv.close()
    qo = np.ascontiguousarray(qoff, np.uint32)
    ids, dist, cnt = np.empty((3, 16), np.uint64), np.empty((3, 16), np.float32), np.empty(3, np.uint32)
    with pytest.raises(ValueError, match="closed"):
        _native.check(_native.load().lgpu_multivec_search(h, q.ctypes.data, qo.ctypes.data, 3,
                                                          _native.C.byref(_native.make_params(16)), ids.ctypes.data,
                                                          dist.ctypes.data, cnt.ctypes.data))


def test_invalid_input_messages():
    rng = np.random.default_rng(12)
    x, off, q, qoff = _data(rng, [3, 4], 8, [2])
    mv = _native.GpuMultivec(x, off)
    lib, C = _native.load(), _native.C
    ids, dist, cnt = np.empty((2, 4), np.uint64), np.empty((2, 4), np.float32), np.empty(2, np.uint32)
    for bad in ([0, 2, 2], [1, 2, 3], [0, 4097, 4098]):
        o = np.asarray(bad, np.uint32)
        qq = np.zeros((int(o[-1]), 8), np.float32)
        rc = lib.lgpu_multivec_search(mv._h, qq.ctypes.data, o.ctypes.data, 2, C.byref(_native.make_params(4)),
                                      ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
        assert rc == _native.LGPU_INVALID_INPUT and lib.lgpu_last_error()
    mv.close()
    o = np.asarray([0, 2, 1], np.uint64)
    h = C.c_void_p()
    assert lib.lgpu_multivec_open(x.ctypes.data, o.ctypes.data, 2, 8, None, 0, C.byref(h)) == _native.LGPU_INVALID_INPUT
    big = np.asarray([0, (1 << 20) + 1], np.uint64)
    assert lib.lgpu_multivec_open(x.ctypes.data, big.ctypes.data, 1, 8, None, 0, C.byref(h)) == _native.LGPU_INVALID_INPUT
    # the limits themselves are accepted: 4096 vectors per query (test_query_sizes) and 2^16 vectors in one row
    lens = [1 << 16, 3]
    _check(*_data(rng, lens, 4, [3]), k=2)


_ENV_SCRIPT = """
import numpy as np
from lancedb_b200 import _native
from tests.multivec_oracle import offsets_of
rng = np.random.default_rng(13)
off = offsets_of(rng.integers(0, 30, 20000))
x = rng.standard_normal((int(off[-1]), 32)).astype(np.float32)
qoff = offsets_of(rng.integers(1, 50, 12))
q = rng.standard_normal((int(qoff[-1]), 32)).astype(np.float32)
mv = _native.GpuMultivec(x, off)
i, d, c = mv.search(q, k=40, q_offsets=qoff)
np.savez({dst!r}, i=i, d=d, c=c)
"""


def test_default_no_tensor_core_and_small_workspace_agree(tmp_path):
    """LGPU_WS_BYTES (read once per process, hence the subprocesses): at 1 MiB the batch runs as sub-batches of
    queries, blocks of query vectors and many row chunks, and must return the same bits as the default run.  (The
    other search kinds under a small budget: tests/test_gpu_sub_batches.py.)"""
    from tests.multivec_oracle import flat_search_mv as ref
    res = {}
    for name, extra in (("default", {}), ("notc", {"LGPU_NO_TENSOR_CORE": "1"}), ("ws", {"LGPU_WS_BYTES": str(1 << 20)})):
        dst = str(tmp_path / f"{name}.npz")
        env = dict(os.environ, PYTHONPATH=ROOT, **extra)
        r = subprocess.run([sys.executable, "-c", _ENV_SCRIPT.format(dst=dst)], cwd=ROOT, env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        res[name] = np.load(dst)
    for name in ("notc", "ws"):
        for f in ("i", "d", "c"):
            assert np.array_equal(res[name][f], res["default"][f]), (name, f)
    rng = np.random.default_rng(13)
    off = offsets_of(rng.integers(0, 30, 20000))
    x = rng.standard_normal((int(off[-1]), 32)).astype(np.float32)
    qoff = offsets_of(rng.integers(1, 50, 12))
    q = rng.standard_normal((int(qoff[-1]), 32)).astype(np.float32)
    _same((res["default"]["i"], res["default"]["d"], res["default"]["c"]), ref(x, off, q, qoff, 40, nthreads=8))


def test_profiling_stats():
    rng = np.random.default_rng(14)
    x, off, q, qoff = _data(rng, rng.integers(1, 5, 700), 8, [2, 3])
    mv = _native.GpuMultivec(x, off)
    _native.set_profiling(True)
    try:
        mv.search(q, k=5, q_offsets=qoff)
        st = _native.last_filter_stats()
    finally:
        _native.set_profiling(False)
    mv.close()
    assert st == {"candidates": 0, "rescored": 2 * 700, "flagged_queries": 0, "queries": 2}    # exact path (T < 65536)


@pytest.mark.parametrize("vt", [pa.float16(), pa.float32(), pa.float64()])
def test_reference_multivector_relations_through_every_surface(vt):
    """python/python/tests/test_query.py:791-850 without the index: [q] -> [q, q] doubles every distance, dimension
    mismatches raise; the same rows through Table, the async surface and remote.handle_query."""
    db = lancedb.connect()
    data = [[[i, i + 1], [i + 2, i + 3]] for i in range(256)]
    df = pa.table({"vector": pa.array(data, type=pa.list_(pa.list_(vt, list_size=2))),
                   "id": pa.array(list(range(1, 257))), "float_field": pa.array([float(i) for i in range(1, 257)])})
    tbl = db.create_table("test", df)
    rs = tbl.search([1, 2]).to_arrow()
    rs2 = tbl.search([[1, 2], [1, 2]]).to_arrow()
    assert len(rs2) == len(rs) == 10 and "query_index" not in rs2.column_names
    for i in range(2):
        assert rs2["_distance"][i].as_py() == rs["_distance"][i].as_py() * 2
    with pytest.raises(Exception):
        tbl.search([1, 2, 3]).to_arrow()
    with pytest.raises(Exception):
        tbl.search([[1, 2], [1, 2, 3]]).to_arrow()
    vals = np.asarray(data, np.float32).reshape(-1, 2)
    if vt == pa.float16():
        vals = vals.astype(np.float16).astype(np.float32)
    want = flat_search_mv(vals, offsets_of(np.full(256, 2)), np.array([[1, 2], [1, 2]], np.float32), [0, 2], 10)
    assert np.array_equal(rs2["_distance"].to_numpy().view(np.uint32), want[1][0].view(np.uint32))

    async def run():
        at = AsyncTable(tbl)
        a = await at.query().nearest_to([[1, 2], [1, 2]]).to_arrow()
        b = await at.query().nearest_to([1, 2]).add_query_vector([1, 2]).to_arrow()
        with pytest.raises(Exception):
            await at.query().nearest_to([[1, 2], [1, 2, 3]]).to_arrow()
        return a, b

    a, b = asyncio.run(run())
    assert a.equals(rs2) and b.equals(rs2)
    out = remote.read_ipc_file(remote.handle_query(tbl, remote.build_query_body([[1, 2], [1, 2]], k=10)))
    assert out.equals(rs2)
    pre = tbl.search([[1, 2], [3, 1]]).where("id > 200").limit(5).with_row_id(True).to_arrow()
    assert len(pre) == 5 and min(pre["id"].to_pylist()) > 200
    assert len(tbl.search([[1, 2]]).limit(1000).to_arrow()) == 256          # k > N

"""Multivector handles whose vectors are kept in pinned host memory (LGPU_MULTIVEC_HBM_BYTES=0) and streamed through the
GPU.

Every column is opened twice from the same rows, with its row data in HBM and on the host; the two handles must return
the same ids, counts and distance bits, and both the C oracle's (tests/multivec_oracle.c).  Covered: columns on both
sides of the tensor-core threshold (65536 stored vectors), a dim that is not a multiple of 8, variable rows with empty
ones; B 1, 7 and 64; k 1, 10, 2048, 2049 and k > N; explicit row ids, a prefilter, distance_range and deleted rows; the
shortlist fix-up, zero / NaN query vectors and a stored NaN vector; timeout_ms; the host, filtered and device routes;
the profiling counters; byte accounting.  Then many chunks and several passes under a small LGPU_WS_BYTES (read once per
process, so in a child process), with near-duplicate rows in different chunks, the LGPU_OOM refusal of a row too long
to stage, and a Table end to end."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests.multivec_oracle import flat_search_mv, offsets_of
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAR = "LGPU_MULTIVEC_HBM_BYTES"


def _open_both(x, off, monkeypatch, **kw):
    """(HBM handle, host handle) of the same rows"""
    monkeypatch.delenv(VAR, raising=False)
    hbm = _native.GpuMultivec(x, off, **kw)
    monkeypatch.setenv(VAR, "0")
    host = _native.GpuMultivec(x, off, **kw)
    monkeypatch.delenv(VAR)
    assert host.rows_on_host and not hbm.rows_on_host
    return hbm, host


def _stats(fn):
    _native.set_profiling(True)
    try:
        return fn(), _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _latent(rng, n, dim):
    A = rng.standard_normal((8, dim)).astype(np.float32)
    return (rng.standard_normal((n, 8)).astype(np.float32) @ A + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)


def _prefix(res, k):
    """the top-k of a top-K result (K >= k): results are ascending by (_distance, _rowid)"""
    ids, dist, cnt = res
    return ids[:, :k], dist[:, :k], np.minimum(cnt, k).astype(cnt.dtype)


def _both(hbm, host, q, qoff, k, what, **kw):
    """the two handles' results and profiling counters equal; returns the HBM handle's result"""
    a, sa = _stats(lambda: hbm.search(q, k=k, q_offsets=qoff, **kw))
    b, sb = _stats(lambda: host.search(q, k=k, q_offsets=qoff, **kw))
    assert_same(b, a, f"{what}: host against HBM")
    assert sa == sb, (what, sa, sb)
    return a, sa


# (name, row lengths, dim): the exact route only (T < 65536), the tensor-core route (T >= 65536, dim a multiple of 8),
# and a large column whose dim is not a multiple of 8 (the exact route at T >= 65536)
COLUMNS = [("exact", (0, 12, 3000), 36), ("tensor-core", (0, 9, 20000), 32), ("dim30", (1, 9, 16000), 30)]


@pytest.fixture(scope="module", params=COLUMNS, ids=[c[0] for c in COLUMNS])
def column(request):
    name, (lo, hi, n), dim = request.param
    rng = np.random.default_rng(dim + n)
    lens = rng.integers(lo, hi, n)
    lens[n // 2] = lens[3]
    off = offsets_of(lens)
    x = _latent(rng, int(off[-1]), dim)
    x[off[n // 2]:off[n // 2 + 1]] = x[off[3]:off[4]]             # a duplicate row: a tie broken by id
    mp = pytest.MonkeyPatch()
    hbm, host = _open_both(x, off, mp)
    mp.undo()
    yield name, x, off, hbm, host, rng
    hbm.close(); host.close()


def test_host_rows_equal_hbm_rows_and_the_oracle(column):
    name, x, off, hbm, host, rng = column
    N = off.size - 1
    qoff_all = offsets_of(rng.integers(1, 33, 64))
    q_all = _latent(rng, int(qoff_all[-1]), x.shape[1])
    q_all[:int(off[4] - off[3])] = x[off[3]:off[4]]           # the duplicated row's vectors open query 0
    for B in (1, 7, 64):
        qoff = qoff_all[:B + 1]
        q = q_all[:int(qoff[-1])]
        want = flat_search_mv(x, off, q, qoff, N + 5, nthreads=16)
        for k in (1, 10, 2048, 2049, N + 5):
            got, st = _both(hbm, host, q, qoff, k, (name, B, k))
            assert_same(got, _prefix(want, k), (name, B, k, "against the oracle"))
            tc = name == "tensor-core" and k <= 2048
            assert (st["rescored"] < B * N) == tc, (name, B, k, st)


def test_row_ids_prefilter_range_and_deletes(column, monkeypatch):
    name, x, off, _, _, rng = column
    N = off.size - 1
    rid = (np.arange(N, dtype=np.uint64) * 3 + 5)[::-1].copy()
    hbm, host = _open_both(x, off, monkeypatch, row_ids=rid)
    qoff = offsets_of(rng.integers(1, 17, 7))
    q = _latent(rng, int(qoff[-1]), x.shape[1])
    got, _ = _both(hbm, host, q, qoff, 20, (name, "row ids"))
    assert_same(got, flat_search_mv(x, off, q, qoff, 20, row_ids=rid, nthreads=16), (name, "row ids: oracle"))
    allow = rng.random(int(rid.max()) + 1) < 0.3
    bm = _native.mask_bitmap(allow)
    got, _ = _both(hbm, host, q, qoff, 20, (name, "prefilter"), allow=bm, allow_bits=allow.size)
    assert_same(got, flat_search_mv(x, off, q, qoff, 20, row_ids=rid, allow=allow, nthreads=16), (name, "prefilter"))
    lo, hi = float(got[1][0, 3]), float(got[1][0, 15])
    got, _ = _both(hbm, host, q, qoff, 20, (name, "range"), lower=lo, upper=hi)
    assert_same(got, flat_search_mv(x, off, q, qoff, 20, row_ids=rid, lower=lo, upper=hi, nthreads=16), (name, "range"))
    gone = rid[rng.choice(N, N // 5, replace=False)]
    assert hbm.delete(gone) == gone.size and host.delete(gone) == gone.size
    live = np.ones(int(rid.max()) + 1, bool)
    live[gone.astype(np.int64)] = False
    got, _ = _both(hbm, host, q, qoff, 20, (name, "deleted"))
    assert_same(got, flat_search_mv(x, off, q, qoff, 20, row_ids=rid, allow=live, nthreads=16), (name, "deleted"))
    hbm.close(); host.close()


def test_the_fix_up_and_bad_query_vectors(monkeypatch):
    """All-equal rows overflow every shortlist (the fix-up streams the f32 rows for the flagged queries); a zero and a
    NaN query vector flag their queries; the next call on the same handle is unflagged."""
    rng = np.random.default_rng(22)
    v = rng.standard_normal((1, 16)).astype(np.float32)
    off = offsets_of(np.full(70_000, 1))
    x = np.repeat(v, 70_000, axis=0)
    x[::7] += np.float32(1e-7)
    hbm, host = _open_both(x, off, monkeypatch)
    q = rng.standard_normal((5, 16)).astype(np.float32)
    qoff = offsets_of([2, 3])
    got, st = _both(hbm, host, q, qoff, 40, "near duplicates")
    assert_same(got, flat_search_mv(x, off, q, qoff, 40, nthreads=16))
    assert st["flagged_queries"] == 2 and st["candidates"] > 2 * 1024
    hbm.close(); host.close()

    off = offsets_of(rng.integers(0, 6, 30_000))
    x = _latent(rng, int(off[-1]), 24)
    hbm, host = _open_both(x, off, monkeypatch)
    qoff = offsets_of([3, 2, 4, 2])
    q = _latent(rng, int(qoff[-1]), 24)
    q[3] = 0.0                                               # query 1: a zero vector
    q[7] = np.nan                                            # query 2: a NaN vector
    got, st = _both(hbm, host, q, qoff, 12, "bad query vectors")
    assert_same(got, flat_search_mv(x, off, q, qoff, 12, nthreads=16))
    assert st["flagged_queries"] == 2 and got[2][1] == 0 and got[2][2] == 0
    q2 = q[:3]
    got, st = _both(hbm, host, q2, [0, 3], 12, "next call")
    assert_same(got, flat_search_mv(x, off, q2, [0, 3], 12, nthreads=16))
    assert st["flagged_queries"] == 0
    hbm.close(); host.close()


def test_a_stored_nan_vector_takes_the_exact_route(monkeypatch):
    rng = np.random.default_rng(31)
    off = offsets_of(rng.integers(1, 6, 25_000))
    x = _latent(rng, int(off[-1]), 16)
    x[100, 3] = np.nan
    x[200] = 0.0
    hbm, host = _open_both(x, off, monkeypatch)
    qoff = offsets_of([4, 1, 9])
    q = _latent(rng, int(qoff[-1]), 16)
    got, st = _both(hbm, host, q, qoff, 10, "stored NaN")
    assert_same(got, flat_search_mv(x, off, q, qoff, 10, nthreads=16))
    assert st["rescored"] == 3 * 25_000
    hbm.close(); host.close()


def test_timeout_is_reported_and_the_handle_still_works(monkeypatch):
    rng = np.random.default_rng(25)
    off = offsets_of(np.full(20_000, 64))
    x = rng.standard_normal((int(off[-1]), 128)).astype(np.float32)
    monkeypatch.setenv(VAR, "0")
    mv = _native.GpuMultivec(x, off)
    assert mv.rows_on_host
    qoff = offsets_of([64] * 16)
    q = rng.standard_normal((int(qoff[-1]), 128)).astype(np.float32)
    with pytest.raises(TimeoutError):
        mv.search(q, k=10, q_offsets=qoff, timeout_ms=1, allow=_native.mask_bitmap(np.ones(20_000, bool)),
                  allow_bits=20_000)
    small = q[:2]
    assert_same(mv.search(small, k=5), flat_search_mv(x, off, small, [0, 2], 5, nthreads=16))
    mv.close()


def test_device_route_and_byte_accounting(monkeypatch):
    import torch
    rng = np.random.default_rng(11)
    off = offsets_of(rng.integers(1, 8, 20_000))
    x = _latent(rng, int(off[-1]), 64)
    T = int(off[-1])
    hbm, host = _open_both(x, off, monkeypatch)
    assert T >= 65536
    assert hbm.host_bytes() == 0 and host.host_bytes() == T * 64 * 6          # f32 vectors + the fp16 operand
    assert host.device_bytes == hbm.device_bytes - host.host_bytes()
    qoff = offsets_of([5, 1, 17])
    q = _latent(rng, int(qoff[-1]), 64)
    want = flat_search_mv(x, off, q, qoff, 16, nthreads=16)
    for h in (hbm, host):
        dq = torch.from_numpy(q).cuda()
        di = torch.empty((3, 16), dtype=torch.int64, device="cuda")
        dd = torch.empty((3, 16), dtype=torch.float32, device="cuda")
        dc = torch.empty(3, dtype=torch.int32, device="cuda")
        h.search_device(dq.data_ptr(), qoff, _native.make_params(16), di.data_ptr(), dd.data_ptr(), dc.data_ptr(),
                        torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert_same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want)
    hbm.close(); host.close()
    # below the tensor-core shape: no operand, on either side
    off = offsets_of(np.full(100, 3))
    x = _latent(rng, 300, 12)
    hbm, host = _open_both(x, off, monkeypatch)
    assert host.host_bytes() == 300 * 12 * 4 and host.device_bytes == hbm.device_bytes - host.host_bytes()
    hbm.close(); host.close()


CHILD = r"""
import numpy as np
from lancedb_b200 import _native
from tests.multivec_oracle import flat_search_mv, offsets_of
from tests.util import assert_same
import os

def both(x, off, tag):
    os.environ.pop("LGPU_MULTIVEC_HBM_BYTES", None)
    hbm = _native.GpuMultivec(x, off)
    os.environ["LGPU_MULTIVEC_HBM_BYTES"] = "0"
    host = _native.GpuMultivec(x, off)
    del os.environ["LGPU_MULTIVEC_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host, tag
    return hbm, host

rng = np.random.default_rng(5)
small = int(os.environ["LGPU_WS_BYTES"]) < (4 << 20)
# fixed rows of 4, 70000 vectors of dim 64: at 8 MiB the tensor-core route over 9 operand chunks of 1 MiB (18 f32
# chunks for the re-score's fix-up), several queries per pass; at 1 MiB the exact route (one query's approximate scores
# exceed a quarter of the budget) over 137 chunks, a few queries per pass.  Duplicate rows at both ends of the column,
# so that ties between chunks are broken by id.  Then variable rows with empty ones (the exact route, dim 20).
for lens, dim in ((np.full(17_500, 4), 64), (rng.integers(0, 7, 6000), 20)):
    off = offsets_of(lens)
    A = rng.standard_normal((8, dim)).astype(np.float32)
    x = (rng.standard_normal((int(off[-1]), 8)).astype(np.float32) @ A
         + 0.3 * rng.standard_normal((int(off[-1]), dim))).astype(np.float32)
    n = off.size - 1
    if lens[5] == lens[n - 5]:
        x[off[n - 5]:off[n - 4]] = x[off[5]:off[6]]
    hbm, host = both(x, off, dim)
    qoff = offsets_of(rng.integers(1, 17, 64))
    q = rng.standard_normal((int(qoff[-1]), dim)).astype(np.float32)
    q[:int(off[6] - off[5])] = x[off[5]:off[6]]
    for B in (1, 7, 64):
        for k in (1, 10, 100):
            qo = qoff[:B + 1]
            qq = q[:int(qo[-1])]
            _native.set_profiling(True)
            a = hbm.search(qq, k=k, q_offsets=qo); sa = _native.last_filter_stats()
            b = host.search(qq, k=k, q_offsets=qo); sb = _native.last_filter_stats()
            _native.set_profiling(False)
            assert_same(b, a, (dim, B, k))
            assert sa == sb, (dim, B, k, sa, sb)
            assert (sa["rescored"] < B * n) == (dim == 64 and not small), (dim, B, k, sa)
            assert_same(a, flat_search_mv(x, off, qq, qo, k, nthreads=16), (dim, B, k, "oracle"))
    allow = rng.random(n) < 0.5
    kw = dict(k=10, q_offsets=qoff, allow=_native.mask_bitmap(allow), allow_bits=n)
    assert_same(host.search(q, **kw), hbm.search(q, **kw), (dim, "prefilter"))
    hbm.close(); host.close()
if not small:
    print("ok")
    raise SystemExit(0)
# a row of 5000 x 64 f32 (1.28 MB) does not fit twice in a 1 MiB budget: the host handle refuses the search, the HBM
# handle serves it
off = offsets_of([3, 5000, 2])
x = rng.standard_normal((5005, 64)).astype(np.float32)
hbm, host = both(x, off, "long row")
q = x[:2].copy()
try:
    host.search(q, k=3)
    raise SystemExit("a host row too long to stage was searched")
except MemoryError as e:
    assert "5000 vectors" in str(e), e
assert_same(hbm.search(q, k=3), flat_search_mv(x, off, q, [0, 2], 3))
hbm.close(); host.close()
print("ok")
"""


@pytest.mark.parametrize("ws_bytes", [1 << 20, 8 << 20])
def test_many_chunks_and_passes_under_a_small_workspace_budget(ws_bytes):
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(ws_bytes))
    env.pop(VAR, None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


def _table_run(data, q):
    t = lancedb.connect().create_table("t", pa.table({"vector": data, "id": pa.array(np.arange(len(data)))}))
    r = t.search(q).limit(10).with_row_id(True).to_arrow()
    return (r["_rowid"].to_pylist(), np.asarray(r["_distance"].to_pylist(), np.float32).view(np.uint32),
            t._multivec["vector"].rows_on_host)


def test_table_end_to_end_with_host_rows(monkeypatch):
    rng = np.random.default_rng(19)
    rows = [rng.standard_normal((int(n), 8)).astype(np.float32) for n in rng.integers(1, 6, 500)]
    data = pa.array([r.tolist() for r in rows], type=pa.list_(pa.list_(pa.float32(), list_size=8)))
    q = rows[7] + 0.01
    monkeypatch.delenv(VAR, raising=False)
    want = _table_run(data, q)
    monkeypatch.setenv(VAR, "0")
    got = _table_run(data, q)
    assert want[2] is False and got[2] is True
    assert got[0] == want[0] and np.array_equal(got[1], want[1])

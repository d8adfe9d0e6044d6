"""Flat handles whose rows are kept in pinned host memory (LGPU_FLAT_HBM_BYTES=0) and streamed through the GPU.

Every column is opened twice from the same rows, with its rows in HBM and on the host; the two handles must return the
same ids, counts and distance bits, and both the C oracle's.  Covered: f32 and fp16 rows; l2, cosine and dot; B on both
sides of the tensor-core threshold (1, 7, 8, 300); N below 4096, above it and above 262144 (the filtering epilogue), and
a dim that is not a multiple of 8; k = 1, 10, 2048, 2049 and k > N; distance_range, a prefilter, deleted rows and
explicit row ids; appends; NaN / inf rows; the host, filtered and device routes, and a host-placed unindexed tail.
Then many chunks and many passes under a small LGPU_WS_BYTES (read once per process, so in a child process), the byte
accounting of both placements, and a Table end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest

import lancedb_b200 as lancedb
import oracle
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS
from tests import unindexed_oracle as U
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, F32 = np.float16, np.float32

# (N, dim): the exact kernels only (N < 4096, and a dim that is not a multiple of 8 at any N), the dense tensor-core
# path, and the sampled threshold with the filtering epilogue (N >= 262144)
SHAPES = [(3000, 36), (20000, 30), (20000, 64), (300000, 40)]
BS = [1, 7, 8, 300]


def _open_both(rows, monkeypatch, **kw):
    """(HBM handle, host handle) of the same rows"""
    monkeypatch.delenv("LGPU_FLAT_HBM_BYTES", raising=False)
    hbm = _native.GpuFlat(rows, **kw)
    monkeypatch.setenv("LGPU_FLAT_HBM_BYTES", "0")
    host = _native.GpuFlat(rows, **kw)
    monkeypatch.delenv("LGPU_FLAT_HBM_BYTES")
    assert host.rows_on_host and not hbm.rows_on_host
    return hbm, host


def _rows(rng, n, d, dtype):
    x = rng.standard_normal((n, d)).astype(dtype)
    m = min(16, n // 2)
    x[n // 2: n // 2 + m] = x[:m]                # duplicates in different chunks: ties broken by id across the merge
    return x


def _both(hbm, host, x, q, what, row_ids=None, **kw):
    """the two handles' results equal, and equal to the oracle's; returns them"""
    a = hbm.search(q, **kw)
    assert_same(host.search(q, **kw), a, f"{what}: host against HBM")
    assert_same(a, oracle.flat_search(x.astype(F32), q, row_ids=row_ids, nthreads=16, **kw), f"{what}: against the oracle")
    return a


@pytest.fixture(scope="module", params=[(n, d, t) for n, d in SHAPES for t in ("f32", "f16")],
                ids=[f"{n}x{d}-{t}" for n, d in SHAPES for t in ("f32", "f16")])
def column(request):
    N, d, t = request.param
    rng = np.random.default_rng(N + d + (t == "f16"))
    x = _rows(rng, N, d, F16 if t == "f16" else F32)
    mp = pytest.MonkeyPatch()
    hbm, host = _open_both(x, mp)
    mp.undo()
    yield x, hbm, host, rng
    hbm.close(); host.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_host_rows_equal_hbm_rows_and_the_oracle(column, metric):
    x, hbm, host, rng = column
    N, d = x.shape
    q = rng.standard_normal((max(BS), d)).astype(F32)
    q[3] = x[7]
    for B in BS:
        for k in (1, 10, 2048, 2049, N + 5):
            if k > 65536:
                continue
            a = hbm.search(q[:B], k=k, metric=metric)
            assert_same(host.search(q[:B], k=k, metric=metric), a, f"B {B} k {k}: host against HBM")
            if k in (10, 2049) and B in (8, 300):
                assert_same(a, oracle.flat_search(x.astype(F32), q[:B], k=k, metric=metric, nthreads=16),
                            f"B {B} k {k}: against the oracle")
    lo, hi = (0.6, 1.2) if metric != "l2" else (d * 1.5, d * 2.5)
    mask = rng.random(N) < 0.3
    bm = _native.mask_bitmap(mask)
    for B in (7, 300):
        for k in (10, 2049):
            kw = dict(k=k, metric=metric, lower=lo, upper=hi)
            a = hbm.search(q[:B], **kw)
            assert_same(host.search(q[:B], **kw), a, f"range B {B} k {k}")
            assert_same(a, oracle.flat_search(x.astype(F32), q[:B], nthreads=16, **kw), f"range oracle B {B} k {k}")
            kw = dict(k=k, metric=metric, allow=bm, allow_bits=N)
            a = hbm.search(q[:B], **kw)                 # lgpu_flat_search_filtered
            assert_same(host.search(q[:B], **kw), a, f"prefilter B {B} k {k}")
            assert_same(a, oracle.flat_search(x.astype(F32), q[:B], k=k, metric=metric, allow=mask, nthreads=16),
                        f"prefilter oracle B {B} k {k}")


def _device_search(h, q, k, metric):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    B = q.shape[0]
    ids = torch.empty((B, k), dtype=torch.int64, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    h.search_device(metric, dq.data_ptr(), B, _native.make_params(k, 0, 0), ids.data_ptr(), dist.data_ptr(),
                    cnt.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("dtype", [F32, F16])
def test_row_ids_deletes_and_the_device_route(dtype, monkeypatch):
    rng = np.random.default_rng(5 + (dtype == F16))
    N, d = 20000, 64
    x = _rows(rng, N, d, dtype)
    ids = (rng.permutation(N).astype(np.uint64) * 3 + 11)
    hbm, host = _open_both(x, monkeypatch, row_ids=ids)
    q = rng.standard_normal((64, d)).astype(F32)
    for metric in ("l2", "cosine", "dot"):
        want = _both(hbm, host, x, q, f"row ids {metric}", row_ids=ids, k=10, metric=metric)
        assert_same(_device_search(host, q, 10, metric), want, f"device route {metric}")
        assert_same(_device_search(host, q[:3], 2049, metric), hbm.search(q[:3], k=2049, metric=metric),
                    f"device route k 2049 {metric}")
    gone = ids[rng.choice(N, N // 10, replace=False)]
    assert hbm.delete(gone) == host.delete(gone) == gone.size
    keep = ~np.isin(ids, gone)
    live = np.zeros(int(ids.max()) + 1, bool)
    live[ids[keep].astype(np.int64)] = True
    for metric in ("l2", "cosine"):
        for k in (10, 2049):
            a = hbm.search(q, k=k, metric=metric)
            assert_same(host.search(q, k=k, metric=metric), a, f"deleted {metric} k {k}")
            assert_same(a, oracle.flat_search(x.astype(F32), q, k=k, metric=metric, row_ids=ids, allow=live,
                                              nthreads=16), f"deleted oracle {metric} k {k}")
        assert_same(_device_search(host, q, 10, metric), hbm.search(q, k=10, metric=metric), f"deleted device {metric}")
    hbm.close(); host.close()


@pytest.mark.parametrize("dtype", [F32, F16])
def test_appends_grow_a_host_handle(dtype, monkeypatch):
    rng = np.random.default_rng(7 + (dtype == F16))
    d = 64
    parts = [_rows(rng, n, d, dtype) for n in (3000, 2000, 30000, 10)]
    hbm, host = _open_both(parts[0], monkeypatch)
    q = rng.standard_normal((32, d)).astype(F32)
    for i, p in enumerate(parts[1:], 1):
        hbm.append(p)
        host.append(p)
        x = np.concatenate(parts[: i + 1])
        monkeypatch.setenv("LGPU_FLAT_HBM_BYTES", "0")
        fresh = _native.GpuFlat(x)
        monkeypatch.delenv("LGPU_FLAT_HBM_BYTES")
        assert host.rows_on_host and fresh.rows_on_host and not hbm.rows_on_host
        assert host.host_bytes() >= x.nbytes
        for metric in ("l2", "cosine", "dot"):
            for k in (10, 2049):
                a = _both(hbm, host, x, q, f"append {i} {metric} k {k}", k=k, metric=metric)
                assert_same(fresh.search(q, k=k, metric=metric), a, f"append {i} {metric} k {k}: a fresh host open")
        fresh.close()
    hbm.close(); host.close()


def test_nonfinite_rows(monkeypatch):
    rng = np.random.default_rng(9)
    N, d = 20000, 64
    x = _rows(rng, N, d, F32)
    x[5, 3] = np.nan
    x[6, 0] = np.inf
    x[7, -1] = -np.inf
    x[8] *= 1e20                                     # |x|^2 overflows
    x[9] = 0.0                                       # cosine: 0 / 0
    hbm, host = _open_both(x, monkeypatch)
    q = rng.standard_normal((40, d)).astype(F32)
    q[1] = x[9]
    for metric in ("l2", "cosine", "dot"):
        for k in (10, 2049):
            _both(hbm, host, x, q, f"non-finite {metric} k {k}", k=k, metric=metric)
    x16 = _rows(rng, N, d, F16)
    x16[11, 2] = np.inf
    x16[12, 5] = np.nan
    h16, g16 = _open_both(x16, monkeypatch)
    for metric in ("l2", "cosine"):
        _both(h16, g16, x16, q, f"non-finite fp16 {metric}", k=10, metric=metric)
    for h in (hbm, host, h16, g16):
        h.close()


def test_a_host_tail_of_an_unindexed_union(monkeypatch):
    rng = np.random.default_rng(11)
    N, NT, d = 4000, 6000, 32
    x = rng.standard_normal((N, d)).astype(F32)
    data = IVF_KINDS["IVF_PQ"].train(x, num_partitions=16, num_sub_vectors=8, max_iterations=4)
    ix = _native.GpuIvfPq(data)
    tail = rng.standard_normal((NT, d)).astype(F32)
    tail_ids = np.arange(N, N + NT, dtype=np.uint64)
    hbm, host = _open_both(tail, monkeypatch, row_ids=tail_ids)
    q = rng.standard_normal((48, d)).astype(F32)
    for k in (10, 2049):
        want = U.union_search(data, tail, tail_ids, q, k, 4)
        a = ix.search_unindexed(hbm, q, k=k, nprobes=4)
        assert_same(ix.search_unindexed(host, q, k=k, nprobes=4), a, f"union k {k}: host tail against HBM tail")
        assert_same(a, want, f"union k {k}: against the oracle", prefix=True)
    allow = rng.random(N + NT) < 0.5
    bm = _native.mask_bitmap(allow)
    a = ix.search_unindexed(hbm, q, k=10, nprobes=4, allow=bm, allow_bits=N + NT)
    assert_same(ix.search_unindexed(host, q, k=10, nprobes=4, allow=bm, allow_bits=N + NT), a, "union prefilter")
    import torch
    dq = torch.from_numpy(q).cuda()
    db = torch.from_numpy(bm.view(np.int32)).cuda()
    out = []
    for tl in (hbm, host):
        ids = torch.empty((48, 10), dtype=torch.int64, device="cuda")
        dist = torch.empty((48, 10), dtype=torch.float32, device="cuda")
        cnt = torch.empty(48, dtype=torch.int32, device="cuda")
        ix.search_unindexed_device(tl, dq.data_ptr(), 48, _native.make_params(10, 4, 0), db.data_ptr(), N + NT,
                                   ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        out.append((ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)))
    assert_same(out[1], out[0], "union device route: host tail against HBM tail")
    assert_same(out[0], a, "union device route against the host route")
    for h in (ix, hbm, host):
        h.close()


def test_byte_accounting(monkeypatch):
    rng = np.random.default_rng(13)
    N, d = 20000, 64
    for dtype, es in ((F32, 4), (F16, 2)):
        x = rng.standard_normal((N, d)).astype(dtype)
        hbm, host = _open_both(x, monkeypatch)
        assert hbm.host_bytes() == 0 and host.host_bytes() == N * d * es
        operand = (0 if dtype == F16 else N * d * 2) + N * 4          # bf16 copy (f32 rows) and |x|^2
        assert hbm.device_bytes - host.device_bytes == N * d * es + operand
        hbm.close(); host.close()


CHILD = r"""
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd())
import oracle
from lancedb_b200 import _native
from tests.util import assert_same
rng = np.random.default_rng(17)
for shape in os.environ["SHAPES"].split():
    N, d, t = shape.split("x")
    N, d, dtype = int(N), int(d), np.float16 if t == "f16" else np.float32
    x = rng.standard_normal((N, d)).astype(dtype)
    x[N - 8:] = x[:8]
    hbm = _native.GpuFlat(x)
    os.environ["LGPU_FLAT_HBM_BYTES"] = "0"
    host = _native.GpuFlat(x)
    del os.environ["LGPU_FLAT_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host
    q = rng.standard_normal((200, d)).astype(np.float32)
    mask = rng.random(N) < 0.5
    for metric in ("l2", "cosine", "dot"):
        for k, B in ((10, 200), (2049, 20), (min(N + 1, 65536), 3), (1, 8)):
            kw = dict(k=k, metric=metric)
            got = host.search(q[:B], **kw)
            assert_same(got, hbm.search(q[:B], **kw), (N, metric, k, "host against HBM"))
            if k in (10, 2049):
                assert_same(got, oracle.flat_search(x.astype(np.float32), q[:B], nthreads=16, **kw),
                            (N, metric, k, "against the oracle"))
        kw = dict(k=10, metric=metric, allow=_native.mask_bitmap(mask), allow_bits=N)
        assert_same(host.search(q, **kw), hbm.search(q, **kw), (N, metric, "prefilter"))
    host.close(); hbm.close()
print("ok")
"""


@pytest.mark.parametrize("ws_bytes, shapes", [(1 << 20, "60000x64xf32 60000x64xf16 3000x64xf32"),
                                              (16 << 20, "60000x64xf32 60000x64xf16"),
                                              (48 << 20, "600000x8xf32")])
def test_many_chunks_under_a_small_workspace_budget(ws_bytes, shapes):
    """1 MiB: chunks of ~800 rows (exact kernels) and a few queries per pass at k = 2049; 16 MiB: chunks above 4096
    rows, each on the tensor cores; 48 MiB: chunks above 262144 rows (the filtering epilogue) after the first"""
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(ws_bytes), SHAPES=shapes)
    env.pop("LGPU_FLAT_HBM_BYTES", None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


def _table_run(x, extra, q):
    """flat search, bypass_vector_index after create_index, and an unindexed tail after add"""
    n = x.shape[0]
    t = lancedb.connect().create_table("t", {"id": np.arange(n), "vector": x})
    out = []

    def search(**kw):
        s = t.search(q).limit(10).with_row_id(True)
        if kw.get("bypass"):
            s = s.bypass_vector_index()
        r = s.nprobes(4).to_arrow()
        out.append((r["_rowid"].to_pylist(), np.asarray(r["_distance"].to_pylist(), F32).view(np.uint32)))

    search()
    placed = [t._flat["vector"].rows_on_host]
    t.create_index(metric="l2", num_partitions=16, num_sub_vectors=8, max_iterations=4)
    search(bypass=True)
    t.add({"id": np.arange(n, n + extra.shape[0]), "vector": extra})
    search()
    search(bypass=True)
    placed.append(t._tail["vector"].rows_on_host)
    return out, placed


def test_table_end_to_end_with_host_rows(monkeypatch):
    rng = np.random.default_rng(19)
    x = rng.standard_normal((6000, 32)).astype(F32)
    extra = rng.standard_normal((5000, 32)).astype(F32)
    q = x[11] + 0.01
    monkeypatch.delenv("LGPU_FLAT_HBM_BYTES", raising=False)
    want, placed = _table_run(x, extra, q)
    assert placed == [False, False]
    monkeypatch.setenv("LGPU_FLAT_HBM_BYTES", "0")
    got, placed = _table_run(x, extra, q)
    assert placed == [True, True]
    for step, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0] and np.array_equal(g[1], w[1]), f"step {step}"

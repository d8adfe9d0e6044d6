"""Binary handles whose packed rows are kept in pinned host memory (LGPU_BINARY_HBM_BYTES=0) and streamed through the
GPU.

Every column is opened twice from the same rows, with its rows in HBM and on the host; the two handles must return the
same ids, counts, distance bits and path counters, and both the C Hamming oracle's.  Covered: every route -- SIMT dense
(N < 4096), wgmma dense (B = 130, 4096 <= N <= 65536) and the list route (N > 65536) at B = 1, 7 and 300 -- with nbytes
3, 32 and 33; k = 1, 10, 2048, 2049 and k > N; N = 0; distance_range, a prefilter, deleted rows and explicit row ids;
the list fix-up on tie-heavy rows; appends across the threshold sample's size; the host, filtered and device entry
points.  Then many chunks and passes under a small LGPU_WS_BYTES (read once per process, so in a child process), the
byte accounting of both placements, and a Table whose binary IVF_FLAT index has a host-placed unindexed tail."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests.hamming_oracle import flat_search_u8
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIST_N = 65536 + 4464          # above the list route's sample size (HAM_SAMPLE, api.cu)


def _open_both(rows, monkeypatch, **kw):
    """(HBM handle, host handle) of the same rows"""
    monkeypatch.delenv("LGPU_BINARY_HBM_BYTES", raising=False)
    hbm = _native.GpuBinary(rows, **kw)
    monkeypatch.setenv("LGPU_BINARY_HBM_BYTES", "0")
    host = _native.GpuBinary(rows, **kw)
    monkeypatch.delenv("LGPU_BINARY_HBM_BYTES")
    assert host.rows_on_host and not hbm.rows_on_host
    return hbm, host


def _stats(fn):
    _native.set_profiling(True)
    try:
        return fn(), _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _mask(allow, allow_bits):
    return np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")[:allow_bits].astype(bool)


def _both(hbm, host, x, q, what, row_ids=None, oracle=True, **kw):
    """the two handles' results and path counters equal, and the results equal to the oracle's; returns them"""
    a, sa = _stats(lambda: hbm.search(q, **kw))
    b, sb = _stats(lambda: host.search(q, **kw))
    assert_same(b, a, f"{what}: host against HBM")
    assert sa == sb, (what, sa, sb)
    if oracle:
        okw = dict(kw)
        if "allow" in okw:
            okw["allow"] = _mask(okw["allow"], okw.pop("allow_bits"))
        k = okw.pop("k")
        assert_same(a, flat_search_u8(x, q, k, row_ids=row_ids, nthreads=16, **okw), f"{what}: against the oracle")
    return a, sa


# (B, N): SIMT dense, wgmma dense, the list route at three batch sizes
ROUTES = [(7, 3000, "simt"), (130, 20000, "wgmma_dense"), (1, LIST_N, "list"), (7, LIST_N, "list"),
          (300, LIST_N, "list")]


@pytest.fixture(scope="module", params=[(n, nb) for n in (3000, 20000, LIST_N) for nb in (3, 32, 33)],
                ids=[f"{n}x{nb}" for n in (3000, 20000, LIST_N) for nb in (3, 32, 33)])
def column(request):
    N, nb = request.param
    rng = np.random.default_rng(N + nb)
    x = rng.integers(0, 256, (N, nb), dtype=np.uint8)
    x[N // 2: N // 2 + 16] = x[:16]              # duplicates far apart: ties broken by id across chunks
    mp = pytest.MonkeyPatch()
    hbm, host = _open_both(x, mp)
    mp.undo()
    yield x, hbm, host, rng
    hbm.close(); host.close()


def test_every_route_equals_hbm_and_the_oracle(column):
    x, hbm, host, rng = column
    N, nb = x.shape
    for B, n, path in ROUTES:
        if n != N:
            continue
        q = rng.integers(0, 256, (B, nb), dtype=np.uint8)
        q[0] = x[5]
        for k in (1, 10, 2048, 2049, N + 5):
            if k > 65536:
                continue
            _, st = _both(hbm, host, x, q, f"B {B} k {k}", k=k, oracle=k in (10, 2049) or B < 300)
            if k == 10:
                assert st["rescored"] == {"simt": 0, "wgmma_dense": B * N, "list": B * (N + 65536)}[path], (path, st)
        lo, hi = 4.0 * nb - 6, 4.0 * nb + 2
        _both(hbm, host, x, q, f"range B {B}", k=10, lower=lo, upper=hi)
        _both(hbm, host, x, q, f"range B {B} k 2049", k=2049, lower=0.0, upper=4.0 * nb)
        bm = _native.mask_bitmap(rng.random(N) < 0.3)
        for k in (10, 2049):
            _both(hbm, host, x, q, f"prefilter B {B} k {k}", k=k, allow=bm, allow_bits=N)   # lgpu_binary_search_filtered


@pytest.mark.parametrize("kind", ["all_equal", "16_patterns"])
def test_tie_heavy_rows_take_the_list_fixup(kind, monkeypatch):
    rng = np.random.default_rng(11)
    if kind == "all_equal":
        x = np.tile(rng.integers(0, 256, (1, 32), dtype=np.uint8), (LIST_N, 1))
    else:
        x = rng.integers(0, 256, (16, 32), dtype=np.uint8)[rng.integers(0, 16, LIST_N)]
    row_ids = rng.permutation(LIST_N).astype(np.uint64) * 3 + 7
    hbm, host = _open_both(x, monkeypatch, row_ids=row_ids)
    q = np.concatenate([x[:4], rng.integers(0, 256, (12, 32), dtype=np.uint8)])
    _, st = _both(hbm, host, x, q, kind, row_ids=row_ids, k=10)
    assert st["flagged_queries"] > 0, st
    assert_same(_device_search(host, q, 10), hbm.search(q, k=10), f"{kind}: device route")
    hbm.close(); host.close()


def _device_search(h, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    B = q.shape[0]
    ids = torch.empty((B, k), dtype=torch.int64, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    h.search_device(dq.data_ptr(), B, _native.make_params(k, 0, 0), ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("N", [3000, 20000, LIST_N])
def test_row_ids_deletes_and_the_device_route(N, monkeypatch):
    rng = np.random.default_rng(5 + N)
    x = rng.integers(0, 256, (N, 24), dtype=np.uint8)
    ids = rng.permutation(N).astype(np.uint64) * 3 + 11
    hbm, host = _open_both(x, monkeypatch, row_ids=ids)
    q = rng.integers(0, 256, (130, 24), dtype=np.uint8)
    for B in (7, 130):
        want, _ = _both(hbm, host, x, q[:B], f"row ids B {B}", row_ids=ids, k=10)
        assert_same(_device_search(host, q[:B], 10), want, f"device route B {B}")
        assert_same(_device_search(host, q[:3], 2049), hbm.search(q[:3], k=2049), f"device route k 2049 B {B}")
    gone = ids[rng.choice(N, N // 10, replace=False)]
    assert hbm.delete(gone) == host.delete(gone) == gone.size
    live = np.zeros(int(ids.max()) + 1, bool)
    live[ids[~np.isin(ids, gone)].astype(np.int64)] = True
    for k in (10, 2049):
        a, _ = _both(hbm, host, x, q, f"deleted k {k}", oracle=False, k=k)
        assert_same(a, flat_search_u8(x, q, k, row_ids=ids, allow=live, nthreads=16), f"deleted oracle k {k}")
    assert_same(_device_search(host, q, 10), hbm.search(q, k=10), "deleted device route")
    hbm.close(); host.close()


def test_an_empty_column(monkeypatch):
    hbm, host = _open_both(np.zeros((0, 4), np.uint8), monkeypatch)
    assert host.host_bytes() == 0
    for h in (hbm, host):
        ids, dist, cnt = h.search(np.zeros((3, 4), np.uint8), k=5)
        assert (cnt == 0).all() and (ids == np.iinfo(np.uint64).max).all() and np.isinf(dist).all()
        assert h.search(np.zeros((0, 4), np.uint8), k=5)[0].shape == (0, 5)
    hbm.close(); host.close()


def test_appends_take_a_host_handle_across_the_sample_size(monkeypatch):
    rng = np.random.default_rng(7)
    nb = 33
    parts = [rng.integers(0, 256, (n, nb), dtype=np.uint8) for n in (3000, 30000, 40000, 10)]
    hbm, host = _open_both(parts[0], monkeypatch)
    q = rng.integers(0, 256, (130, nb), dtype=np.uint8)
    for i, p in enumerate(parts[1:], 1):
        hbm.append(p)
        host.append(p)
        x = np.concatenate(parts[: i + 1])
        monkeypatch.setenv("LGPU_BINARY_HBM_BYTES", "0")
        fresh = _native.GpuBinary(x)
        monkeypatch.delenv("LGPU_BINARY_HBM_BYTES")
        assert host.rows_on_host and fresh.rows_on_host and not hbm.rows_on_host
        assert host.host_bytes() >= x.shape[0] * 64
        for B in (7, 130):
            for k in (10, 2049):
                a, _ = _both(hbm, host, x, q[:B], f"append {i} B {B} k {k}", k=k)
                assert_same(fresh.search(q[:B], k=k), a, f"append {i} B {B} k {k}: a fresh host open")
        fresh.close()
    hbm.close(); host.close()


def test_byte_accounting(monkeypatch):
    rng = np.random.default_rng(13)
    for N, nb, nbp in ((20000, 33, 64), (LIST_N, 32, 32)):
        x = rng.integers(0, 256, (N, nb), dtype=np.uint8)
        hbm, host = _open_both(x, monkeypatch)
        assert hbm.host_bytes() == 0 and host.host_bytes() == N * nbp
        assert hbm.device_bytes - host.device_bytes == N * (nbp + 4)
        hbm.close(); host.close()


CHILD = r"""
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd())
from lancedb_b200 import _native
from tests.hamming_oracle import flat_search_u8
from tests.util import assert_same
rng = np.random.default_rng(17)
N = 70000
cols = [rng.integers(0, 256, (N, 32), dtype=np.uint8),
        np.tile(rng.integers(0, 256, (1, 32), dtype=np.uint8), (N, 1)),            # every list overflows
        rng.integers(0, 256, (3000, 3), dtype=np.uint8)]
for x in cols:
    n, nb = x.shape
    rid = rng.permutation(n).astype(np.uint64) * 2 + 1
    hbm = _native.GpuBinary(x, row_ids=rid)
    os.environ["LGPU_BINARY_HBM_BYTES"] = "0"
    host = _native.GpuBinary(x, row_ids=rid)
    del os.environ["LGPU_BINARY_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host
    q = np.concatenate([x[:3], rng.integers(0, 256, (197, nb), dtype=np.uint8)])
    mask = rng.random(2 * n + 2) < 0.5
    for k, B in ((10, 200), (10, 1), (2049, 20), (min(n + 1, 65536), 3)):
        got = host.search(q[:B], k=k)
        assert_same(got, hbm.search(q[:B], k=k), (n, k, B, "host against HBM"))
        if k <= 2049:
            assert_same(got, flat_search_u8(x, q[:B], k, row_ids=rid, nthreads=16), (n, k, B, "against the oracle"))
    bm = _native.mask_bitmap(mask)
    assert_same(host.search(q, k=10, allow=bm, allow_bits=mask.size), hbm.search(q, k=10, allow=bm, allow_bits=mask.size),
                (n, "prefilter"))
    assert_same(host.search(q, k=10, lower=100.0, upper=130.0), hbm.search(q, k=10, lower=100.0, upper=130.0),
                (n, "range"))
    host.close(); hbm.close()
print("ok")
"""


@pytest.mark.parametrize("ws_bytes", [1 << 20, 4 << 20])
def test_many_chunks_and_passes_under_a_small_workspace_budget(ws_bytes):
    """1 MiB: list-route chunks of ~7700 rows, one query per sub-batch, and a few queries per dense pass at k = 2049;
    4 MiB: three chunks of ~31000 rows, the fix-up's running top-k merged across them"""
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(ws_bytes))
    env.pop("LGPU_BINARY_HBM_BYTES", None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


def _table_run(x, extra, q):
    """flat Hamming search, the binary IVF_FLAT index, and its unindexed tail after add"""
    nb = x.shape[1]
    schema = pa.schema([pa.field("vector", pa.list_(pa.uint8(), nb)), pa.field("id", pa.int64())])
    t = lancedb.connect().create_table(
        "t", pa.table({"vector": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), nb),
                       "id": np.arange(x.shape[0])}, schema=schema))
    out = []

    def search(**kw):
        s = t.search(q).distance_type("hamming").limit(10).with_row_id(True)
        if kw.get("bypass"):
            s = s.bypass_vector_index()
        r = s.nprobes(4).to_arrow()
        out.append((r["_rowid"].to_pylist(), np.asarray(r["_distance"].to_pylist(), np.float32).view(np.uint32)))

    search()
    placed = [t._binary["vector"].rows_on_host]
    t.create_index(metric="hamming", num_partitions=16, index_type="IVF_FLAT", max_iterations=4)
    search()
    t.add({"vector": pa.FixedSizeListArray.from_arrays(pa.array(extra.reshape(-1)), nb),
           "id": np.arange(x.shape[0], x.shape[0] + extra.shape[0])})
    search()
    search(bypass=True)
    placed.append(t._tail["vector"].rows_on_host)
    return out, placed


def test_table_end_to_end_with_a_host_tail(monkeypatch):
    rng = np.random.default_rng(19)
    x = rng.integers(0, 256, (6000, 32), dtype=np.uint8)
    extra = rng.integers(0, 256, (5000, 32), dtype=np.uint8)
    q = x[11].copy()
    monkeypatch.delenv("LGPU_BINARY_HBM_BYTES", raising=False)
    want, placed = _table_run(x, extra, q)
    assert placed == [False, False]
    monkeypatch.setenv("LGPU_BINARY_HBM_BYTES", "0")
    got, placed = _table_run(x, extra, q)
    assert placed == [True, True]
    for step, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0] and np.array_equal(g[1], w[1]), f"step {step}"
    full = np.concatenate([x, extra])
    oi, od, oc = flat_search_u8(full, q[None], 10, nthreads=16)
    assert got[-1][0] == oi[0, :oc[0]].tolist()            # bypass_vector_index: the exact answer

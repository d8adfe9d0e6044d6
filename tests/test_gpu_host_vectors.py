"""IVF indexes whose raw vectors are kept in pinned host memory (LGPU_VECTORS_HBM_BYTES=0) and refined over PCIe.

- The host-rows refine kernel alone (lgpu_debug_refine_host) against orc_distance_f32, bit for bit: l2, cosine and dot,
  dims on both sides of 16 and of the 1024-float chunk, dims that are not a multiple of 4, UINT64_MAX positions, and rows
  and queries holding NaN, +-inf and squares that overflow.
- Every float IVF kind opened twice from the same trained data, with its vectors in HBM and on the host: ids, counts and
  distance bits equal between the two handles and equal to the kind's C oracle, over refine_factor 1, 3 and 20,
  k x refine_factor above 2048, prefilter with maximum_nprobes widening, distance_range, deleted rows, the host, device,
  async and coalesced entry points and the union with an unindexed tail.  Then the accounting of both handles.
- Sub-batches under a small LGPU_WS_BYTES (read once per process, so in a child process), and a Table end to end."""
import os
import subprocess
import sys
import threading

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
f32 = np.float32
MAX = np.iinfo(np.uint64).max
DIM, NLIST, N, NT, B = 30, 16, 4000, 500, 48        # dim 30: host rows are padded to 32 floats

KINDS = {
    "pq8-l2": ("IVF_PQ", dict(num_sub_vectors=15), "l2"),
    "pq8-cosine": ("IVF_PQ", dict(num_sub_vectors=15), "cosine"),
    "pq8-dot": ("IVF_PQ", dict(num_sub_vectors=15), "dot"),
    "pq4-l2": ("IVF_PQ", dict(num_sub_vectors=30, num_bits=4), "l2"),
    "sq-l2": ("IVF_SQ", dict(), "l2"),
    "rq-cosine": ("IVF_RQ", dict(num_bits=1), "cosine"),
    "hnsw_sq-l2": ("IVF_HNSW_SQ", dict(m=6, ef_construction=40), "l2"),
}


def _bits_or_nan(a):
    """f32 bits, with every NaN as one value: the C oracle's NaN (x86) and the GPU's differ in sign and payload, and a
    NaN distance is never returned by a search"""
    a = np.asarray(a, f32)
    return np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_refine_host_kernel_matches_the_oracle(metric):
    rng = np.random.default_rng({"l2": 1, "cosine": 2, "dot": 3}[metric])
    orc = oracle.load()
    for dim in (1, 3, 15, 16, 17, 100, 768, 1536, 4099):
        n, Bq, nc = 41, 5, 23
        x = rng.standard_normal((n, dim)).astype(f32)
        q = rng.standard_normal((Bq, dim)).astype(f32)
        x[3, dim // 2] = np.nan
        x[4, 0] = np.inf
        x[5, -1] = -np.inf
        x[6] *= 1e20                                      # squares overflow to inf
        x[7] = 0.0                                        # cosine: 0 / 0
        q[1, dim - 1] = np.nan
        q[2] *= 3e19
        q[3, 0] = -np.inf
        pos = rng.integers(0, n, (Bq, nc)).astype(np.uint64)
        pos[:, :8] = np.arange(3, 11)                     # every awkward row for every query
        pos[0, 5] = pos[4, 22] = pos[2, 0] = MAX
        got = _native.debug_refine_host(q, x, pos, metric)
        want = np.empty((Bq, nc), f32)
        m = _native.METRICS[metric]
        for b in range(Bq):
            for c in range(nc):
                p = int(pos[b, c])
                want[b, c] = np.inf if p == MAX else orc.orc_distance_f32(m, q[b].ctypes.data, x[p].ctypes.data, dim)
        assert np.array_equal(_bits_or_nan(got), _bits_or_nan(want)), f"dim {dim}"
        assert np.isposinf(got[0, 5]) and np.isposinf(got[4, 22])


def test_refine_host_kernel_refuses_a_position_outside_the_rows():
    x = np.ones((4, 8), f32)
    with pytest.raises(ValueError, match="position"):
        _native.debug_refine_host(np.ones((1, 8), f32), x, np.array([[1, 4]], np.uint64))


def _device_search(h, q, p, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    dist = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    cnt = torch.empty(q.shape[0], dtype=torch.int32, device="cuda")
    h.search_device(dq.data_ptr(), q.shape[0], p, ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _open_both(monkeypatch, kind, data):
    """(HBM handle, host handle) of the same data"""
    cls = getattr(_native, IVF_KINDS[kind].handle)
    monkeypatch.delenv("LGPU_VECTORS_HBM_BYTES", raising=False)
    hbm = cls(data, device=0)
    monkeypatch.setenv("LGPU_VECTORS_HBM_BYTES", "0")
    host = cls(data, device=0)
    monkeypatch.delenv("LGPU_VECTORS_HBM_BYTES")
    return hbm, host


@pytest.mark.parametrize("name", list(KINDS))
def test_host_placement_equals_hbm_placement_and_the_oracle(name, monkeypatch):
    # the coalescing window is read once per process: take the one the other entry-point tests use
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")
    kind, params, metric = KINDS[name]
    rng = np.random.default_rng(sorted(KINDS).index(name) + 60)
    x = rng.standard_normal((N, DIM)).astype(f32)
    data = IVF_KINDS[kind].train(x, num_partitions=NLIST, distance_type=metric, max_iterations=4, keep_vectors=True,
                                 **params)
    hbm, host = _open_both(monkeypatch, kind, data)
    assert not hbm.vectors_on_host and host.vectors_on_host
    assert hbm.host_bytes() == 0 and host.host_bytes() == N * 32 * 4
    assert hbm.device_bytes() - host.device_bytes() == N * DIM * 4
    q = rng.standard_normal((B, DIM)).astype(f32)
    q[3] = data.vectors[7]

    def both(what, want, **kw):
        a, b = hbm.search(q, **kw), host.search(q, **kw)
        assert_same(b, a, what + ": host against HBM")
        assert_same(b, want, what + ": host against the oracle")

    for rf in (1, 3, 20):
        both(f"refine_factor {rf}", U.index_search(data, q, 10, 4, rf), k=10, nprobes=4, refine_factor=rf)
    k, rf = (60, 30) if kind == "IVF_HNSW_SQ" else (150, 20)      # HNSW_SQ's beam holds at most 2048 rows
    a = hbm.search(q[:8], k=k, nprobes=NLIST, refine_factor=rf)
    assert_same(host.search(q[:8], k=k, nprobes=NLIST, refine_factor=rf), a, f"k x rf {k * rf}: host against HBM")
    assert_same(a, U.index_search(data, q[:8], k, NLIST, rf), f"k x rf {k * rf}: against the oracle")
    allow = rng.random(N) < 0.03
    bm = _native.mask_bitmap(allow)
    both("prefilter + maximum_nprobes", U.index_search(data, q, 10, 2, 3, allow=allow, max_nprobes=NLIST),
         k=10, nprobes=2, refine_factor=3, allow=bm, allow_bits=N, max_nprobes=NLIST)
    d = U.index_search(data, q[:1], 40, 4)[1][0]
    lo, hi = float(d[3]), float(d[25])
    both("distance_range", U.index_search(data, q, 10, 4, 3, lower=lo, upper=hi),
         k=10, nprobes=4, refine_factor=3, lower=lo, upper=hi)
    # the union with an unindexed tail
    tail = rng.standard_normal((NT, DIM)).astype(f32)
    tail_ids = np.arange(N, N + NT, dtype=np.uint64)
    th = _native.GpuFlat(tail, row_ids=tail_ids)
    want = U.union_search(data, tail, tail_ids, q, 10, 4, 3)
    assert_same(host.search_unindexed(th, q, k=10, nprobes=4, refine_factor=3), want, "union", prefix=True)
    assert_same(hbm.search_unindexed(th, q, k=10, nprobes=4, refine_factor=3), want, "union (HBM)", prefix=True)
    # deleted rows
    dead = rng.permutation(N)[:N // 3]
    assert hbm.delete(dead) == host.delete(dead) == dead.size
    live = np.ones(N, bool)
    live[dead] = False
    want = U.index_search(data, q, 10, 4, 5, allow=live)
    both("deleted rows", want, k=10, nprobes=4, refine_factor=5)
    # the device, async and coalesced entry points
    p = _native.make_params(10, 4, 5)
    assert_same(_device_search(host, q, p, 10), want, "device")
    ids, dist, cnt = np.empty((B, 10), np.uint64), np.empty((B, 10), f32), np.empty(B, np.uint32)
    _native.ticket_wait(host.search_async(q, p, ids, dist, cnt))
    assert_same((ids, dist, cnt), want, "async")
    res = [None] * 8

    def one(i):
        res[i] = host.search_one(q[i], k=10, nprobes=4, refine_factor=5)

    th_ = [threading.Thread(target=one, args=(i,)) for i in range(8)]
    for t in th_:
        t.start()
    for t in th_:
        t.join()
    for i in range(8):
        gi, gd, gc = res[i]
        assert gc == want[2][i] and np.array_equal(gi, want[0][i]), f"coalesced query {i}"
        assert np.array_equal(gd.view(np.uint32), want[1][i].view(np.uint32)), f"coalesced query {i}"
    for h in (hbm, host, th):
        h.close()


def test_a_handle_without_vectors_still_refuses_refine(monkeypatch):
    rng = np.random.default_rng(70)
    x = rng.standard_normal((N, DIM)).astype(f32)
    data = IVF_KINDS["IVF_SQ"].train(x, num_partitions=NLIST, max_iterations=4, keep_vectors=True)
    monkeypatch.setenv("LGPU_VECTORS_HBM_BYTES", "0")
    h = _native.GpuIvfSq(data, with_vectors=False)
    assert not h.vectors_on_host and h.host_bytes() == 0
    with pytest.raises(ValueError, match="refine_factor"):
        h.search(x[:2], k=5, nprobes=4, refine_factor=2)
    h.close()


CHILD = r"""
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd())
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS
from tests import unindexed_oracle as U
from tests.util import assert_same
rng = np.random.default_rng(71)
x = rng.standard_normal((20000, 64)).astype(np.float32)
for kind, params in (("IVF_PQ", dict(num_sub_vectors=8)), ("IVF_SQ", {})):
    data = IVF_KINDS[kind].train(x, num_partitions=64, max_iterations=4, keep_vectors=True, **params)
    cls = getattr(_native, IVF_KINDS[kind].handle)
    hbm = cls(data)
    os.environ["LGPU_VECTORS_HBM_BYTES"] = "0"
    host = cls(data)
    del os.environ["LGPU_VECTORS_HBM_BYTES"]
    assert host.vectors_on_host and not hbm.vectors_on_host, kind
    q = rng.standard_normal((3000, 64)).astype(np.float32)
    assert host.debug_sub_batch_size(3000, 8) < 3000, kind
    got = host.search(q, k=10, nprobes=8, refine_factor=10)
    assert_same(got, hbm.search(q, k=10, nprobes=8, refine_factor=10), kind + ": host against HBM")
    assert_same(got, U.index_search(data, q, 10, 8, 10), kind + ": host against the oracle")
print("ok")
"""


def test_sub_batches_under_a_small_workspace_budget():
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(1 << 20))
    env.pop("LGPU_VECTORS_HBM_BYTES", None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


def _table_run(x, extra, q):
    """create_index, a refined search, delete, add, optimize: the results and the index handle of each step"""
    t = lancedb.connect().create_table("t", {"id": np.arange(N), "grp": np.arange(N) % 3, "vector": x})
    t.create_index(metric="l2", num_partitions=NLIST, num_sub_vectors=15, max_iterations=4)
    out, on_host = [], [t._index["vector"].vectors_on_host]

    def search():
        r = t.search(q).nprobes(4).refine_factor(10).limit(10).with_row_id(True).to_arrow()
        out.append((r["_rowid"].to_pylist(), np.asarray(r["_distance"].to_pylist(), f32).view(np.uint32)))

    search()
    t.delete("grp = 0")
    search()
    t.add({"id": np.arange(N, N + 300), "grp": np.arange(N, N + 300) % 3, "vector": extra})
    search()
    t.optimize()
    on_host.append(t._index["vector"].vectors_on_host)
    search()
    return out, on_host


def test_table_end_to_end_with_host_vectors(monkeypatch):
    rng = np.random.default_rng(72)
    x = rng.standard_normal((N, DIM)).astype(f32)
    extra = rng.standard_normal((300, DIM)).astype(f32)
    q = x[11] + 0.01
    monkeypatch.delenv("LGPU_VECTORS_HBM_BYTES", raising=False)
    want, on_host = _table_run(x, extra, q)
    assert on_host == [False, False]
    monkeypatch.setenv("LGPU_VECTORS_HBM_BYTES", "0")
    got, on_host = _table_run(x, extra, q)
    assert on_host == [True, True]
    for step, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0] and np.array_equal(g[1], w[1]), f"step {step}"

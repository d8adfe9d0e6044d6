"""IVF_SQ, IVF_RQ and binary IVF_FLAT indexes whose codes are kept in pinned host memory (LGPU_CODES_HBM_BYTES=0) and
staged through HBM, the probed partitions of one chunk at a time.

- Each kind (IVF_SQ l2 and cosine, IVF_RQ l2 and cosine, binary IVF_FLAT) opened twice from the same data, codes in
  HBM and on the host: ids, counts and distance bits equal between the two handles and equal to the kind's C oracle,
  over B 1, 7, 130 and 1024, nprobes 1, a few and nlist, k 1, 10, 100 and 2049, empty partitions, prefilter with
  maximum_nprobes widening, distance_range, refine_factor with the raw vectors in HBM and on the host, deleted rows,
  the union with an unindexed tail and every entry point of the kind.  Then the accounting of both handles.
- Chunks of one to three partitions and a refused index under a small LGPU_WS_BYTES (read once per process, so in a
  child process); the kinds that keep their codes in HBM whatever the cap says; a Table end to end."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS, IvfBinaryIndexData, IvfRqIndexData, IvfSqIndexData, rq_rotation
from tests import unindexed_oracle as U
from tests.util import assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
DIM, NBYTES = 40, 20                 # SQ rows padded to 64 bytes, RQ to 256 bits, binary to 32 bytes


def _layout(rng, sizes):
    """part_offsets and permuted, non-contiguous row ids of partitions of `sizes` rows"""
    off = np.zeros(len(sizes) + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    n = int(off[-1])
    return off, (rng.permutation(n).astype(np.uint64) * 3 + 7)


def make_data(kind, metric, rng, sizes, dim=DIM, nbytes=NBYTES):
    """An index of `kind` over random codes in partitions of `sizes` rows: parity between placements and the oracle's
    contract need no training"""
    off, rid = _layout(rng, sizes)
    n, nlist = rid.size, len(sizes)
    if kind == "IVF_FLAT":
        return IvfBinaryIndexData(nbytes=nbytes, nlist=nlist, centroids=rng.integers(0, 256, (nlist, nbytes), np.uint8),
                                  part_offsets=off, vectors=rng.integers(0, 256, (n, nbytes), np.uint8), row_ids=rid)
    c = rng.standard_normal((nlist, dim)).astype(f32)
    if metric == "cosine":
        c /= np.linalg.norm(c, axis=1, keepdims=True).astype(f32)
    x = rng.standard_normal((n, dim)).astype(f32)
    if kind == "IVF_SQ":
        return IvfSqIndexData(dim=dim, nlist=nlist, metric=metric, centroids=c, part_offsets=off,
                              codes=rng.integers(0, 256, (n, dim), np.uint8), row_ids=rid, lo=-2.5, hi=2.5, vectors=x)
    return IvfRqIndexData(dim=dim, nlist=nlist, metric=metric, centroids=c, rotation=rq_rotation(dim, 5),
                          part_offsets=off, codes=rng.integers(0, 256, (n, (dim + 7) // 8), np.uint8),
                          add_factors=(rng.random(n) * 4).astype(f32), scale_factors=-(rng.random(n) * 2).astype(f32),
                          row_ids=rid, vectors=x)


def code_bytes(data):
    """the padded layout's bytes"""
    if data.index_type == "IVF_FLAT":
        return data.nrows * ((data.nbytes + 31) // 32 * 32)
    if data.index_type == "IVF_SQ":
        return data.nrows * ((data.dim + 63) // 64 * 64)
    return data.nrows * ((data.dim + 255) // 256 * 32)


def open_handle(data, env, with_vectors=True):
    """a handle of `data` opened with the placement caps in `env` (None: unset)"""
    saved = {k: os.environ.get(k) for k in env}
    try:
        for k, v in env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        cls = getattr(_native, IVF_KINDS[data.index_type].handle)
        if data.index_type == "IVF_FLAT":
            return cls(data, device=0)
        return cls(data, device=0, with_vectors=with_vectors)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


HBM = {"LGPU_CODES_HBM_BYTES": None, "LGPU_VECTORS_HBM_BYTES": None}
HOST = {"LGPU_CODES_HBM_BYTES": "0", "LGPU_VECTORS_HBM_BYTES": None}
ALL_HOST = {"LGPU_CODES_HBM_BYTES": "0", "LGPU_VECTORS_HBM_BYTES": "0"}

CASES = {
    "sq-l2": ("IVF_SQ", "l2"),
    "sq-cosine": ("IVF_SQ", "cosine"),
    "rq-l2": ("IVF_RQ", "l2"),
    "rq-cosine": ("IVF_RQ", "cosine"),
    "binary": ("IVF_FLAT", "hamming"),
}
SIZES = [700, 0, 450, 900, 30, 0, 610, 820, 300, 1, 560, 990, 400, 0, 720, 515]   # empty partitions 1, 5, 13
NLIST = len(SIZES)


def _queries(data, rng, B):
    if data.index_type == "IVF_FLAT":
        q = rng.integers(0, 256, (B, data.nbytes), np.uint8)
        q[:2] = data.vectors[[3, 500]]
        return q
    q = rng.standard_normal((B, data.dim)).astype(f32)
    q[:2] = data.vectors[[3, 500]]
    return q


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


@pytest.mark.parametrize("name", list(CASES))
def test_host_codes_equal_hbm_codes_and_the_oracle(name, monkeypatch):
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")     # read once per process: the other entry-point tests' window
    kind, metric = CASES[name]
    binary = kind == "IVF_FLAT"
    rng = np.random.default_rng(sorted(CASES).index(name) + 90)
    data = make_data(kind, metric, rng, SIZES)
    N = data.nrows
    hbm, host = open_handle(data, HBM), open_handle(data, HOST)
    assert not hbm.codes_on_host and host.codes_on_host
    assert hbm.code_host_bytes() == 0 and host.code_host_bytes() == code_bytes(data)
    if not binary:
        assert hbm.device_bytes() - host.device_bytes() == code_bytes(data)
        assert not host.vectors_on_host
    q = _queries(data, rng, 1024)

    def both(what, want, qq=q, **kw):
        a, b = hbm.search(qq, **kw), host.search(qq, **kw)
        assert_same(b, a, what + ": host against HBM")
        assert_same(b, want, what + ": host against the oracle")

    for B in (1, 7, 130, 1024):
        for nprobes in (1, 3, NLIST):
            both(f"B {B} nprobes {nprobes}", U.index_search(data, q[:B], 10, nprobes), q[:B], k=10, nprobes=nprobes)
    for k in (1, 100, 2049):
        both(f"k {k}", U.index_search(data, q[:7], k, NLIST), q[:7], k=k, nprobes=NLIST)
    both("k 100 nprobes 3", U.index_search(data, q[:130], 100, 3), q[:130], k=100, nprobes=3)
    qs = q[:130]
    allow = rng.random(N * 3 + 7) < 0.02
    bm = _native.mask_bitmap(allow)
    both("prefilter + maximum_nprobes", U.index_search(data, qs, 10, 2, allow=allow, max_nprobes=NLIST), qs,
         k=10, nprobes=2, allow=bm, allow_bits=allow.size, max_nprobes=NLIST)
    d = U.index_search(data, qs[:1], 60, 4)[1][0]
    lo, hi = float(d[3]), float(d[40])
    both("distance_range", U.index_search(data, qs, 10, 4, lower=lo, upper=hi), qs, k=10, nprobes=4, lower=lo,
         upper=hi)
    if not binary:
        both_host = open_handle(data, ALL_HOST)
        assert both_host.codes_on_host and both_host.vectors_on_host
        for rf in (3, 20):
            want = U.index_search(data, qs, 10, 4, rf)
            both(f"refine_factor {rf}", want, qs, k=10, nprobes=4, refine_factor=rf)
            assert_same(both_host.search(qs, k=10, nprobes=4, refine_factor=rf), want, f"refine_factor {rf}, "
                        "codes and vectors on the host")
        both_host.close()
    # the union with an unindexed tail
    NT = 300
    tail_ids = np.arange(N * 3 + 7, N * 3 + 7 + NT, dtype=np.uint64)
    if binary:
        tail = rng.integers(0, 256, (NT, data.nbytes), np.uint8)
        th = _native.GpuBinary(tail, row_ids=tail_ids)
    else:
        tail = rng.standard_normal((NT, data.dim)).astype(f32)
        th = _native.GpuFlat(tail, row_ids=tail_ids)
    want = U.union_search(data, tail, tail_ids, qs, 10, 4)
    assert_same(host.search_unindexed(th, qs, k=10, nprobes=4), want, "union", prefix=True)
    assert_same(hbm.search_unindexed(th, qs, k=10, nprobes=4), want, "union (HBM)", prefix=True)
    # deleted rows
    dead = rng.permutation(data.row_ids)[:N // 3]
    assert hbm.delete(dead) == host.delete(dead) == dead.size
    live = np.ones(N * 3 + 7, bool)
    live[dead.astype(np.int64)] = False
    want = U.index_search(data, qs, 10, 4, allow=live)
    both("deleted rows", want, qs, k=10, nprobes=4)
    # the device entry point, and the async and coalesced ones of the float kinds
    p = _native.make_params(10, 4)
    assert_same(_device_search(host, qs, p, 10), want, "device")
    if not binary:
        B = qs.shape[0]
        ids, dist, cnt = np.empty((B, 10), np.uint64), np.empty((B, 10), f32), np.empty(B, np.uint32)
        _native.ticket_wait(host.search_async(qs, p, ids, dist, cnt))
        assert_same((ids, dist, cnt), want, "async")
        res = [None] * 8

        def one(i):
            res[i] = host.search_one(qs[i], k=10, nprobes=4)

        ts = [threading.Thread(target=one, args=(i,)) for i in range(8)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for i in range(8):
            gi, gd, gc = res[i]
            assert gc == want[2][i] and np.array_equal(gi, want[0][i]), f"coalesced query {i}"
            assert np.array_equal(gd.view(np.uint32), want[1][i].view(np.uint32)), f"coalesced query {i}"
    for h in (hbm, host, th):
        h.close()


def test_profiled_search_counts_the_bytes_it_streamed():
    rng = np.random.default_rng(95)
    data = make_data("IVF_SQ", "l2", rng, SIZES)
    host = open_handle(data, HOST)
    q = _queries(data, rng, 2)[:1]
    _native.set_profiling(True)
    try:
        host.search(q, k=10, nprobes=NLIST)
        assert _native.last_streamed_code_bytes() == code_bytes(data)     # every partition, once
        host.search(q, k=10, nprobes=3)                                    # three partitions at most
        b = _native.last_streamed_code_bytes()
        assert b % 64 == 0 and b <= 3 * max(SIZES) * 64
    finally:
        _native.set_profiling(False)
    host.close()


CHILD = r"""
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd())
from lancedb_b200 import _native
from tests import unindexed_oracle as U
from tests.test_gpu_host_codes import make_data, open_handle, HBM, HOST
from tests.util import assert_same
rng = np.random.default_rng(96)
# LGPU_WS_BYTES = 1 MiB: a staging buffer holds 128 KiB, or the largest partition when that is larger.  Rows of 128
# bytes (SQ dim 128, binary 128 bytes) in partitions of 1 .. 1000 rows: chunks of one to three partitions, and the
# 1000-row partitions (128000 bytes) fill a chunk alone
sizes = [int(s) for s in rng.integers(250, 700, 40)]
sizes[3] = sizes[17] = 1000
sizes[9] = 0
sizes[20] = 1
for kind, metric, kw in (("IVF_SQ", "l2", dict(dim=128)), ("IVF_RQ", "cosine", dict(dim=1000)),
                         ("IVF_FLAT", "hamming", dict(nbytes=128))):
    data = make_data(kind, metric, rng, sizes, **kw)
    hbm, host = open_handle(data, HBM), open_handle(data, HOST)
    assert host.codes_on_host and not hbm.codes_on_host, kind
    B = 60 if kind == "IVF_RQ" else 300                      # (the RQ oracle at dim 1000 is the slow one)
    q = rng.integers(0, 256, (B, data.nbytes), np.uint8) if kind == "IVF_FLAT" else \
        rng.standard_normal((B, data.dim)).astype(np.float32)
    if kind != "IVF_FLAT":
        assert host.debug_sub_batch_size(300, 8) < hbm.debug_sub_batch_size(300, 8), kind
    for nprobes in (1, 8, 40):
        got = host.search(q, k=10, nprobes=nprobes)
        assert_same(got, hbm.search(q, k=10, nprobes=nprobes), f"{kind} nprobes {nprobes}: host against HBM")
        assert_same(got, U.index_search(data, q, 10, nprobes), f"{kind} nprobes {nprobes}: host against the oracle")
    hbm.close(); host.close()
# a partition whose codes (600 x 1024 bytes) cannot be staged twice in 1 MiB is refused at open
data = make_data("IVF_SQ", "l2", rng, [10, 600, 10], dim=1024)
try:
    open_handle(data, HOST)
    raise SystemExit("opened")
except MemoryError as e:
    assert "partition" in str(e), str(e)
h = open_handle(data, HBM)                                   # in HBM nothing is staged
assert not h.codes_on_host
h.close()
print("ok")
"""


def test_many_chunks_and_a_refused_index_under_a_small_workspace_budget():
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_WS_BYTES=str(1 << 20))
    env.pop("LGPU_CODES_HBM_BYTES", None)
    env.pop("LGPU_VECTORS_HBM_BYTES", None)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-6000:]


@pytest.mark.parametrize("kind,params", [("IVF_PQ", dict(num_sub_vectors=8)),
                                         ("IVF_PQ", dict(num_sub_vectors=16, num_bits=4)),
                                         ("IVF_HNSW_SQ", dict(m=6, ef_construction=40))])
def test_kinds_that_keep_their_codes_in_hbm(kind, params, monkeypatch):
    rng = np.random.default_rng(97)
    x = rng.standard_normal((3000, 32)).astype(f32)
    data = IVF_KINDS[kind].train(x, num_partitions=8, max_iterations=3, **params)
    monkeypatch.setenv("LGPU_CODES_HBM_BYTES", "0")
    h = getattr(_native, IVF_KINDS[kind].handle)(data, device=0, with_vectors=False)
    assert not h.codes_on_host and h.code_host_bytes() == 0
    q = x[:5] + 0.01
    assert_same(h.search(q, k=10, nprobes=3), U.index_search(data, q, 10, 3), kind)
    h.close()


def _table_run(x, extra, q):
    """create_index(IVF_SQ), search, add, search, optimize, delete, search: the results and the placement of each
    index handle"""
    n = x.shape[0]
    t = lancedb.connect().create_table("t", {"id": np.arange(n), "grp": np.arange(n) % 3, "vector": x})
    t.create_index(metric="l2", num_partitions=12, index_type="IVF_SQ", max_iterations=4)
    out, on_host = [], [t._index["vector"].codes_on_host]

    def search():
        r = t.search(q).nprobes(4).limit(10).with_row_id(True).to_arrow()
        out.append((r["_rowid"].to_pylist(), np.asarray(r["_distance"].to_pylist(), f32).view(np.uint32)))

    search()
    t.add({"id": np.arange(n, n + 300), "grp": np.arange(n, n + 300) % 3, "vector": extra})
    search()
    t.optimize()
    on_host.append(t._index["vector"].codes_on_host)
    t.delete("grp = 0")
    search()
    return out, on_host


def test_table_end_to_end_with_host_codes(monkeypatch):
    rng = np.random.default_rng(98)
    x = rng.standard_normal((4000, 48)).astype(f32)
    extra = rng.standard_normal((300, 48)).astype(f32)
    q = x[11] + 0.01
    monkeypatch.delenv("LGPU_CODES_HBM_BYTES", raising=False)
    want, on_host = _table_run(x, extra, q)
    assert on_host == [False, False]
    monkeypatch.setenv("LGPU_CODES_HBM_BYTES", "0")
    got, on_host = _table_run(x, extra, q)
    assert on_host == [True, True]
    for step, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0] and np.array_equal(g[1], w[1]), f"step {step}"

"""Binary vectors on the GPU: Hamming-distance flat search (lgpu_binary_*) and the b1 tensor-core kernel, bit for bit
against the CPU oracle, on every path (SIMT dense, wgmma dense, wgmma list + dense fix-up) reached by shape."""
import asyncio
import json

import numpy as np
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests.hamming_oracle import flat_search_u8, hamming_u8

pytestmark = pytest.mark.gpu

LIST_N = 65536 + 4464          # above the list path's sample size (HAM_SAMPLE, api.cu)


def _stats(fn):
    _native.set_profiling(True)
    try:
        out = fn()
        return out, _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _same(got, want):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc)
    assert np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))


def _check(x, q, k, row_ids=None, **kw):
    bx = _native.GpuBinary(x, row_ids=row_ids)
    got, st = _stats(lambda: bx.search(q, k=k, **kw))
    allow = kw.pop("allow", None)
    mask = None
    if allow is not None:
        bits = np.unpackbits(np.asarray(allow, np.uint32).view(np.uint8), bitorder="little")
        mask = bits[:kw.pop("allow_bits")].astype(bool)
    _same(got, flat_search_u8(x, q, k, row_ids=row_ids, allow=mask, **kw))
    bx.close()
    return st


@pytest.mark.parametrize("B,N,nbytes", [(1, 1, 1), (7, 130, 3), (8, 128, 8), (129, 257, 33), (130, 1000, 160),
                                        (64, 300, 128), (3, 4099, 32)])
def test_debug_hamming_gemm_equals_numpy(B, N, nbytes):
    rng = np.random.default_rng(B * 1000 + nbytes)
    q = rng.integers(0, 256, (B, nbytes), dtype=np.uint8)
    x = rng.integers(0, 256, (N, nbytes), dtype=np.uint8)
    x[0] = 255
    q[0] = 0
    assert np.array_equal(_native.debug_hamming_gemm(q, x), hamming_u8(q, x))


@pytest.mark.parametrize("nbytes", [1, 3, 8, 32, 33, 128, 160])
def test_every_path_matches_the_oracle(nbytes):
    rng = np.random.default_rng(nbytes)
    # each shape reaches one path, told apart by the counters: stats[1] ("rescored" slot) = distances the tensor cores
    # computed, stats[0] = list appends
    for B, N, k, path in [(1, 1000, 10, "simt"), (7, 5000, 100, "simt"), (127, 9000, 10, "simt"),
                          (128, 3000, 10, "simt"), (128, 5000, 10, "wgmma_dense"), (129, 9000, 1, "wgmma_dense"),
                          (1, LIST_N, 10, "list"), (8, LIST_N, 10, "list")]:
        x = rng.integers(0, 256, (N, nbytes), dtype=np.uint8)
        q = rng.integers(0, 256, (B, nbytes), dtype=np.uint8)
        st = _check(x, q, k)
        assert st["queries"] == B
        assert st["rescored"] == {"simt": 0, "wgmma_dense": B * N, "list": B * (N + 65536)}[path], (B, N, path, st)
        assert (st["candidates"] > 0) == (path == "list")


def test_list_path_sub_batches_inside_a_small_workspace_budget():
    """LGPU_WS_BYTES (read once per process, hence the subprocess) bounds the list path's workspace: at 1 MiB a batch
    of 16 runs as sub-batches of 2 queries with a one-query fix-up matrix, and still returns the oracle's rows.  (The
    dense branch and the other search kinds under a small budget: tests/test_gpu_sub_batches.py.)"""
    import os
    import subprocess
    import sys
    code = """
import numpy as np
from lancedb_b200 import _native
from tests.hamming_oracle import flat_search_u8
rng = np.random.default_rng(31)
for x in (rng.integers(0, 256, (70000, 16), dtype=np.uint8),
          np.tile(rng.integers(0, 256, (1, 16), dtype=np.uint8), (70000, 1))):   # all rows tie: every list overflows
    q = np.concatenate([x[:3], rng.integers(0, 256, (13, 16), dtype=np.uint8)])
    rid = rng.permutation(70000).astype(np.uint64) * 2 + 1
    bx = _native.GpuBinary(x, row_ids=rid)
    _native.set_profiling(True)
    gi, gd, gc = bx.search(q, k=10)
    st = _native.last_filter_stats()
    _native.set_profiling(False)
    oi, od, oc = flat_search_u8(x, q, 10, row_ids=rid)
    assert np.array_equal(gi, oi) and np.array_equal(gc, oc) and np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    assert st["queries"] == 16 and st["candidates"] > 0, st
    for _ in range(2):                                     # graph capture + replay of the sub-batched sequence
        assert np.array_equal(bx.search(q, k=10)[0], oi)
    bx.close()
print("ok", st["flagged_queries"])
"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, LGPU_WS_BYTES=str(1 << 20), PYTHONPATH=root)
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.split()[-1] == "16"                   # the all-equal rows sent every query to the fix-up


def test_large_batches_and_k():
    rng = np.random.default_rng(5)
    x = rng.integers(0, 256, (LIST_N, 8), dtype=np.uint8)
    st = _check(x, rng.integers(0, 256, (1024, 8), dtype=np.uint8), 10)
    assert st["candidates"] > 0 and st["queries"] == 1024
    for k in (100, 2048):
        _check(x, rng.integers(0, 256, (16, 8), dtype=np.uint8), k)
    _check(x[:5000], rng.integers(0, 256, (1024, 8), dtype=np.uint8), 2048)


@pytest.mark.parametrize("kind", ["all_equal", "16_patterns", "i_times_128"])
def test_tie_heavy_data_overflows_into_the_fixup(kind):
    rng = np.random.default_rng(11)
    nb = 128 if kind == "i_times_128" else 32
    if kind == "all_equal":
        x = np.tile(rng.integers(0, 256, (1, nb), dtype=np.uint8), (LIST_N, 1))
    elif kind == "16_patterns":
        x = rng.integers(0, 256, (16, nb), dtype=np.uint8)[rng.integers(0, 16, LIST_N)]
    else:                                        # python/python/tests/test_index.py:67-84: rows [i]*128
        x = np.repeat((np.arange(LIST_N) % 256).astype(np.uint8)[:, None], nb, axis=1)
    row_ids = rng.permutation(LIST_N).astype(np.uint64) * 3 + 7      # neither storage order nor dense
    q = np.concatenate([x[:4], rng.integers(0, 256, (12, nb), dtype=np.uint8)])
    st = _check(x, q, 10, row_ids=row_ids)
    assert st["flagged_queries"] > 0, st
    if kind == "i_times_128":                    # nearest_to([v]*128) -> a row holding v
        bx = _native.GpuBinary(x[:256])
        ids, dist, _ = bx.search(np.full((1, nb), 77, np.uint8), k=1)
        assert ids[0, 0] == 77 and dist[0, 0] == 0
        bx.close()


def test_row_ids_prefilter_range_and_short_results():
    rng = np.random.default_rng(12)
    for N, B in [(3000, 4), (20000, 16), (LIST_N, 9)]:
        x = rng.integers(0, 256, (N, 16), dtype=np.uint8)
        q = rng.integers(0, 256, (B, 16), dtype=np.uint8)
        rid = rng.permutation(N).astype(np.uint64) * 2
        _check(x, q, 10, row_ids=rid)
        bm = _native.mask_bitmap(rng.random(2 * N) < 0.1)
        _check(x, q, 10, row_ids=rid, allow=bm, allow_bits=2 * N)
        _check(x, q, 10, lower=50.0, upper=60.0)
        _check(x, q, 50, lower=0.0, upper=40.0)
    x = rng.integers(0, 256, (5, 4), dtype=np.uint8)
    st = _check(x, rng.integers(0, 256, (9, 4), dtype=np.uint8), 10)            # k > N
    bx = _native.GpuBinary(np.zeros((0, 4), np.uint8))                            # N = 0
    ids, dist, cnt = bx.search(np.zeros((3, 4), np.uint8), k=5)
    assert (cnt == 0).all() and (ids == np.iinfo(np.uint64).max).all() and np.isinf(dist).all()
    ids, dist, cnt = bx.search(np.zeros((0, 4), np.uint8), k=5)                  # B = 0
    assert ids.shape == (0, 5)
    bx.close()


@pytest.mark.parametrize("N", [3000, 20000, LIST_N])
def test_device_entry_point_and_graph_replay_match_the_host_call(N):
    import torch
    rng = np.random.default_rng(N)
    x = rng.integers(0, 256, (N, 24), dtype=np.uint8)
    q = rng.integers(0, 256, (32, 24), dtype=np.uint8)
    bx = _native.GpuBinary(x)
    want = flat_search_u8(x, q, 10)
    for _ in range(3):                          # warm-up, capture, replay
        _same(bx.search(q, k=10), want)
    dq = torch.from_numpy(q).cuda()
    oi = torch.empty(32, 10, dtype=torch.int64, device="cuda"); od = torch.empty(32, 10, device="cuda")
    oc = torch.empty(32, dtype=torch.int32, device="cuda")
    for _ in range(2):
        bx.search_device(dq.data_ptr(), 32, _native.make_params(k=10, nprobes=0), oi.data_ptr(), od.data_ptr(),
                         oc.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        _same((oi.cpu().numpy().view(np.uint64), od.cpu().numpy(), oc.cpu().numpy().view(np.uint32)), want)
    bx.close()


def _table(rng, n=5000, nbytes=32):
    x = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    data = [{"id": i, "grp": i % 5, "vector": x[i]} for i in range(n)]
    import pyarrow as pa
    schema = pa.schema([pa.field("id", pa.int64()), pa.field("grp", pa.int64()),
                        pa.field("vector", pa.list_(pa.uint8(), nbytes))])
    return lancedb.connect("memory://").create_table("bin", data, schema=schema), x


def test_python_surface_returns_the_oracle_rows():
    rng = np.random.default_rng(21)
    t, x = _table(rng)
    q = rng.integers(0, 256, (3, 32), dtype=np.uint8)
    out = t.search(q[0]).distance_type("hamming").limit(7).with_row_id(True).to_arrow()
    oi, od, _ = flat_search_u8(x, q[:1], 7)
    assert out["_rowid"].to_pylist() == oi[0].tolist() and out["id"].to_pylist() == oi[0].tolist()
    assert np.array_equal(out["_distance"].to_numpy(), od[0])
    assert t.search(q[0]).limit(7).to_arrow().equals(t.search(q[0]).distance_type("hamming").limit(7).to_arrow())
    # prefilter, postfilter, offset, select, multi-vector
    mask = np.arange(5000) % 5 == 2
    pre = t.search(q[1]).where("grp = 2").limit(5).offset(2).select(["id"]).to_arrow()
    oi, od, _ = flat_search_u8(x, q[1:2], 7, allow=mask)
    assert pre["id"].to_pylist() == oi[0, 2:].tolist() and pre.column_names == ["id", "_distance"]
    post = t.search(q[1]).where("grp = 2", prefilter=False).limit(20).to_arrow()
    assert all(g == 2 for g in post["grp"].to_pylist()) and post.num_rows < 20
    multi = t.search(q).limit(4).to_arrow()
    oi, _, _ = flat_search_u8(x, q, 4)
    assert multi["id"].to_pylist() == oi.reshape(-1).tolist() and multi["query_index"].to_pylist() == [0] * 4 + [1] * 4 + [2] * 4
    # distance_range on the integer distances
    rng_out = t.search(q[2]).distance_range(100.0, 120.0).limit(50).to_arrow()
    oi, _, oc = flat_search_u8(x, q[2:3], 50, lower=100.0, upper=120.0)
    assert rng_out["id"].to_pylist() == oi[0, :oc[0]].tolist()


def test_async_and_remote_surfaces_return_the_oracle_rows():
    from lancedb_b200 import aio, remote
    rng = np.random.default_rng(22)
    t, x = _table(rng, n=3000, nbytes=16)
    q = rng.integers(0, 256, 16, dtype=np.uint8)
    oi, od, _ = flat_search_u8(x, q[None], 6)

    async def main():
        at = aio.AsyncTable(t)
        return await at.query().nearest_to(q).distance_type("hamming").limit(6).to_arrow()
    out = asyncio.run(main())
    assert out["id"].to_pylist() == oi[0].tolist() and np.array_equal(out["_distance"].to_numpy(), od[0])
    body = remote.build_query_body(q, k=6, distance_type="hamming", columns=["id"])
    assert json.loads(json.dumps(body))["distance_type"] == "hamming"
    out = remote.read_ipc_file(remote.handle_query(t, json.dumps(body)))
    assert out["id"].to_pylist() == oi[0].tolist() and np.array_equal(out["_distance"].to_numpy(), od[0])

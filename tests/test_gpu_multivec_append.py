"""Multivector columns that change: lgpu_multivec_append[_f16] and the MaxSim tensor-core route under a row filter.

Every case compares ids, counts and distance bits with the C oracle (tests/multivec_oracle.c).  Appends: sequences of
appends against a fresh open of the concatenated column, f32 and fp16, rows in HBM and in pinned host memory
(LGPU_MULTIVEC_HBM_BYTES=0), explicit ids and positions, empty rows, every entry point; a column that crosses 65536
vectors by appends takes the tensor-core route, and an appended zero or NaN vector sends it back to the exact route;
refused appends change nothing.  The tensor-core route under prefilters of 1 %, 30 % and 99 %, deleted rows, both, a
duplicate row whose allowed copy wins, fewer than k allowed rows and an overflowing filtered shortlist, with HBM and
host handles reporting equal counters; the adversarial band data under a filter; and Table.add / delete / optimize."""
import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests.multivec_oracle import flat_search_mv, offsets_of
from tests.util import assert_same

pytestmark = pytest.mark.gpu
VAR = "LGPU_MULTIVEC_HBM_BYTES"
F32 = np.float32


def _open(x, off, host, monkeypatch, **kw):
    if host:
        monkeypatch.setenv(VAR, "0")
    else:
        monkeypatch.delenv(VAR, raising=False)
    h = _native.GpuMultivec(x, off, **kw)
    monkeypatch.delenv(VAR, raising=False)
    assert h.rows_on_host == host
    return h


def _stats(fn):
    _native.set_profiling(True)
    try:
        return fn(), _native.last_filter_stats()
    finally:
        _native.set_profiling(False)


def _latent(rng, n, dim, dtype=F32):
    A = rng.standard_normal((8, dim)).astype(F32)
    return (rng.standard_normal((n, 8)).astype(F32) @ A + 0.3 * rng.standard_normal((n, dim))).astype(dtype)


def _device_search(h, q, qoff, k):
    import torch
    B = len(qoff) - 1
    dq = torch.from_numpy(np.ascontiguousarray(q, F32)).cuda()
    di = torch.empty((B, k), dtype=torch.int64, device="cuda")
    dd = torch.empty((B, k), dtype=torch.float32, device="cuda")
    dc = torch.empty(B, dtype=torch.int32, device="cuda")
    h.search_device(dq.data_ptr(), qoff, _native.make_params(k), di.data_ptr(), dd.data_ptr(), dc.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)


def _pieces(off, cuts):
    """(offsets of rows [a, b), vector range) for consecutive row ranges"""
    for a, b in zip(cuts[:-1], cuts[1:]):
        yield (off[a:b + 1] - off[a]).astype(np.uint64), slice(int(off[a]), int(off[b])), a, b


@pytest.mark.parametrize("ids", [False, True], ids=["positions", "row-ids"])
@pytest.mark.parametrize("host", [False, True], ids=["hbm", "host"])
@pytest.mark.parametrize("dtype", [F32, np.float16], ids=["f32", "f16"])
def test_appends_equal_a_fresh_open_of_the_whole_column(dtype, host, ids, monkeypatch):
    rng = np.random.default_rng(3 + host + 2 * ids)
    n, dim = 9000, 24
    lens = rng.integers(0, 9, n)
    lens[[0, 4000, 4001, 8999]] = 0                              # rows with no vectors, some at a piece's edge
    off = offsets_of(lens)
    x = _latent(rng, int(off[-1]), dim, dtype)
    rid = (rng.permutation(3 * n)[:n] + 7).astype(np.uint64) if ids else None
    cuts = [0, 2500, 2500, 2501, 4001, 9000]                     # (an empty append and a one-row append included)
    first = next(_pieces(off, cuts))
    h = _open(x[first[1]], first[0], host, monkeypatch, row_ids=None if rid is None else rid[:2500])
    for o, sl, a, b in list(_pieces(off, cuts))[1:]:
        h.append(x[sl], o, row_ids=None if rid is None else rid[a:b])
    assert h.nrows == n
    fresh = _open(x, off, host, monkeypatch, row_ids=rid)
    qoff = offsets_of(rng.integers(1, 12, 9))
    q = _latent(rng, int(qoff[-1]), dim)
    xf = x.astype(F32)
    for k in (10, 700):
        want = flat_search_mv(xf, off, q, qoff, k, row_ids=rid, nthreads=16)
        assert_same(h.search(q, k=k, q_offsets=qoff), want, ("host entry", k))
        assert_same(fresh.search(q, k=k, q_offsets=qoff), want, ("fresh open", k))
        assert_same(_device_search(h, q, qoff, k), want, ("device entry", k))
    top = int((rid if ids else np.arange(n)).max()) + 1
    allow = rng.random(top) < 0.4
    want = flat_search_mv(xf, off, q, qoff, 25, row_ids=rid, allow=allow, nthreads=16)
    got = h.search(q, k=25, q_offsets=qoff, allow=_native.mask_bitmap(allow), allow_bits=top)
    assert_same(got, want, "filtered entry")
    assert h.device_bytes > 0 and (h.host_bytes() > 0) == host
    h.close(); fresh.close()


@pytest.mark.parametrize("host", [False, True], ids=["hbm", "host"])
@pytest.mark.parametrize("dtype", [F32, np.float16], ids=["f32", "f16"])
def test_crossing_65536_vectors_by_appends_switches_to_the_tensor_core_route(dtype, host, monkeypatch):
    rng = np.random.default_rng(11 + host)
    dim = 32
    lens = rng.integers(1, 8, 20_000)
    off = offsets_of(lens)
    x = _latent(rng, int(off[-1]), dim, dtype)
    assert int(off[-1]) > 65536
    cut = int(np.searchsorted(off, 60_000))                      # the first piece holds fewer than 65536 vectors
    h = _open(x[:int(off[cut])], off[:cut + 1], host, monkeypatch)
    qoff = offsets_of(rng.integers(1, 17, 6))
    q = _latent(rng, int(qoff[-1]), dim)
    got, st = _stats(lambda: h.search(q, k=20, q_offsets=qoff))
    assert_same(got, flat_search_mv(x[:int(off[cut])].astype(F32), off[:cut + 1], q, qoff, 20, nthreads=16))
    assert st["rescored"] == 6 * cut                             # the exact route
    h.append(x[int(off[cut]):], (off[cut:] - off[cut]).astype(np.uint64))
    N = lens.size
    got, st = _stats(lambda: h.search(q, k=20, q_offsets=qoff))
    assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 20, nthreads=16), "after crossing")
    assert st["rescored"] < 6 * N                                # the tensor-core route: a shortlist
    # an appended zero vector, then a NaN one, send the column back to the exact route (as an open would)
    for bad in ("zero", "nan"):
        v = _latent(rng, 3, dim, dtype)
        v[1] = 0 if bad == "zero" else np.nan
        h.append(v, np.asarray([0, 3], np.uint64))
        x = np.concatenate([x, v]); off = np.concatenate([off, [off[-1] + 3]]).astype(np.uint64); N += 1
        got, st = _stats(lambda: h.search(q, k=20, q_offsets=qoff))
        assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 20, nthreads=16), bad)
        assert st["rescored"] == 6 * N, bad
    h.close()


@pytest.mark.parametrize("host", [False, True], ids=["hbm", "host"])
@pytest.mark.parametrize("dtype", [F32, np.float16], ids=["f32", "f16"])
def test_appends_to_a_tensor_core_column_keep_the_tensor_core_route(dtype, host, monkeypatch):
    """Appends to a column already past 65536 vectors take the operand, the row of each vector and |v| of the new
    vectors only: a few rows, rows with no vectors, then about 280 000 vectors at d 256, which a host handle stages in
    more than one 128 MiB chunk.  On every entry point the tensor-core route returns the oracle's bits, and a fresh open
    of the whole column (the same operand) reports the same counters."""
    rng = np.random.default_rng(51 + host)
    dim, n = 256, 90_000
    lens = rng.integers(1, 8, n)
    lens[20_010:20_015] = 0                                      # an append of rows with no vectors
    off = offsets_of(lens)
    x = _latent(rng, int(off[-1]), dim, dtype)
    cuts = [0, 20_000, 20_010, 20_015, n]
    assert int(off[20_000]) > 65536 and int(off[n] - off[20_015]) * dim * x.itemsize > 128 << 20
    pieces = list(_pieces(off, cuts))
    h = _open(x[pieces[0][1]], pieces[0][0], host, monkeypatch)
    for o, sl, _, _ in pieces[1:]:
        h.append(x[sl], o)
    fresh = _open(x, off, host, monkeypatch)
    qoff = offsets_of(rng.integers(1, 17, 6))
    q = _latent(rng, int(qoff[-1]), dim)
    xf = x.astype(F32)
    allow = rng.random(n) < 0.5
    for k in (10, 200):
        want = flat_search_mv(xf, off, q, qoff, k, nthreads=16)
        got, st = _stats(lambda: h.search(q, k=k, q_offsets=qoff))
        assert_same(got, want, ("host entry", k))
        _, sf = _stats(lambda: fresh.search(q, k=k, q_offsets=qoff))
        assert st == sf and st["rescored"] < 6 * n, (k, st, sf)
        assert_same(_device_search(h, q, qoff, k), want, ("device entry", k))
        kw = dict(allow=_native.mask_bitmap(allow), allow_bits=n)
        got, st = _stats(lambda: h.search(q, k=k, q_offsets=qoff, **kw))
        assert_same(got, flat_search_mv(xf, off, q, qoff, k, allow=allow, nthreads=16), ("filtered entry", k))
        _, sf = _stats(lambda: fresh.search(q, k=k, q_offsets=qoff, **kw))
        assert st == sf and st["rescored"] < 6 * n, (k, st, sf)
    h.close(); fresh.close()


def test_refused_appends_change_nothing(monkeypatch):
    rng = np.random.default_rng(5)
    lib = _native.load()
    off = offsets_of(rng.integers(0, 6, 2000))
    x = _latent(rng, int(off[-1]), 16)
    for dtype in (F32, np.float16):
        h = _open(x.astype(dtype), off, False, monkeypatch, row_ids=np.arange(2000, dtype=np.uint64))
        q = _latent(rng, 5, 16)
        assert h.delete(np.asarray([3, 9], np.uint64)) == 2
        before = h.search(q, k=30)
        v = _latent(rng, 4, 16)
        o = np.asarray([0, 4], np.uint64)
        other = "lgpu_multivec_append" if dtype == np.float16 else "lgpu_multivec_append_f16"
        w = v.astype(F32 if dtype == np.float16 else np.float16)
        assert getattr(lib, other)(h._h, w.ctypes.data, o.ctypes.data, 1, None) == _native.LGPU_INVALID_INPUT
        with pytest.raises(ValueError, match="needs values of that type"):
            h.append(w, o)
        with pytest.raises(ValueError, match="deleted"):                # the id of a deleted row
            h.append(v.astype(dtype), o, row_ids=np.asarray([9], np.uint64))
        with pytest.raises(ValueError, match="dimension"):
            h.append(_latent(rng, 4, 17, dtype), o)
        own = "lgpu_multivec_append_f16" if dtype == np.float16 else "lgpu_multivec_append"
        long_row = np.asarray([0, (1 << 20) + 1], np.uint64)
        vv = v.astype(dtype)
        assert getattr(lib, own)(h._h, vv.ctypes.data, long_row.ctypes.data, 1, None) == _native.LGPU_INVALID_INPUT
        assert getattr(lib, own)(h._h, vv.ctypes.data, o.ctypes.data, 0, None) == _native.LGPU_OK    # n = 0
        assert h.nrows == 2000
        assert_same(h.search(q, k=30), before, dtype)
        h.append(vv, o, row_ids=np.asarray([5000], np.uint64))        # the handle still takes a good append
        live = np.ones(5001, bool); live[[3, 9]] = False; live[2000:5000] = False
        xx, oo = np.concatenate([x, vv.astype(F32)]), np.concatenate([off, [off[-1] + 4]]).astype(np.uint64)
        rid = np.concatenate([np.arange(2000), [5000]]).astype(np.uint64)
        want = flat_search_mv(xx.astype(dtype).astype(F32), oo, q, [0, 5], 30, row_ids=rid, allow=live)
        assert_same(h.search(q, k=30), want, (dtype, "after a good append"))
        h.close()


# the tensor-core column of the filter cases: 20 000 rows of 1..7 vectors at dim 32, row N // 2 a copy of row 3
@pytest.fixture(scope="module", params=[F32, np.float16], ids=["f32", "f16"])
def tc_column(request):
    dtype = request.param
    rng = np.random.default_rng(17)
    n = 20_000
    lens = rng.integers(1, 8, n)
    lens[n // 2] = lens[3]
    off = offsets_of(lens)
    x = _latent(rng, int(off[-1]), 32, dtype)
    x[off[n // 2]:off[n // 2 + 1]] = x[off[3]:off[4]]
    mp = pytest.MonkeyPatch()
    hbm, host = _open(x, off, False, mp), _open(x, off, True, mp)
    mp.undo()
    yield x, off, hbm, host, rng
    hbm.close(); host.close()


def _both(hbm, host, q, qoff, k, allow, what):
    """the HBM and host handles' results and counters agree; returns the result and the counters"""
    kw = {} if allow is None else dict(allow=_native.mask_bitmap(allow), allow_bits=allow.size)
    a, sa = _stats(lambda: hbm.search(q, k=k, q_offsets=qoff, **kw))
    b, sb = _stats(lambda: host.search(q, k=k, q_offsets=qoff, **kw))
    assert_same(b, a, f"{what}: host against HBM")
    assert sa == sb, (what, sa, sb)
    return a, sa


def test_tensor_core_route_under_prefilters_and_deletes(tc_column):
    x, off, hbm, host, rng = tc_column
    N = off.size - 1
    xf = x.astype(F32)
    qoff = offsets_of([int(off[4] - off[3])] + list(rng.integers(1, 17, 7)))
    q = _latent(rng, int(qoff[-1]), 32)
    q[:int(qoff[1])] = xf[off[3]:off[4]]                        # query 0: the duplicated row's vectors
    for share in (0.01, 0.3, 0.99):
        allow = rng.random(N) < share
        allow[3], allow[N // 2] = False, True                    # the allowed copy of the duplicate must win
        got, st = _both(hbm, host, q, qoff, 10, allow, share)
        assert_same(got, flat_search_mv(xf, off, q, qoff, 10, allow=allow, nthreads=16), share)
        assert st["rescored"] < 8 * N and st["candidates"] <= 8 * int(allow.sum()), (share, st)
        assert N // 2 in got[0][0] and 3 not in got[0][0]
    allow = rng.random(N) < 0.3
    allow[3] = allow[N // 2] = True                              # both copies: the tie goes to the lower id
    got, _ = _both(hbm, host, q, qoff, 10, allow, "both copies")
    assert_same(got, flat_search_mv(xf, off, q, qoff, 10, allow=allow, nthreads=16), "both copies")
    few = np.zeros(N, bool)
    few[rng.choice(N, 20, replace=False)] = True                 # fewer than k allowed rows: tau is +inf
    got, st = _both(hbm, host, q, qoff, 50, few, "fewer than k")
    assert_same(got, flat_search_mv(xf, off, q, qoff, 50, allow=few, nthreads=16), "fewer than k")
    assert list(got[2]) == [20] * 8 and st["candidates"] == 8 * 20 and st["flagged_queries"] == 0
    # deleted rows, alone and under a prefilter (the handles are the module's: delete on copies of them)
    mp = pytest.MonkeyPatch()
    h2, host2 = _open(x, off, False, mp), _open(x, off, True, mp)
    mp.undo()
    gone = rng.choice(N, N // 10, replace=False).astype(np.uint64)
    assert h2.delete(gone) == gone.size and host2.delete(gone) == gone.size
    live = np.ones(N, bool); live[gone.astype(np.int64)] = False
    got, st = _both(h2, host2, q, qoff, 10, None, "deleted")
    assert_same(got, flat_search_mv(xf, off, q, qoff, 10, allow=live, nthreads=16), "deleted")
    assert st["rescored"] < 8 * N
    allow = rng.random(N) < 0.3
    got, st = _both(h2, host2, q, qoff, 10, allow, "deleted and prefilter")
    assert_same(got, flat_search_mv(xf, off, q, qoff, 10, allow=allow & live, nthreads=16), "deleted and prefilter")
    assert st["rescored"] < 8 * N
    h2.close(); host2.close()


@pytest.mark.parametrize("dtype", [F32, np.float16], ids=["f32", "f16"])
def test_a_filtered_shortlist_that_overflows_takes_the_filtered_fix_up(dtype, monkeypatch):
    """Near-duplicate rows: every allowed row lies in the band, every list overflows, and the fix-up (the exact route)
    must leave the filtered rows out as well."""
    rng = np.random.default_rng(22)
    v = rng.standard_normal((1, 16)).astype(F32)
    off = offsets_of(np.full(70_000, 1))
    x = np.repeat(v, 70_000, axis=0)
    x[::7] += F32(1e-7)
    x = x.astype(dtype)
    hbm, host = _open(x, off, False, monkeypatch), _open(x, off, True, monkeypatch)
    q = rng.standard_normal((5, 16)).astype(F32)
    qoff = offsets_of([2, 3])
    allow = rng.random(70_000) < 0.3
    got, st = _both(hbm, host, q, qoff, 40, allow, "overflow")
    assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, 40, allow=allow, nthreads=16))
    assert st["flagged_queries"] == 2 and st["candidates"] > 2 * 1024
    hbm.close(); host.close()


@pytest.mark.parametrize("dtype", [F32, np.float16], ids=["f32", "f16"])
def test_adversarial_band_data_under_a_filter(dtype, monkeypatch):
    """The midpoint data behind mv_band / mv_band_f16 (copies of the query vectors, where the fp16 errors add up, among
    midpoint decoys), padded past 65536 vectors with far rows, some of the copies and decoys deleted."""
    from tests.test_multivec_host import _unit_at_midpoints
    rng = np.random.default_rng(40)
    d = 64
    q = np.stack([_unit_at_midpoints(rng, d, up) for up in (True, False, True, True, False, True)])
    if dtype == np.float16:
        from tests.test_multivec_f16_host import adversarial_f16_column
        xa, offa = adversarial_f16_column(rng, q)
    else:
        base = np.stack([_unit_at_midpoints(rng, d, True) for _ in range(40)])
        xa = np.concatenate([q, base, q[::-1], q + F32(2.0 ** -12)]).astype(F32)
        offa = offsets_of([1] * 6 + [2] * 20 + [1] * 12)
    far = (-np.repeat(q, 11_000, axis=0) + 0.05 * rng.standard_normal((66_000, d))).astype(dtype)
    x = np.concatenate([xa.astype(dtype), far])
    off = np.concatenate([offa, offa[-1] + np.arange(1, 66_001, dtype=np.uint64)]).astype(np.uint64)
    Na, N = offa.size - 1, off.size - 1
    hbm, host = _open(x, off, False, monkeypatch), _open(x, off, True, monkeypatch)
    gone = np.arange(1, Na, 3, dtype=np.uint64)                  # a third of the copies and decoys
    assert hbm.delete(gone) == gone.size and host.delete(gone) == gone.size
    live = np.ones(N, bool); live[gone.astype(np.int64)] = False
    qoff = offsets_of([1, 2, 3])
    for k in (1, 3, 10):
        got, st = _both(hbm, host, q, qoff, k, None, ("adversarial", k))
        assert_same(got, flat_search_mv(x.astype(F32), off, q, qoff, k, allow=live, nthreads=16), ("adversarial", k))
        assert st["rescored"] < 3 * N
    hbm.close(); host.close()


def _in(ids):
    return "id IN (" + ", ".join(str(i) for i in ids) + ")"


@pytest.mark.parametrize("vt", [pa.float32(), pa.float16()])
def test_table_add_delete_optimize_grow_the_open_cache(vt):
    rng = np.random.default_rng(31)
    dim = 16

    def rows(n):
        return [rng.standard_normal((int(m), dim)).astype(np.float32).tolist() for m in rng.integers(0, 6, n)]

    def table(name, data):
        return lancedb.connect().create_table(name, pa.table({
            "id": pa.array(np.arange(len(data))), "vector": pa.array(data, type=pa.list_(pa.list_(vt, dim)))}))

    def top(t, q):
        r = t.search(q).limit(15).with_row_id(True).to_arrow()
        return r["_rowid"].to_pylist(), r["_distance"].to_numpy().view(np.uint32).tolist()

    def add(t, data, start):
        t.add(pa.table({"id": pa.array(np.arange(start, start + len(data))),
                        "vector": pa.array(data, type=pa.list_(pa.list_(vt, dim)))}))

    a, b, c = rows(3000), rows(400), rows(300)
    q = rng.standard_normal((3, dim)).astype(np.float32).tolist()
    t = table("t", a)
    top(t, q)                                                    # opens the cache
    cache = t._multivec["vector"]
    add(t, b, 3000)
    assert t._multivec["vector"] is cache and cache.nrows == 3400     # grown in place, not reopened
    assert top(t, q) == top(table("all", a + b), q)
    t.delete(_in(range(0, 3400, 7)))
    add(t, c, 3400)                                              # add after delete: the cache holds explicit ids
    assert t._multivec["vector"] is cache
    ref = table("ref", a + b + c)
    ref.delete(_in(range(0, 3400, 7)))
    assert top(t, q) == top(ref, q)
    t.delete(_in(range(1, 3700, 5)))                             # delete after add
    ref.delete(_in(range(1, 3700, 5)))
    assert top(t, q) == top(ref, q)
    t.optimize()
    assert top(t, q) == top(ref, q)

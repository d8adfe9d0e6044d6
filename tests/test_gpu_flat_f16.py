"""Float16 flat handles on the H100 (lgpu_flat_open_f16): an fp16 handle opened on rows x16 returns exactly what an f32
handle opened on x16.astype(float32) returns -- ids, counts and distance bits -- and both match the C oracle on the
upcast rows.  Covered: the exact path (N < 4096, or B < 8), the dense tensor-core path (4096 <= N < 262144, B >= 8)
and the sampled-threshold path (N >= 262144), each with k from 1 to above N, distance_range, a prefilter and deleted
rows; adversarial queries for the fp16 band (rounding midpoints, subnormal and near-65504 components, ties, duplicated
rows, cancellation, queries beyond fp16's range); whether the fp16 MMA consumes subnormal fp16 operands exactly;
appends across both thresholds; an fp16 tail of an unindexed union; inf / NaN rows; sub-batches under a small
LGPU_WS_BYTES; the handle's device bytes; and float16 tables end to end."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import oracle
import lancedb_b200 as lancedb
from lancedb_b200 import _native
from tests.util import assert_same, random_index

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, F32 = np.float16, np.float32

# (N, dim, B, path): every path of flat_search_device for l2
SHAPES = [(3000, 64, 16, "exact"), (20000, 64, 4, "exact"), (20000, 64, 16, "dense"), (300000, 64, 16, "sampled")]
KS = [1, 10, 100, 2048, 2049, 65536]


def _rows(rng, n, d, scale=1.0):
    return (rng.standard_normal((n, d)) * scale).astype(F16)


def _pair(x16, row_ids=None):
    return _native.GpuFlat(x16, row_ids=row_ids), _native.GpuFlat(x16.astype(F32), row_ids=row_ids)


@pytest.fixture(scope="module", params=SHAPES, ids=[s[3] + f"-{s[0]}x{s[2]}" for s in SHAPES])
def shape(request):
    N, d, B, path = request.param
    rng = np.random.default_rng(N + B)
    x16 = _rows(rng, N, d)
    q = rng.standard_normal((B, d)).astype(F32)
    h16, h32 = _pair(x16)
    yield N, d, B, path, x16, q, h16, h32
    h16.close(); h32.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_parity_on_every_path(shape, metric):
    N, d, B, path, x16, q, h16, h32 = shape
    x32 = x16.astype(F32)
    rng = np.random.default_rng(1)
    mask = rng.random(N) < 0.7
    for k in KS:
        kw = dict(k=k, metric=metric)
        _native.set_profiling(True)
        got = h16.search(q, **kw)
        st = _native.last_filter_stats()
        _native.set_profiling(False)
        assert_same(got, h32.search(q, **kw), (metric, k))
        tc = metric == "l2" and path != "exact" and k <= 2048
        assert st["rescored"] == (B * N if tc else 0), (path, metric, k, st)   # [1]: tensor-core distances
        if k in (10, 2049) or (k == 65536 and N <= 20000):
            assert_same(got, oracle.flat_search(x32, q, k=k, metric=metric, nthreads=16), ("oracle", metric, k))
    lo, hi = (0.5, 1.5) if metric != "l2" else (float(d) * 1.5, float(d) * 2.5)
    for k in (10, 2049):
        kw = dict(k=k, metric=metric, lower=lo, upper=hi)
        got = h16.search(q, **kw)
        assert_same(got, h32.search(q, **kw), ("range", metric, k))
        assert_same(got, oracle.flat_search(x32, q, k=k, metric=metric, lower=lo, upper=hi, nthreads=16),
                    ("range oracle", k))
        kw = dict(k=k, metric=metric, allow=_native.mask_bitmap(mask), allow_bits=N)
        got = h16.search(q, **kw)
        assert_same(got, h32.search(q, **kw), ("prefilter", metric, k))
        assert_same(got, oracle.flat_search(x32, q, k=k, metric=metric, allow=mask, nthreads=16),
                    ("prefilter oracle", k))


def test_deleted_rows_on_every_path(shape):
    N, d, B, path, x16, q, _, _ = shape
    h16, h32 = _pair(x16)
    gone = np.random.default_rng(2).choice(N, N // 50, replace=False).astype(np.uint64)
    assert h16.delete(gone) == h32.delete(gone) == gone.size
    live = np.ones(N, bool)
    live[gone.astype(np.int64)] = False
    for metric in ("l2", "cosine"):
        for k in (10, 2049):
            got = h16.search(q, k=k, metric=metric)
            assert_same(got, h32.search(q, k=k, metric=metric), ("deleted", metric, k))
            assert_same(got, oracle.flat_search(x16.astype(F32), q, k=k, metric=metric, allow=live, nthreads=16),
                        "oracle")
    h16.close(); h32.close()


def _midpoint_queries(rng, x16, B):
    """queries whose every component sits one f32 ulp beside an fp16 rounding midpoint near a stored row"""
    base = x16[rng.integers(0, x16.shape[0], B)]
    a = np.abs(base)
    a[a == 0] = F16(2.0 ** -24)
    with np.errstate(over="ignore"):
        nxt = np.nextafter(a, F16(np.inf))
    nxt = np.where(np.isinf(nxt), a, nxt)                  # 65504: the query stays next to it, inside fp16's range
    mid = ((a.astype(np.float64) + nxt.astype(np.float64)) / 2).astype(F32)
    side = np.where(rng.random(base.shape) < 0.5, F32(0), F32(np.inf))
    return (np.sign(base.astype(F32) + F32(1e-30)) * np.nextafter(mid, side)).astype(F32)


@pytest.mark.parametrize("N", [20000, 300000])
def test_band_on_adversarial_queries(N):
    rng = np.random.default_rng(N)
    d = 64
    x16 = _rows(rng, N, d)
    x16[: N // 4] *= F16(2.0 ** -16)                         # subnormal fp16 rows
    x16[N // 4: N // 2] = (x16[N // 4: N // 2].astype(F32) * 3e4).clip(-65504, 65504).astype(F16)   # near 65504
    x16[N // 2: N // 2 + 64] = x16[N // 2 + 64: N // 2 + 128]                                       # duplicated rows
    q = np.concatenate([
        _midpoint_queries(rng, x16[: N // 4], 8),
        _midpoint_queries(rng, x16[N // 4: N // 2], 8),
        x16[N // 2 + 64: N // 2 + 72].astype(F32),          # ties: each query equals two stored rows
        x16[N // 2: N // 2 + 8].astype(F32) + F32(2.0 ** -14),                          # cancellation
    ])
    q_over = q[:8].copy()
    q_over[:, 5] = 70000.0                                  # beyond fp16: these queries take the exact path
    q = np.concatenate([q, q_over])
    h16, h32 = _pair(x16)
    for k in (1, 10, 100):
        got = h16.search(q, k=k)
        assert_same(got, h32.search(q, k=k), ("band", k))
        assert_same(got, oracle.flat_search(x16.astype(F32), q, k=k, nthreads=16), ("band oracle", k))
    h16.close(); h32.close()


def test_fp16_mma_consumes_subnormal_operands_exactly():
    """The fp16 wgmma (the instruction F16Dist shares with F16MaxSim, read here through lgpu_debug_maxsim_gemm) returns
    normal x subnormal products exactly: the stored rows' h(x) = x, so xerr = 0 is a bound, not an assumption."""
    d = 8
    sub = np.array([2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -20, 1023 * 2.0 ** -24], np.float64)   # fp16 subnormals
    vals = np.zeros((sub.size, d), F32)
    vals[:, 0] = 1.0
    vals[:, 1] = sub                                        # |v| rounds to 1 in f32: v / |v| keeps the subnormal
    off = np.arange(sub.size + 1, dtype=np.uint64)
    qv = np.zeros((1, d), F32)
    qv[0, 1] = 1.0
    out = np.empty((1, sub.size), F32)
    _native.check(_native.load().lgpu_debug_maxsim_gemm(_native._ptr(qv), 1, _native._ptr(vals), _native._ptr(off),
                                                        sub.size, d, 0, _native._ptr(out)))
    assert np.array_equal(out[0].astype(np.float64), sub), out
    # and a search over subnormal-only rows on the tensor-core path equals the f32 handle and the oracle
    rng = np.random.default_rng(3)
    x16 = (rng.integers(-1023, 1024, (8192, 32)) * 2.0 ** -24).astype(F16)
    q = (rng.standard_normal((16, 32)) * 2.0 ** -12).astype(F32)
    h16, h32 = _pair(x16)
    _native.set_profiling(True)
    got = h16.search(q, k=10)
    st = _native.last_filter_stats()
    _native.set_profiling(False)
    assert st["rescored"] == 16 * 8192                     # the tensor cores scored every row
    assert_same(got, h32.search(q, k=10), "subnormal rows")
    assert_same(got, oracle.flat_search(x16.astype(F32), q, k=10, nthreads=16), "subnormal rows oracle")
    h16.close(); h32.close()


def test_appends_across_both_thresholds_and_after_deletes():
    rng = np.random.default_rng(5)
    d = 32
    x16 = _rows(rng, 300000, d)
    q = rng.standard_normal((16, d)).astype(F32)
    h = _native.GpuFlat(x16[:3000])
    assert h.dtype == F16
    for n1 in (5000, 100000, 300000):                       # exact -> dense (4096) -> sampled (262144)
        h.append(x16[h.nrows:n1])
        ref = _native.GpuFlat(x16[:n1])
        for metric in ("l2", "cosine"):
            for k in (10, 2049):
                assert_same(h.search(q, k=k, metric=metric), ref.search(q, k=k, metric=metric), (n1, metric, k))
        ref.close()
    h.close()
    h16, h32 = _pair(x16[:200000])
    gone = rng.choice(200000, 3000, replace=False).astype(np.uint64)
    h16.delete(gone); h32.delete(gone)
    h16.append(x16[200000:]); h32.append(x16[200000:].astype(F32))
    for k in (10, 2049):
        assert_same(h16.search(q, k=k), h32.search(q, k=k), ("delete then append", k))
    with pytest.raises(ValueError):
        h16.append(x16[:2].astype(F32))
    with pytest.raises(ValueError):
        h32.append(x16[:2])
    h16.close(); h32.close()


def test_fp16_tail_of_an_unindexed_union():
    rng = np.random.default_rng(6)
    d = 32
    ix = random_index(rng, dim=d, nlist=8, m=8, n=4000, with_vectors=True)
    gi = _native.GpuIvfPq(ix)
    tail16 = _rows(rng, 6000, d)
    ids = np.arange(4000, 10000, dtype=np.uint64)
    t16, t32 = _pair(tail16, row_ids=ids)
    q = rng.standard_normal((16, d)).astype(F32)
    allow = _native.mask_bitmap(rng.random(10000) < 0.8)
    for kw in (dict(k=10), dict(k=2049), dict(k=10, refine_factor=2), dict(k=10, allow=allow, allow_bits=10000)):
        assert_same(gi.search_unindexed(t16, q, nprobes=4, **kw), gi.search_unindexed(t32, q, nprobes=4, **kw),
                    kw.keys())
    t16.close(); t32.close(); gi.close()


def test_non_finite_rows_give_the_f32_handles_results():
    rng = np.random.default_rng(7)
    for N in (3000, 20000):
        x16 = _rows(rng, N, 64)
        x16[5, 3] = F16(np.inf)
        x16[17, 0] = F16(-np.inf)
        x16[29, 9] = F16(np.nan)
        q = rng.standard_normal((16, 64)).astype(F32)
        h16, h32 = _pair(x16)
        for metric in ("l2", "cosine", "dot"):
            for k in (10, 2049):
                assert_same(h16.search(q, k=k, metric=metric), h32.search(q, k=k, metric=metric), (N, metric, k))
        h16.close(); h32.close()


def _sub_batch_child(path):
    """Under LGPU_WS_BYTES = 12 MiB the 256 queries run in sub-batches of 157 (N 20000) and of 10 (N 300000: the
    tensor-core paths, and the exact path for the last 6)"""
    rng = np.random.default_rng(8)
    x16 = _rows(rng, 300000, 64)
    q = rng.standard_normal((256, 64)).astype(F32)
    out = {}
    for N in (20000, 300000):
        h16 = _native.GpuFlat(x16[:N])
        for metric in ("l2", "cosine"):
            for k in (10, 2049):
                i, dd, c = h16.search(q, k=k, metric=metric)
                out[f"{N}-{metric}-{k}-ids"], out[f"{N}-{metric}-{k}-dist"], out[f"{N}-{metric}-{k}-cnt"] = i, dd, c
        h16.close()
    np.savez(path, **out)


def test_sub_batches_under_a_small_workspace_budget(tmp_path):
    res = []
    for budget in (None, 12 << 20):
        env = dict(os.environ, PYTHONPATH=ROOT)
        env.pop("LGPU_WS_BYTES", None)
        if budget:
            env["LGPU_WS_BYTES"] = str(budget)
        path = tmp_path / f"r{budget}.npz"
        r = subprocess.run([sys.executable, "-m", "tests.test_gpu_flat_f16", "sub-batch-child", str(path)], cwd=ROOT,
                           env=env, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0, r.stderr[-4000:]
        res.append(np.load(path))
    a, b = res
    for key in a.files:
        assert np.array_equal(a[key].view(np.uint8), b[key].view(np.uint8)), key


def test_device_bytes_of_a_fresh_handle_after_a_cosine_search():
    rng = np.random.default_rng(9)
    N, d = 100000, 128
    x16 = _rows(rng, N, d)
    ids = np.arange(N, dtype=np.uint64) * 3
    h16, h32 = _pair(x16, row_ids=ids)
    q = rng.standard_normal((4, d)).astype(F32)
    for h in (h16, h32):
        h.search(q, k=10, metric="cosine")                   # allocates the row norms
    b16, b32 = h16.device_bytes, h32.device_bytes
    assert b16 <= 2 * N * d + 16 * N + (1 << 20), b16
    assert b16 < 0.4 * b32, (b16, b32)
    h16.close(); h32.close()


# ---- float16 tables (the reference's test_create_f16_table*, test_query_with_f16), and f16 == f32-cast tables ----
def _f16_table_data(n=512, d=32):
    values = pa.array(np.random.default_rng(42).standard_normal(n * d).astype(F16))
    return pa.table({"text": [f"s-{i}" for i in range(n)], "vector": pa.FixedSizeListArray.from_arrays(values, d)})


def test_create_f16_table_from_arrow_data():
    df = _f16_table_data()
    table = lancedb.connect().create_table("f16_tbl", data=df)
    assert table.schema.field("vector").type == pa.list_(pa.float16(), 32)
    table.create_index(num_partitions=2, num_sub_vectors=2)
    expected = table.search(df["vector"][2].as_py()).limit(2).to_arrow()
    assert "s-2" in expected["text"].to_pylist()


def test_create_f16_table():
    df = _f16_table_data()
    schema = pa.schema([pa.field("text", pa.string()), pa.field("vector", pa.list_(pa.float16(), 32))])
    table = lancedb.connect().create_table("f16_tbl", schema=schema)
    table.add(df)
    table.create_index(num_partitions=2, num_sub_vectors=2)
    expected = table.search(df["vector"][2].as_py()).limit(2).to_arrow()
    assert "s-2" in expected["text"].to_pylist()


def test_query_with_f16():
    import asyncio
    from lancedb_b200 import aio

    async def run():
        db = await aio.connect_async("memory://")
        df = pa.table({"vector": pa.FixedSizeListArray.from_arrays(np.array([1.0, 2.0, 3.0, 4.0], F16), 2),
                       "id": pa.array([1, 2])})
        tbl = await db.create_table("test", df)
        return await tbl.vector_search([np.float16(1), np.float16(2)]).to_pandas()

    assert len(asyncio.run(run())) == 2


def _key(t):
    return t["id"].to_pylist(), np.asarray(t["_distance"].to_numpy(), F32).view(np.uint32).tolist()


def test_float16_table_equals_the_same_table_cast_to_f32():
    rng = np.random.default_rng(10)
    n, d = 6000, 32
    x16 = rng.standard_normal((n, d)).astype(F16)
    tables = []
    for vt in (pa.float16(), pa.float32()):
        data = pa.table({"id": np.arange(n), "vector": pa.FixedSizeListArray.from_arrays(
            pa.array(x16.reshape(-1)).cast(vt), d)})
        tables.append(lancedb.connect().create_table("t", data))
    q = [rng.standard_normal(d).astype(F32) for _ in range(3)]
    extra16 = rng.standard_normal((500, d)).astype(F16)

    def results():
        out = []
        for t in tables:
            r = []
            for qq in q:
                r.append(_key(t.search(qq).limit(20).to_arrow()))
                r.append(_key(t.search(qq).bypass_vector_index().limit(20).to_arrow()))
                r.append(_key(t.search(qq).bypass_vector_index().distance_type("cosine").limit(20).to_arrow()))
            out.append(r)
        return out

    a, b = results()
    assert a == b
    for t in tables:
        t.create_index(num_partitions=4, num_sub_vectors=4)
        vt = t.schema.field("vector").type.value_type
        t.add(pa.table({"id": np.arange(n, n + 500),
                        "vector": pa.FixedSizeListArray.from_arrays(pa.array(extra16.reshape(-1)).cast(vt), d)}))
    a, b = results()                                         # the index and its unindexed tail
    assert a == b
    for t in tables:
        t.delete("id < 100 OR id >= 6400")
    a, b = results()
    assert a == b
    for t in tables:
        t.optimize()
    a, b = results()
    assert a == b


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "sub-batch-child":
    _sub_batch_child(sys.argv[2])

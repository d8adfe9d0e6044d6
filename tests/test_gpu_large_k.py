"""k above 2048: limit + offset and limit x refine_factor up to LGPU_K_MAX = 65536 on every single-GPU search kind.

Above SELECT_KMAX the searches take their exact routes and end in the global-memory radix select (csrc/select_large.cu).
This file checks
  1. the select alone (lgpu_debug_select_large) against the exact restatement in tests/select_oracle.py, in modes 0, 1
     and 2 with every optional field, on adversarial key sets (all equal, two values, NaN, +-inf, -0 / +0, descending
     ids), at k = 2049, 4097 and 65536, bit for bit and with guard bands around every output;
  2. every search kind against its C oracle (ids, counts, distance bits) at k = 2049 and 10000, k > N, refine pools of
     limit 100 x refine_factor 30, prefilter with maximum_nprobes widening, range searches, tie-heavy Hamming rows and
     4-bit codes, NaN / inf rows;
  3. pagination: offset(o).limit(l) pages concatenate to limit(o + l);
  4. the host, filtered, device, async and coalesced entry points agree bit for bit;
  5. a workspace budget (LGPU_WS_BYTES) that cuts a large-k batch into sub-batches gives the unsplit result.  The budget
     is read once per process, so that part runs this module as a child: python -m tests.test_gpu_large_k <out.npz>.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from lancedb_b200 import _native  # noqa: E402
from tests import select_oracle as so  # noqa: E402
from tests.util import assert_same  # noqa: E402

pytestmark = pytest.mark.gpu
NTH = min(16, os.cpu_count() or 1)
U64_MAX = np.iinfo(np.uint64).max
GUARD = 256
FILL = 0xA5
INPUTS = ("dist", "seg_off", "probes", "part_n", "part_off", "row_ids", "dense", "col_ids", "cand_ids", "cand_pos",
          "ncols_q", "cand_rec", "only", "gate", "allow")
SCALARS = ("mode", "nprobes", "nlist", "ncols", "row_stride", "inner", "outer_stride", "B", "k", "has_lower",
           "has_upper", "lower", "upper", "allow_bits", "dist_len")


# ---------------------------------------------------------------- 1. the select alone
def _upload(arr):
    import torch
    b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    t = torch.zeros(b.size + 16, dtype=torch.uint8, device="cuda")
    t[:b.size].copy_(torch.from_numpy(b.copy()))
    return t, t.data_ptr()


def run_select(a, what, pos=False, rec=False):
    """lgpu_debug_select_large on device copies of case `a`, every output byte (guard bands included) against the
    restatement"""
    import torch
    keep, args = [], {n: (float if n in ("lower", "upper") else int)(a[n]) for n in SCALARS if a.get(n) is not None}
    for n in INPUTS:
        if a.get(n) is not None:
            t, args[n] = _upload(a[n])
            keep.append(t)
    B, k = a["B"], a["k"]
    exp = so.outputs(B, k, pos, rec, FILL)
    bufs = {}
    for n, arr in exp.items():
        bufs[n] = torch.full((arr.nbytes + 2 * GUARD,), FILL, dtype=torch.uint8, device="cuda")
        args["out_" + n] = bufs[n].data_ptr() + GUARD
    _native.debug_select_large(**args)
    so.select(a, exp)
    torch.cuda.synchronize()
    for n, t in bufs.items():
        got = t.cpu().numpy()
        assert np.all(got[:GUARD] == FILL) and np.all(got[-GUARD:] == FILL), f"{what}: write outside {n}"
        g = got[GUARD:-GUARD].view(np.uint8).reshape(B, -1)
        e = np.ascontiguousarray(exp[n]).view(np.uint8).reshape(B, -1)
        bad = np.nonzero((g != e).any(axis=1))[0]
        assert bad.size == 0, f"{what}: {n} differs in {bad.size} queries, first q={bad[0]}"


def _keys(order, n, rng, shift=0.0):
    """adversarial value sets: the select_oracle orders plus NaN-only, +-inf only, -0 / +0 only and a few distinct
    values with huge multiplicities"""
    if order == "nan":
        return np.full(n, np.nan, np.float32)
    if order == "inf":
        return np.where(rng.random(n) < 0.5, np.inf, -np.inf).astype(np.float32)
    if order == "zeros":
        return np.where(rng.random(n) < 0.5, 0.0, -0.0).astype(np.float32)
    if order == "few":
        return rng.choice(np.array([-1.0, 0.5, 0.5000001, 3.0], np.float32) + np.float32(shift), n)
    return so.values(order, n, rng, shift=shift)


ORDERS = ["asc", "desc", "equal", "two", "mixed", "nan", "inf", "zeros", "few"]


@pytest.mark.parametrize("k", [2049, 4097, 65536])
def test_dense_rows(k):
    """mode 1: n = k - 1, k, k + 1 and 2 k + 3 candidates in every order, ids the column, descending ids or scattered
    40-bit ids; outputs as ids + values or as records, with positions"""
    rng = np.random.default_rng(k)
    i = 0
    for n in (k - 1, k, k + 1, 2 * k + 3):
        for order in ORDERS:
            B = 2
            V = np.stack([_keys(order, n, rng, 0.25 * q) for q in range(B)])
            ids = [None, np.arange(n, dtype=np.uint64)[::-1] * 3 + 5, so.unique_ids(rng, n)][i % 3]
            run_select(so.dense_case(V, k, col_ids=ids), f"dense k={k} n={n} {order}", pos=i % 2 == 0, rec=i % 4 == 1)
            i += 1


@pytest.mark.parametrize("k", [2049, 4097, 65536])
def test_segments_and_lists(k):
    """mode 0 (partitions, unused probe slots, empty partitions, shuffled row ids, positions) and mode 2 (lists of
    different lengths with unused slots, cut by ncols_q, positions from cand_pos, packed records in the merge layout)"""
    rng = np.random.default_rng(10 + k)
    sizes = [0, 1, 5, k // 3, k // 2 + 1, k, 3001, 0]
    B, nprobes = 3, 5
    for order in ("mixed", "equal", "few"):
        parts = [_keys(order, n, rng, shift=p) for p, n in enumerate(sizes)]
        row_ids = rng.permutation(sum(sizes)).astype(np.uint64) * 5 + 3
        probes = np.stack([rng.permutation(len(sizes))[:nprobes] for _ in range(B)]).astype(np.uint64)
        probes[0, 1] = U64_MAX
        probes[2] = [0, 7, 2, 3, 5]
        for pos in (False, True):
            a = so.segments_case(parts, probes, k, row_ids=None if order == "equal" else row_ids)
            run_select(a, f"segments k={k} {order} pos={pos}", pos=pos, rec=order == "few")
    lens = np.array([0, k, k + 7, 2 * k + 1])
    vals = [_keys("mixed", int(m), rng) for m in lens]
    ids = [so.unique_ids(rng, int(m)) for m in lens]
    posv = [rng.integers(0, 1 << 40, int(m)).astype(np.uint64) for m in lens]
    for cut in (False, True):
        a = so.cands_case(vals, ids, k, pos=posv, ncols_q=cut)
        run_select(a, f"cands k={k} ncols_q={cut}", pos=True, rec=cut)
    L, Bm = 3, 2
    kk = k // 2 + 1
    counts = np.array([[kk, 0], [kk // 2, kk], [kk, 3]])
    lids, ldist = so.search_lists(rng, L, Bm, kk, counts, so.values("two", 64, rng))
    run_select(so.merge_case(lids, ldist, k, rec=True), f"merge layout k={k}", pos=True)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("k", [2049, 4097])
def test_filters(k, mode):
    """distance range at its edges, allow bitmaps shorter than the largest id, `only`, and the gate"""
    rng = np.random.default_rng(600 + 10 * k + mode)
    B, n = 4, 3 * k
    rows = [_keys("mixed", n, rng) for _ in range(B)]
    if mode == 0:
        a = so.segments_case(rows, np.arange(B, dtype=np.uint64)[:, None], k,
                             row_ids=rng.permutation(B * n).astype(np.uint64))
        top = B * n
    elif mode == 1:
        a = so.dense_case(np.stack(rows), k, col_ids=rng.permutation(n).astype(np.uint64))
        top = n
    else:
        a = so.cands_case(rows, [rng.permutation(B * n)[:n].astype(np.uint64) for _ in range(B)], k)
        top = B * n
    finite = np.sort(np.concatenate(rows)[np.isfinite(np.concatenate(rows))])
    v1, v2 = float(finite[len(finite) // 5]), float(finite[len(finite) // 2])
    bitmap = rng.integers(0, 1 << 32, (top + 31) // 32, dtype=np.uint64).astype(np.uint32)
    only = np.array([1, 0, 1, 0], np.uint32)
    variants = [
        dict(has_lower=1, lower=v1, has_upper=1, upper=v1),
        dict(has_lower=1, lower=v1, has_upper=1, upper=v2),
        dict(has_lower=1, lower=-np.inf, has_upper=1, upper=np.inf),
        dict(has_upper=1, upper=0.0),
        dict(allow=bitmap, allow_bits=int(top * 0.6)),
        dict(allow=bitmap, allow_bits=0),
        dict(only=only),
        dict(gate=np.array([0], np.uint32)),
        dict(has_lower=1, lower=v1, has_upper=1, upper=np.inf, allow=bitmap, allow_bits=top - 7, only=only,
             gate=np.array([2], np.uint32)),
    ]
    for i, v in enumerate(variants):
        run_select({**a, **v}, f"filters mode {mode} k={k} variant {i}", pos=i % 2 == 1, rec=i % 3 == 2)


def test_debug_select_large_refuses_k_outside_its_range():
    a = so.dense_case(np.zeros((1, 10), np.float32), 2048)
    with pytest.raises(ValueError, match="2049"):
        run_select(a, "k = 2048")
    with pytest.raises(ValueError, match="65536"):
        run_select({**a, "k": 65537}, "k = 65537")


def test_searches_refuse_k_above_k_max_before_device_work():
    """k = 65537, or k x refine_factor above 65536, is refused with the limit in the message; nothing is launched and
    the outputs are untouched"""
    from tests.util import random_index
    rng = np.random.default_rng(12)
    ix = random_index(rng, dim=16, nlist=4, m=4, n=2000, with_vectors=True)
    gpu, fl = _native.GpuIvfPq(ix), _native.GpuFlat(rng.standard_normal((100, 16)).astype(np.float32))
    q = np.zeros((2, 16), np.float32)
    try:
        for call in (lambda: gpu.search(q, k=65537, nprobes=2), lambda: gpu.search(q, k=100, refine_factor=656),
                     lambda: fl.search(q, k=65537)):
            n0 = _native.kernel_launch_count()
            with pytest.raises(ValueError, match="65536"):
                call()
            assert _native.kernel_launch_count() == n0
        assert (gpu.search(q, k=100, nprobes=2, refine_factor=655)[2] == 100).all()      # 65500: served
    finally:
        gpu.close()
        fl.close()


# ---------------------------------------------------------------- 2. every search kind against its oracle
@pytest.fixture(scope="module")
def pq8():
    import oracle
    from tests.util import queries, random_index
    rng = np.random.default_rng(1)
    ix = random_index(rng, dim=64, nlist=16, m=16, n=40000, with_vectors=True)
    gpu = _native.GpuIvfPq(ix)
    yield ix, gpu, oracle.OracleIndex.from_data(ix), queries(rng, 12, 64)
    gpu.close()


@pytest.mark.parametrize("k", [2049, 10000, 50000])
def test_ivf_pq(pq8, k):
    """k = 2049 and 10000 over 8 of 16 partitions, and k = 50000 above the 40000 rows of the index"""
    ix, gpu, orc, q = pq8
    np_ = 16 if k > 40000 else 8
    assert_same(gpu.search(q, k=k, nprobes=np_), orc.search(q, k=k, nprobes=np_, nthreads=NTH), f"pq8 k={k}")


def test_ivf_pq_refine_range_prefilter(pq8):
    """limit 100 x refine_factor 30 (3000 candidates re-ranked on the raw vectors); a range search (distance_range
    with a limit above the rows inside it); a prefilter whose starved queries widen to maximum_nprobes"""
    import oracle
    ix, gpu, orc, q = pq8
    assert_same(gpu.search(q, k=100, nprobes=8, refine_factor=30),
                orc.search(q, k=100, nprobes=8, refine_factor=30, nthreads=NTH), "pq8 refine 100x30")
    assert_same(gpu.search(q, k=3000, nprobes=8, refine_factor=2),
                orc.search(q, k=3000, nprobes=8, refine_factor=2, nthreads=NTH), "pq8 refine 3000x2")
    d = orc.search(q[:1], k=5000, nprobes=8, nthreads=NTH)[1][0]
    lo, hi = float(d[100]), float(d[4000])
    got = gpu.search(q, k=20000, nprobes=8, lower=lo, upper=hi)
    assert_same(got, orc.search(q, k=20000, nprobes=8, lower=lo, upper=hi, nthreads=NTH), "pq8 range")
    assert (got[2] < 20000).all() and got[2][0] > 3000                    # everything inside the range came back
    ids = np.asarray(ix.row_ids, np.int64)
    off = np.asarray(ix.part_offsets, np.int64)
    mask = np.zeros(int(ids.max()) + 1, bool)
    mask[ids[:off[4]]] = True                                             # the rows of partitions 0..3
    bm = _native.mask_bitmap(mask)
    assert_same(gpu.search(q, k=3000, nprobes=1, max_nprobes=8, allow=bm, allow_bits=mask.size),
                orc.search(q, k=3000, nprobes=1, max_nprobes=8,
                           allow=oracle.allow_bitmap(np.nonzero(mask)[0], mask.size), allow_bits=mask.size,
                           nthreads=NTH), "pq8 prefilter + widening")


@pytest.mark.parametrize("kind", ["pq4", "sq", "rq"])
def test_other_ivf_kinds(kind):
    """IVF_PQ 4-bit (tie-heavy: 4-bit table sums), IVF_SQ and IVF_RQ at k = 2049, 10000, k > N and limit 100 x
    refine_factor 30"""
    from tests import pq4_oracle, rq_oracle, sq_oracle
    from tests.util import queries
    rng = np.random.default_rng({"pq4": 2, "sq": 3, "rq": 4}[kind])
    if kind == "pq4":
        data = pq4_oracle.random_pq4_index(rng, n=20000, dim=32, nlist=16, m=8, empty=(3,))
        gpu, mod = _native.GpuIvfPq(data), pq4_oracle
    elif kind == "sq":
        data = sq_oracle.random_sq_index(rng, n=20000, dim=32, nlist=16, empty=(3,))
        gpu, mod = _native.GpuIvfSq(data), sq_oracle
    else:
        data = rq_oracle.random_rq_index(rng, n=20000, dim=32, nlist=16, empty=(3,))
        gpu, mod = _native.GpuIvfRq(data), rq_oracle
    q = queries(rng, 8, 32)
    try:
        for k, np_, rf in ((2049, 8, 0), (10000, 8, 0), (25000, 16, 0), (100, 8, 30)):
            assert_same(gpu.search(q, k=k, nprobes=np_, refine_factor=rf),
                        mod.search(data, q, k=k, nprobes=np_, refine_factor=rf, nthreads=NTH),
                        f"{kind} k={k} refine={rf}")
    finally:
        gpu.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_flat(metric):
    """flat float search at k = 2049, 10000 and k > N (30000 rows), B = 9 (the tensor-core shortlist's size for l2, so
    k above 2048 must leave it), with NaN and infinite rows and a NaN query"""
    import oracle
    rng = np.random.default_rng(5)
    v = rng.standard_normal((30000, 64)).astype(np.float32)
    v[7, 3] = np.nan
    v[11] = np.inf
    v[13, 0] = -np.inf
    q = rng.standard_normal((9, 64)).astype(np.float32)
    q[4, 1] = np.nan
    fl = _native.GpuFlat(v)
    try:
        for k in (2049, 10000, 40000):
            assert_same(fl.search(q, k=k, metric=metric),
                        oracle.flat_search(v, q, k=k, metric=metric, nthreads=NTH), f"flat {metric} k={k}")
    finally:
        fl.close()


def test_binary_flat_and_ivf():
    """tie-heavy Hamming rows (16-byte rows drawn from 40 patterns: distances in 0..128 tie in runs of thousands):
    flat binary at k = 2049, 10000 (B = 130: the tensor-core dense path) and k = 65536 > N, binary IVF_FLAT at
    k = 4097"""
    from tests import ivf_binary_oracle
    from tests.hamming_oracle import flat_search_u8
    rng = np.random.default_rng(6)
    pat = rng.integers(0, 256, (40, 16), dtype=np.uint8)
    x = pat[rng.integers(0, 40, 60000)]
    x[rng.random(x.shape) < 0.02] ^= 1
    bx = _native.GpuBinary(x)
    try:
        for k, B in ((2049, 3), (10000, 130), (65536, 2)):
            q = x[rng.integers(0, 60000, B)]
            assert_same(bx.search(q, k=k), flat_search_u8(x, q, k=k, nthreads=NTH), f"binary k={k} B={B}")
    finally:
        bx.close()
    bix = ivf_binary_oracle.random_index(rng, 30000, 32, 64, patterns=50)
    ib = _native.GpuIvfBinary(bix)
    q = bix.vectors[rng.integers(0, 30000, 16)]
    try:
        for k, np_, rf in ((4097, 8, 0), (4097, 8, 30)):          # refine_factor is ignored: k x 30 is not limited
            assert_same(ib.search(q, k=k, nprobes=np_, refine_factor=rf),
                        ivf_binary_oracle.search(bix, q, k=k, nprobes=np_, nthreads=NTH), f"ivf binary k={k}")
    finally:
        ib.close()


def test_multivector():
    """multivector (MaxSim) search at k = 2049 and k > N, rows of 0..8 vectors (empty rows have no distance)"""
    from tests.multivec_oracle import flat_search_mv, offsets_of
    rng = np.random.default_rng(7)
    off = offsets_of(rng.integers(0, 9, 5000))
    x = rng.standard_normal((int(off[-1]), 16)).astype(np.float32)
    qoff = offsets_of([1, 3, 7])
    q = rng.standard_normal((int(qoff[-1]), 16)).astype(np.float32)
    mv = _native.GpuMultivec(x, off)
    try:
        for k in (2049, 6000):
            assert_same(mv.search(q, k=k, q_offsets=qoff),
                        flat_search_mv(x, off, q, qoff, k=k, nthreads=NTH), f"multivector k={k}")
    finally:
        mv.close()


# ---------------------------------------------------------------- 3. pagination, 4. entry points
def test_pages_concatenate():
    """through the table API: offset(o).limit(l) pages of one query concatenate to limit(o + l) (pages across the
    2048 boundary and deep ones), and limit(100).refine_factor(30) returns the oracle's 100 rows"""
    import lancedb_b200 as lancedb
    import oracle
    rng = np.random.default_rng(8)
    x = rng.standard_normal((20000, 32)).astype(np.float32)
    db = lancedb.connect("memory://")
    t = db.create_table("v", {"vector": x, "id": np.arange(20000)})
    t.create_index(metric="l2", num_partitions=8, num_sub_vectors=8, max_iterations=2, accelerator="cuda")
    q = rng.standard_normal(32).astype(np.float32)
    whole = t.search(q).nprobes(8).limit(6100).with_row_id(True).to_arrow()
    assert whole.num_rows == 6100
    rows, dist = whole["_rowid"].to_pylist(), np.asarray(whole["_distance"].to_pylist(), np.float32)
    for o, l in ((0, 2049), (2000, 100), (2049, 2049), (4098, 2002)):
        page = t.search(q).nprobes(8).offset(o).limit(l).with_row_id(True).to_arrow()
        assert page["_rowid"].to_pylist() == rows[o:o + l], (o, l)
        assert np.array_equal(np.asarray(page["_distance"].to_pylist(), np.float32).view(np.uint32),
                              dist[o:o + l].view(np.uint32))
    out = t.search(q).nprobes(8).limit(100).refine_factor(30).with_row_id(True).to_arrow()
    ri, rd, rc = oracle.OracleIndex.from_data(t._index_data["vector"]).search(q[None], k=100, nprobes=8,
                                                                              refine_factor=30, nthreads=NTH)
    assert out["_rowid"].to_pylist() == [int(v) for v in ri[0]]
    assert np.array_equal(np.asarray(out["_distance"].to_pylist(), np.float32).view(np.uint32), rd[0].view(np.uint32))


def test_entry_points_agree():
    """host, filtered (every row allowed), device, async and coalesced entry points at k = 3000 and limit 100 x
    refine_factor 30, bit for bit"""
    import torch
    from tests.util import queries, random_index
    rng = np.random.default_rng(9)
    ix = random_index(rng, dim=32, nlist=8, m=8, n=20000, with_vectors=True)
    gpu = _native.GpuIvfPq(ix)
    q = queries(rng, 5, 32)
    allow = np.ones(int(np.max(ix.row_ids)) + 1, bool)
    try:
        for k, rf in ((3000, 0), (100, 30)):
            host = gpu.search(q, k=k, nprobes=4, refine_factor=rf)
            filt = gpu.search(q, k=k, nprobes=4, refine_factor=rf, allow=_native.mask_bitmap(allow),
                              allow_bits=allow.size)
            p = _native.make_params(k, 4, rf)
            dq = torch.from_numpy(q).cuda()
            di = torch.empty((5, k), dtype=torch.int64, device="cuda")
            dd = torch.empty((5, k), dtype=torch.float32, device="cuda")
            dc = torch.empty(5, dtype=torch.int32, device="cuda")
            gpu.search_device(dq.data_ptr(), 5, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr())
            torch.cuda.synchronize()
            dev = (di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32))
            ai, ad, ac = np.empty((5, k), np.uint64), np.empty((5, k), np.float32), np.empty(5, np.uint32)
            _native.ticket_wait(gpu.search_async(np.ascontiguousarray(q), p, ai, ad, ac))
            one = [gpu.search_one(q[i], k=k, nprobes=4, refine_factor=rf) for i in range(5)]
            co = (np.stack([o[0] for o in one]), np.stack([o[1] for o in one]),
                  np.array([o[2] for o in one], np.uint32))
            for name, got in (("filtered", filt), ("device", dev), ("async", (ai, ad, ac)), ("coalesced", co)):
                assert_same(got, host, f"{name} k={k} refine={rf}")
    finally:
        gpu.close()


# ---------------------------------------------------------------- 5. sub-batches
SPLIT_BYTES = 4 << 20


def _child_cases(out_path):
    """every large-k case of the sub-batch check, results into out_path (one npz)"""
    from tests.multivec_oracle import offsets_of
    from tests.util import queries, random_index
    rng = np.random.default_rng(11)
    res = {}

    def put(name, call):
        n0 = _native.kernel_launch_count()
        ids, dist, cnt = call()
        res[f"{name}/launches"] = np.array(_native.kernel_launch_count() - n0)
        res[f"{name}/ids"], res[f"{name}/dist"], res[f"{name}/cnt"] = ids, dist, cnt

    ix = random_index(rng, dim=32, nlist=16, m=8, n=30000, with_vectors=True)
    gpu = _native.GpuIvfPq(ix)
    q = queries(rng, 40, 32)
    put("pq8_k3000", lambda: gpu.search(q, k=3000, nprobes=8))
    put("pq8_refine", lambda: gpu.search(q, k=100, nprobes=8, refine_factor=30))
    gpu.close()
    v = rng.standard_normal((30000, 32)).astype(np.float32)
    fl = _native.GpuFlat(v)
    put("flat_k4000", lambda: fl.search(q, k=4000))
    fl.close()
    x = rng.integers(0, 4, (30000, 16), dtype=np.uint8)
    bx = _native.GpuBinary(x)
    put("binary_k4000", lambda: bx.search(x[:40], k=4000))
    bx.close()
    off = offsets_of(rng.integers(0, 5, 8000))
    mx = rng.standard_normal((int(off[-1]), 16)).astype(np.float32)
    qoff = offsets_of(rng.integers(1, 4, 40))
    mq = rng.standard_normal((int(qoff[-1]), 16)).astype(np.float32)
    mv = _native.GpuMultivec(mx, off)
    put("multivec_k2100", lambda: mv.search(mq, k=2100, q_offsets=qoff))
    mv.close()
    np.savez(out_path, **res)


def _child(path, budget):
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_NO_GRAPH="1")
    env.pop("LGPU_WS_BYTES", None)
    if budget:
        env["LGPU_WS_BYTES"] = str(budget)
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_large_k", str(path)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"LGPU_WS_BYTES={budget or 'default'}:\n{r.stdout[-2000:]}\n{r.stderr[-6000:]}"
    return dict(np.load(path))


def test_sub_batches_give_the_unsplit_result(tmp_path):
    """a 4 MiB workspace budget cuts each 40-query batch into three or more sub-batches (about 0.3 MB a query: the
    large select's scratch and the refine buffers count in the budget); every case equals the unsplit run bit for bit,
    and launched more kernels"""
    split = _child(tmp_path / "split.npz", SPLIT_BYTES)
    whole = _child(tmp_path / "whole.npz", 0)
    names = sorted({k.split("/")[0] for k in whole})
    assert len(names) == 5
    for n in names:
        for f in ("ids", "cnt"):
            assert np.array_equal(split[f"{n}/{f}"], whole[f"{n}/{f}"]), f"{n}: {f} differ when split"
        assert np.array_equal(split[f"{n}/dist"].view(np.uint32), whole[f"{n}/dist"].view(np.uint32)), n
        assert split[f"{n}/launches"] > whole[f"{n}/launches"], f"{n}: the budget did not split the batch"


if __name__ == "__main__":
    _child_cases(sys.argv[1])

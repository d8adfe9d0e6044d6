"""IVF_HNSW_SQ on the GPU: GpuIvfHnswSq against the C oracle (ids, counts and distance bits) over metrics, dims 24,
100 (padding) and 768, ef below / at / above k and above the partition size, refine, prefilter with maximum_nprobes,
distance_range, nprobes >= nlist, sub-batches and every search entry point; a complete graph against the GPU IVF_SQ
search; and the refusals."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from lancedb_b200 import _native
from tests import hnsw_sq_oracle as H
from tests.util import assert_same

pytestmark = pytest.mark.gpu
f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


_IX = {}


def _index(dim, metric):
    key = (dim, metric)
    if key not in _IX:
        rng = np.random.default_rng(dim + (7 if metric == "cosine" else 0))
        data = H.random_hnsw_index(rng, n=1500 if dim < 700 else 900, dim=dim, nlist=5, metric=metric, m=6,
                                   ef_construction=40, empty=(1,))
        _IX[key] = (data, _native.GpuIvfHnswSq(data))
    return _IX[key]


def _queries(rng, data, B):
    q = rng.standard_normal((B, data.dim)).astype(f32)
    q[1] = data.vectors[7]                                 # a stored row and its duplicates
    q[2] *= 1000.0                                        # codes saturate
    return q


CASES = [dict(k=10, nprobes=3), dict(k=10, nprobes=3, ef=4), dict(k=10, nprobes=2, ef=10),
         dict(k=7, nprobes=2, ef=2048), dict(k=10, nprobes=9), dict(k=5, nprobes=2, refine_factor=4),
         dict(k=10, nprobes=3, lower=1000.0, upper=200000.0), dict(k=1, nprobes=1), dict(k=300, nprobes=5, ef=700)]


@pytest.mark.parametrize("dim", [24, 100, 768])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_search_equals_the_c_oracle(dim, metric, case):
    data, g = _index(dim, metric)
    q = _queries(np.random.default_rng(case), data, 37)
    kw = CASES[case]
    assert_same(g.search(q, **kw), H.search(data, q, **kw), f"{dim} {metric} {kw}")


@pytest.mark.parametrize("dim", [24, 100])
def test_prefilter_with_widening_equals_the_c_oracle(dim):
    data, g = _index(dim, "l2")
    rng = np.random.default_rng(3)
    q = _queries(rng, data, 20)
    nbits = int(data.row_ids.max()) + 1
    mask = rng.random(nbits) < 0.03                        # selective: many queries widen
    bm = _native_bitmap(mask)
    for kw in (dict(k=10, nprobes=1, max_nprobes=5), dict(k=10, nprobes=2, max_nprobes=5, ef=30, refine_factor=2)):
        got = g.search(q, allow=bm, allow_bits=nbits, **kw)
        assert_same(got, H.search(data, q, allow=mask, **kw), str(kw))


def _native_bitmap(mask):
    import oracle
    return oracle.allow_bitmap(np.nonzero(mask)[0], mask.size)


def test_complete_graph_equals_the_gpu_ivf_sq_search():
    from tests.sq_oracle import random_sq_index
    sq = random_sq_index(np.random.default_rng(9), n=300, dim=24, nlist=5)
    big = int(np.diff(sq.part_offsets.astype(np.int64)).max())
    assert big <= 2 * 64 + 1                               # a complete level-0 list fits in 2m <= 128 entries
    full = H.complete_graph(sq)
    g, s = _native.GpuIvfHnswSq(full), _native.GpuIvfSq(sq)
    q = _queries(np.random.default_rng(5), full, 16)
    for kw in (dict(k=10, nprobes=5), dict(k=10, nprobes=2, refine_factor=3)):
        assert_same(g.search(q, ef=2048, **kw), s.search(q, **kw), str(kw))


def test_every_entry_point_returns_the_host_result():
    import torch
    data, g = _index(100, "cosine")
    q = _queries(np.random.default_rng(9), data, 12)
    kw = dict(k=10, nprobes=3, ef=40)
    want = g.search(q, **kw)
    assert_same(want, H.search(data, q, **kw), "host")
    p = _native.make_params(10, 3, ef=40)
    dq = torch.as_tensor(q, device="cuda")
    di = torch.empty((12, 10), dtype=torch.int64, device="cuda")
    dd = torch.empty((12, 10), dtype=torch.float32, device="cuda")
    dc = torch.empty(12, dtype=torch.int32, device="cuda")
    g.search_device(dq.data_ptr(), 12, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(), 0)
    torch.cuda.synchronize()
    assert_same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want, "device")
    ids, dist, cnt = np.empty((12, 10), np.uint64), np.empty((12, 10), f32), np.empty(12, np.uint32)
    t = g.search_async(q, p, ids, dist, cnt)
    _native.ticket_wait(t)
    assert_same((ids, dist, cnt), want, "async")
    out = [None] * 12

    def one(i):
        out[i] = g.search_one(q[i], k=10, nprobes=3, ef=40)
    th = [threading.Thread(target=one, args=(i,)) for i in range(12)]
    [x.start() for x in th]
    [x.join() for x in th]
    for i, (oi, od, oc) in enumerate(out):
        assert_same((oi[None], od[None], np.array([oc], np.uint32)), tuple(a[i:i + 1] for a in want), f"coalesced {i}")


_CHILD = r"""
import numpy as np
from lancedb_b200 import _native
from tests import hnsw_sq_oracle as H
rng = np.random.default_rng(11)
data = H.random_hnsw_index(rng, n=1500, dim=100, nlist=5, m=6, ef_construction=40)
g = _native.GpuIvfHnswSq(data)
q = rng.standard_normal((300, 100)).astype(np.float32)
assert g.debug_sub_batch_size(300, 5) < 300
for kw in (dict(k=10, nprobes=5, ef=64), dict(k=10, nprobes=2, refine_factor=3)):
    a, b = g.search(q, **kw), H.search(data, q, **kw)
    assert all(np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y) for x, y in zip(a, b)), kw
print("ok")
"""


def test_sub_batches_equal_the_c_oracle():
    env = dict(os.environ, LGPU_WS_BYTES=str(4 << 20))
    r = subprocess.run([sys.executable, "-c", _CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_refusals():
    data, g = _index(24, "l2")
    q = np.zeros((2, 24), f32)
    with pytest.raises(ValueError, match="2048"):
        g.search(q, k=10, nprobes=2, ef=2049)
    with pytest.raises(ValueError, match="2048"):
        g.search(q, k=100, nprobes=2, refine_factor=21)
    with pytest.raises(ValueError):
        bad = H.random_hnsw_index(np.random.default_rng(1), n=200, dim=24, nlist=3)
        bad.adj0[0, 0] = 100000
        _native.GpuIvfHnswSq(bad)
    lib = _native.load()                                   # the handle is an lgpu_index, not a binary IVF_FLAT one
    qb, ids, dist, cnt = np.zeros(3, np.uint8), np.empty(1, np.uint64), np.empty(1, f32), np.empty(1, np.uint32)
    p = _native.make_params(1, 1)
    rc = lib.lgpu_ivf_binary_search(g._h, qb.ctypes.data, 1, p, ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
    assert rc == _native.LGPU_INVALID_INPUT and b"handle expected" in lib.lgpu_last_error()


def test_ef_sweep_with_one_shape_equals_the_c_oracle_on_every_call():
    # repeated calls with one (B, k, nprobes) replay a captured launch sequence: ef must select its own
    data, g = _index(24, "l2")
    q = _queries(np.random.default_rng(21), data, 16)
    ids, dist, cnt = np.empty((16, 10), np.uint64), np.empty((16, 10), f32), np.empty(16, np.uint32)
    for ef in (16, 16, 16, 40, 11, 200, 16, 40):
        want = H.search(data, q, k=10, nprobes=3, ef=ef)
        assert_same(g.search(q, k=10, nprobes=3, ef=ef), want, f"sync ef {ef}")
        _native.ticket_wait(g.search_async(q, _native.make_params(10, 3, ef=ef), ids, dist, cnt))
        assert_same((ids, dist, cnt), want, f"async ef {ef}")


def test_wide_lists_duplicate_neighbours_and_a_single_row_partition():
    # m 40: level-0 lists of 80 and upper lists of 40 entries (over a warp); every level-0 list repeats its first neighbour;
    # partition 3 holds one row
    from lancedb_b200.index import IvfHnswSqIndexData, build_hnsw_graph
    from tests.sq_oracle import random_sq_index
    sq = random_sq_index(np.random.default_rng(12), n=3000, dim=100, nlist=5, empty=(1,))
    off = sq.part_offsets.astype(np.int64)
    keep = np.ones(sq.nrows, bool)
    keep[off[3] + 1:off[4]] = False                      # partition 3 -> one row
    new_off = np.zeros(6, np.uint64)
    new_off[1:] = np.cumsum([int(keep[off[p]:off[p + 1]].sum()) for p in range(5)])
    sq.codes, sq.row_ids, sq.vectors, sq.part_offsets = sq.codes[keep], sq.row_ids[keep], sq.vectors[keep], new_off
    lv, adj0, ui, ua, entry, top = build_hnsw_graph(sq.codes, sq.part_offsets, 40, 100)
    full = adj0 != H.NONE
    last = full.sum(1)
    rows = np.nonzero((last > 0) & (last < 80))[0]
    adj0[rows, last[rows]] = adj0[rows, 0]                # a repeated neighbour
    a2 = int(new_off[2])                                  # partition 2: 50 rows on level 1, each listing 40 of them
    lv[a2:int(new_off[3])] = 0
    lv[a2:a2 + 50] = 1
    ui[a2:int(new_off[3])] = H.NONE
    ui[a2:a2 + 50] = ua.shape[0] + np.arange(50)
    ua = np.concatenate([ua, ((np.arange(50)[:, None] + 1 + np.arange(40)[None, :]) % 50).astype(np.uint32)])
    entry[2], top[2] = 0, 1
    data = IvfHnswSqIndexData(sq, 40, lv, adj0, ui, ua, entry, top)
    data.validate()
    assert int(np.diff(new_off.astype(np.int64))[3]) == 1 and int((ua != H.NONE).sum(1).max()) > 32
    g = _native.GpuIvfHnswSq(data)
    q = _queries(np.random.default_rng(13), data, 40)
    for kw in (dict(k=10, nprobes=5), dict(k=10, nprobes=5, ef=150), dict(k=3, nprobes=2, ef=3)):
        assert_same(g.search(q, **kw), H.search(data, q, **kw), str(kw))


# recall@10 of a CUDA-built graph against IVF_SQ over the same probes; the CPU build of this fixture reaches 0.974
# (tests/test_hnsw_sq_host.py), and the CUDA build must meet the same floor
def test_cuda_built_index_validates_and_meets_the_recall_floor():
    from lancedb_b200.index import train_ivf_hnsw_sq
    from tests import sq_oracle
    from tests.test_hnsw_sq_host import RECALL_FLOOR
    rng = np.random.default_rng(1)
    centres = rng.standard_normal((12, 32)).astype(f32) * 4
    x = (centres[rng.integers(0, 12, 2000)] + rng.standard_normal((2000, 32))).astype(f32)
    data = train_ivf_hnsw_sq(x, num_partitions=4, m=8, ef_construction=64, max_iterations=10, device="cuda")
    data.validate()
    assert (data.adj0 != H.NONE).sum(1).mean() > 4       # the lists are not collapsed
    q = (centres[rng.integers(0, 12, 50)] + rng.standard_normal((50, 32))).astype(f32)
    gi, gd, gc = _native.GpuIvfHnswSq(data).search(q, k=10, nprobes=2)
    assert_same((gi, gd, gc), H.search(data, q, k=10, nprobes=2), "cuda-built")
    si, _, _ = sq_oracle.search(data.sq, q, k=10, nprobes=2)
    assert np.mean([len(set(a) & set(b)) / 10 for a, b in zip(gi.tolist(), si.tolist())]) >= RECALL_FLOOR


def test_create_index_and_query_ef_through_the_table():
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(4)
    x = rng.standard_normal((3000, 32)).astype(f32)
    t = lancedb.connect("memory://").create_table("t", {"vector": x, "id": np.arange(3000)})
    t.create_index(metric="l2", num_partitions=4, index_type="IVF_HNSW_SQ", m=8, ef_construction=64,
                   accelerator="cuda", max_iterations=5)
    assert t.list_indices()[0]["index_type"] == "IVF_HNSW_SQ"
    data = t._index_data["vector"]
    for ef in (None, 12, 80):
        b = t.search(x[5]).limit(10).nprobes(2)
        if ef:
            b = b.ef(ef)
        got = b.with_row_id(True).to_arrow()
        oi, od, oc = H.search(data, x[5:6], k=10, nprobes=2, ef=ef or 0)
        assert got["_rowid"].to_pylist() == oi[0, :oc[0]].tolist()
        assert np.array_equal(np.asarray(got["_distance"], f32).view(np.uint32), od[0, :oc[0]].view(np.uint32))

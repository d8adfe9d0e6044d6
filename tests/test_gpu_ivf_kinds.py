"""IVF_SQ, IVF_RQ and 4-bit IVF_PQ on the GPU, from one kind table: each kind's handle against its C oracle (ids, counts
and distance bits) over metrics, list counts, batch sizes, k, partition shapes, awkward queries, prefilter,
maximum_nprobes, distance_range, refine_factor and every search entry point; then create_index through the builder.
What only one kind has (its scan kernel's debug entry, its refusals) is in test_gpu_ivf_sq.py, test_gpu_ivf_rq.py and
test_gpu_ivf_pq4.py."""
import threading
from dataclasses import dataclass
from types import ModuleType
from typing import Callable, Tuple

import numpy as np
import pytest

import lancedb_b200 as lancedb
import oracle
from lancedb_b200 import _native
from lancedb_b200.index import IVF_KINDS
from tests import pq4_oracle, rq_oracle, sq_oracle
from tests.pq4_oracle import random_pq4_index
from tests.rq_oracle import random_rq_index
from tests.sq_oracle import random_sq_index
from tests.util import assert_same, ivf_queries

pytestmark = pytest.mark.gpu
f32 = np.float32


def _gaussian(rng):
    x = rng.standard_normal((5000, 64)).astype(f32)
    return x, rng.standard_normal((3, 64)).astype(f32)


def _clustered(rng):
    """rows around 32 centres, queries near the first three rows"""
    centers = rng.standard_normal((32, 64)).astype(f32) * 3
    x = (centers[rng.integers(0, 32, 5000)] + rng.standard_normal((5000, 64))).astype(f32)
    return x, (x[:3] + 0.1 * rng.standard_normal((3, 64))).astype(f32)


@dataclass(frozen=True)
class Kind:
    """One IVF kind and the data of each test.  `seed` is a {metric: seed} dict where each metric has its own; index
    arguments go to random_index(rng, metric=metric, **arguments).
      small_lists: seed, main (the index), tiny (the index searched with k > N)
      coarse: seed, index (1024 lists: the tensor-core coarse step)
      prefilter: seed, index, allow_bits(ix) (the prefilter bitmap's length)
      entry_points: seed, index (l2, the generators' default metric), device_bytes(ix) (a floor), code_bytes(ix)
        (per scanned row)
      create_index: seed, index_type, args (the other create_index arguments), accelerator (per metric),
        draw(rng) -> (rows, queries), trained (attributes of the trained data), refine_factor, and recall:
        (floor, refine_factor) against the exact flat search, or None"""
    random_index: Callable          # random_{sq,rq,pq4}_index
    oracle: ModuleType              # its C oracle: search(ix, q, k, nprobes, ...)
    handle: type                    # the _native handle class
    metrics: Tuple[str, ...]
    far: float                      # the scale that sends query 1 far away
    small_lists: dict
    coarse: dict
    prefilter: dict
    entry_points: dict
    create_index: dict


KINDS = {
    "sq": Kind(
        random_sq_index, sq_oracle, _native.GpuIvfSq, ("l2", "cosine"), far=1000.0,     # codes saturate
        small_lists=dict(seed={"l2": 21, "cosine": 22}, main=dict(n=6000, dim=40, nlist=16, empty=(2, 9)),
                         tiny=dict(n=150, dim=40, nlist=16, empty=(0, 3, 4))),
        coarse=dict(seed={"l2": 23, "cosine": 24}, index=dict(n=60000, dim=128, nlist=1024, empty=(5, 77))),
        prefilter=dict(seed={"l2": 25, "cosine": 26}, index=dict(n=8000, dim=48, nlist=32),
                       allow_bits=lambda ix: ix.nrows * 3 + 7),
        entry_points=dict(seed=27, index=dict(n=5000, dim=32, nlist=24),
                          device_bytes=lambda ix: ix.nrows * (64 + 4 + 8),     # codes padded to 64 bytes, |k|^2, ids
                          code_bytes=lambda ix: ix.dim),
        create_index=dict(seed=29, index_type="IVF_SQ", args={}, accelerator={"l2": "cuda", "cosine": "cuda"},
                          draw=_gaussian, trained={}, refine_factor=3,
                          recall=(0.6, 0)),                                     # SQ ranks close to f32
    ),
    "rq": Kind(
        random_rq_index, rq_oracle, _native.GpuIvfRq, ("l2", "cosine"), far=1e4,        # huge magnitude
        small_lists=dict(seed={"l2": 31, "cosine": 32}, main=dict(n=6000, dim=40, nlist=16, empty=(2, 9)),
                         tiny=dict(n=150, dim=40, nlist=16, empty=(0, 3, 4))),
        coarse=dict(seed={"l2": 33, "cosine": 34}, index=dict(n=60000, dim=128, nlist=1024, empty=(5, 77))),
        prefilter=dict(seed={"l2": 35, "cosine": 36}, index=dict(n=8000, dim=300, nlist=32),
                       allow_bits=lambda ix: ix.nrows * 3 + 7),
        # codes padded to 256 bits, add / scale / popc, row ids, the rotation
        entry_points=dict(seed=37, index=dict(n=5000, dim=100, nlist=24),
                          device_bytes=lambda ix: ix.nrows * (32 + 12 + 8) + ix.dim * ix.dim * 4,
                          code_bytes=lambda ix: 32),                             # dim 100 -> 256 bits = 32 bytes
        create_index=dict(seed=39, index_type="IVF_RQ", args=dict(num_bits=1),
                          accelerator={"l2": "cuda", "cosine": "cuda"}, draw=_clustered, trained={}, refine_factor=10,
                          recall=(0.6, 10)),                        # loose and refined: RQ is a refine-first index
    ),
    "pq4": Kind(
        random_pq4_index, pq4_oracle, _native.GpuIvfPq, ("l2", "cosine", "dot"), far=1000.0,  # off every codeword
        small_lists=dict(seed={"l2": 31, "cosine": 32, "dot": 33}, main=dict(n=6000, dim=48, nlist=16, m=12,
                                                                             empty=(2, 9)),
                         tiny=dict(n=150, dim=48, nlist=16, m=12,
                                   sizes=[0, 1, 0, 30, 1, 20, 0, 18, 1, 40, 0, 10, 9, 10, 0, 10])),
        coarse=dict(seed={"l2": 34, "cosine": 35, "dot": 36},
                    index=dict(n=60000, dim=128, nlist=1024, m=16, empty=(5, 77), with_vectors=False)),
        prefilter=dict(seed={"l2": 41, "cosine": 42, "dot": 43}, index=dict(n=8000, dim=48, nlist=32, m=24),
                       allow_bits=lambda ix: int(ix.row_ids.max()) + 1 - 37),
        entry_points=dict(seed=45, index=dict(n=5000, dim=32, nlist=24, m=8),
                          device_bytes=lambda ix: ix.nrows * (ix.m // 2 + 8),   # packed codes, row ids
                          code_bytes=lambda ix: ix.m // 2),
        create_index=dict(seed=47, index_type="IVF_PQ", args=dict(num_bits=4),
                          accelerator={"l2": None, "cosine": "cuda", "dot": "cuda"}, draw=_gaussian,
                          trained=dict(num_bits=4, m=4), refine_factor=3, recall=None),
    ),
}
CASES = [(name, metric) for name, kind in KINDS.items() for metric in kind.metrics]
each_kind_and_metric = pytest.mark.parametrize("name,metric", CASES, ids=[f"{n}-{m}" for n, m in CASES])


@each_kind_and_metric
def test_small_lists_vs_oracle(name, metric):
    kind = KINDS[name]
    case = kind.small_lists
    rng = np.random.default_rng(case["seed"][metric])
    ix = kind.random_index(rng, metric=metric, **case["main"])
    gpu = kind.handle(ix)
    for B in (1, 7, 8, 37):
        q = ivf_queries(rng, ix, B, kind.far)
        for k, nprobes in ((1, 3), (10, 5), (100, 16)):
            got = gpu.search(q, k=k, nprobes=nprobes)
            assert_same(got, kind.oracle.search(ix, q, k=k, nprobes=nprobes), f"B={B} k={k} nprobes={nprobes}")
            if B > 3:
                assert got[2][2] == 0
    gpu.close()
    # k > N, tiny and empty partitions, every partition probed
    tiny = kind.random_index(rng, metric=metric, **case["tiny"])
    gpu = kind.handle(tiny)
    q = ivf_queries(rng, tiny, 9, kind.far)
    got = gpu.search(q, k=200, nprobes=16)
    assert_same(got, kind.oracle.search(tiny, q, k=200, nprobes=16), "k > N")
    assert got[2][0] == 150
    gpu.close()


@each_kind_and_metric
def test_tensor_core_coarse_step_vs_oracle(name, metric):
    kind = KINDS[name]
    case = kind.coarse
    rng = np.random.default_rng(case["seed"][metric])
    ix = kind.random_index(rng, metric=metric, **case["index"])
    gpu = kind.handle(ix)
    q = ivf_queries(rng, ix, 1024, kind.far)
    for k, nprobes in ((10, 20), (100, 8)):
        assert_same(gpu.search(q, k=k, nprobes=nprobes), kind.oracle.search(ix, q, k=k, nprobes=nprobes), f"k={k}")
    gpu.close()


@each_kind_and_metric
def test_prefilter_range_refine_vs_oracle(name, metric):
    kind = KINDS[name]
    case = kind.prefilter
    rng = np.random.default_rng(case["seed"][metric])
    ix = kind.random_index(rng, metric=metric, **case["index"])
    gpu = kind.handle(ix)
    q = ivf_queries(rng, ix, 40, kind.far)
    nbits = case["allow_bits"](ix)
    mask = rng.random(nbits) < 0.02                           # narrow: many queries need maximum_nprobes
    bm = _native.mask_bitmap(mask)
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits, max_nprobes=32)
    assert_same(got, kind.oracle.search(ix, q, k=10, nprobes=2, allow=mask, max_nprobes=32),
                "prefilter + maximum_nprobes")
    got = gpu.search(q, k=10, nprobes=2, allow=bm, allow_bits=nbits)
    assert_same(got, kind.oracle.search(ix, q, k=10, nprobes=2, allow=mask), "prefilter")
    d = kind.oracle.search(ix, q[:1], k=50, nprobes=4)[1][0]
    lo, hi = float(d[5]), float(d[30])
    got = gpu.search(q, k=20, nprobes=4, lower=lo, upper=hi)
    assert_same(got, kind.oracle.search(ix, q, k=20, nprobes=4, lower=lo, upper=hi), "distance_range")
    got = gpu.search(q, k=7, nprobes=4, refine_factor=5)
    assert_same(got, kind.oracle.search(ix, q, k=7, nprobes=4, refine_factor=5), "refine_factor")
    gpu.close()


def _check_entry_points(name, monkeypatch):
    """the device, async and coalesced entry points against the oracle on an l2 index; device bytes, scanned bytes"""
    import torch
    # the coalescing window is read once per process, at the first coalesced call: take the one
    # test_gpu_api.py's batching test needs, whichever of the two runs first
    monkeypatch.setenv("LGPU_COALESCE_US", "3000")
    kind = KINDS[name]
    case = kind.entry_points
    rng = np.random.default_rng(case["seed"])
    ix = kind.random_index(rng, **case["index"])
    gpu = kind.handle(ix)
    q = ivf_queries(rng, ix, 19, kind.far)
    want = kind.oracle.search(ix, q, k=9, nprobes=6)
    p = _native.make_params(9, 6)
    dq = torch.from_numpy(q).cuda()
    di = torch.empty((19, 9), dtype=torch.int64, device="cuda")
    dd = torch.empty((19, 9), dtype=torch.float32, device="cuda")
    dc = torch.empty(19, dtype=torch.int32, device="cuda")
    gpu.search_device(dq.data_ptr(), 19, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(), 0)
    torch.cuda.synchronize()
    assert_same((di.cpu().numpy().view(np.uint64), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32)), want, "device")
    ids = np.empty((19, 9), np.uint64); dist = np.empty((19, 9), f32); cnt = np.empty(19, np.uint32)
    _native.ticket_wait(gpu.search_async(q, p, ids, dist, cnt))
    assert_same((ids, dist, cnt), want, "async")
    res = [None] * 19

    def one(i):
        res[i] = gpu.search_one(q[i], k=9, nprobes=6)

    th = [threading.Thread(target=one, args=(i,)) for i in range(19)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i in range(19):
        gi, gd, gc = res[i]
        assert gc == want[2][i] and np.array_equal(gi, want[0][i])
        assert np.array_equal(gd.view(np.uint32), want[1][i].view(np.uint32))
    assert gpu.device_bytes() >= case["device_bytes"](ix)
    _native.set_profiling(True)
    gpu.search(q, k=9, nprobes=6)
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    assert scanned > 0 and scanned % case["code_bytes"](ix) == 0
    gpu.close()


def test_ivf_sq_device_async_and_coalesced_entry_points(monkeypatch):
    _check_entry_points("sq", monkeypatch)


def test_ivf_rq_device_async_and_coalesced_entry_points(monkeypatch):
    _check_entry_points("rq", monkeypatch)


def test_ivf_pq4_device_async_and_coalesced_entry_points(monkeypatch):
    _check_entry_points("pq4", monkeypatch)


@each_kind_and_metric
def test_create_index_search_to_arrow(name, metric):
    kind = KINDS[name]
    case = kind.create_index
    rng = np.random.default_rng(case["seed"])
    x, q = case["draw"](rng)
    db = lancedb.connect("memory://")
    t = db.create_table("v", {"vector": x, "id": np.arange(5000)})
    t.create_index(metric=metric, num_partitions=16, index_type=case["index_type"], max_iterations=4,
                   accelerator=case["accelerator"][metric], **case["args"])
    assert t.list_indices()[0]["index_type"] == case["index_type"]
    data = t._index_data["vector"]
    assert isinstance(data, IVF_KINDS[case["index_type"]].data)
    assert {a: getattr(data, a) for a in case["trained"]} == case["trained"]
    oi, od, oc = kind.oracle.search(data, q, k=12, nprobes=4)
    for i in range(3):
        out = t.search(q[i]).distance_type(metric).nprobes(4).limit(10).offset(2).with_row_id(True).to_arrow()
        assert out["_rowid"].to_pylist() == [int(v) for v in oi[i, 2:12]]
        assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32).view(np.uint32), od[i, 2:12].view(np.uint32))
        assert out["id"].to_pylist() == out["_rowid"].to_pylist()
    rf = case["refine_factor"]
    out = t.search(q[0]).distance_type(metric).nprobes(4).refine_factor(rf).limit(5).to_arrow()
    rd = kind.oracle.search(data, q[:1], k=5, nprobes=4, refine_factor=rf)[1]
    assert np.array_equal(np.asarray(out["_distance"].to_pylist(), f32), rd[0])
    if case["recall"] is not None:
        floor, refine_factor = case["recall"]
        fi = oracle.flat_search(x, q, k=10, metric=metric)[0]
        gi = t._index["vector"].search(q, k=10, nprobes=16, refine_factor=refine_factor)[0]
        assert np.mean([len(set(fi[b]) & set(gi[b])) / 10 for b in range(3)]) >= floor

"""Every IVF search path of the library, one request each, against the oracle (bit-identical ids, counts and distance
bits), with the number of kernel launches one host call makes pinned and the seven profiled stage times checked.

The launch counts identify the path a request took: the small path, the filter scan in candidate and dense mode (and
its overflow fix-up), the exact scan, the two tensor-core coarse variants, the IVF_SQ scan, prefilter widening,
distance range and the three metrics.  A count that changes means a launch was added, dropped or moved to another
path."""
import math

import numpy as np
import pytest

import oracle
from lancedb_b200 import _native
from tests import sq_oracle
from tests.sq_oracle import random_sq_index
from tests.util import assert_same, queries, random_index

pytestmark = pytest.mark.gpu

_INDEXES = {}


def _index(name):
    """the indexes of the cases, built once per module"""
    if name not in _INDEXES:
        rng = np.random.default_rng(301)
        if name == "sq":
            _INDEXES[name] = random_sq_index(rng, n=8000, dim=48, nlist=32)
        elif name == "big":                               # nlist >= 1024: the tensor-core coarse variants
            _INDEXES[name] = random_index(rng, dim=64, nlist=1024, m=8, n=60000)
        else:                                             # "l2", "cosine", "dot"
            _INDEXES[name] = random_index(rng, dim=64, nlist=64, m=8, n=40000, metric=name, with_vectors=True)
    return _INDEXES[name]


def _allow(n):
    rng = np.random.default_rng(302)
    return np.sort(rng.choice(n, n // 50, replace=False))  # 2 % of the rows: most queries need maximum_nprobes


# name: (index, batch, search arguments, environment)
CASES = {
    "small": ("l2", 2, dict(k=10, nprobes=6), {"LGPU_SMALL_SLOTS": "1024"}),
    "small_refine": ("l2", 2, dict(k=7, nprobes=6, refine_factor=5), {"LGPU_SMALL_SLOTS": "1024"}),
    "filter_candidate": ("l2", 64, dict(k=10, nprobes=8), {}),
    "filter_candidate_refine": ("l2", 64, dict(k=7, nprobes=8, refine_factor=5), {}),
    "filter_dense": ("l2", 64, dict(k=10, nprobes=8), {"LGPU_DENSE_FILTER": "1"}),
    "filter_overflow": ("l2", 64, dict(k=10, nprobes=8), {"LGPU_CAND_CAP": "32"}),
    "exact": ("l2", 64, dict(k=10, nprobes=8), {"LGPU_EXACT_SCAN": "1"}),
    "tc_dense_coarse": ("big", 16, dict(k=10, nprobes=20), {"LGPU_FORCE_TC_COARSE": "1"}),
    "tc_list_coarse": ("big", 64, dict(k=10, nprobes=20), {"LGPU_FORCE_TC_COARSE": "1", "LGPU_COARSE_LIST_MIN": "1024"}),
    "sq": ("sq", 40, dict(k=10, nprobes=4), {}),
    "prefilter_widening": ("l2", 16, dict(k=10, nprobes=2, max_nprobes=64, allow=True), {}),
    "distance_range": ("l2", 16, dict(k=20, nprobes=8, lower=True), {}),
    "cosine": ("cosine", 64, dict(k=10, nprobes=8), {}),
    "dot": ("dot", 64, dict(k=10, nprobes=8), {}),
}

# kernel launches of one host call of each case, after a warm-up call of the same shape
LAUNCHES = {
    "small": 4, "small_refine": 6,
    "filter_candidate": 22, "filter_candidate_refine": 24, "filter_dense": 22, "filter_overflow": 22, "exact": 9,
    "tc_dense_coarse": 25, "tc_list_coarse": 27, "sq": 10, "prefilter_widening": 32, "distance_range": 9,
    "cosine": 23, "dot": 22,
}


def _request(name):
    """(index data, queries, GPU search arguments, oracle search)"""
    ixname, B, kw, _ = CASES[name]
    ix = _index(ixname)
    q = queries(np.random.default_rng(303), B, ix.dim)
    kw = dict(kw)
    if kw.pop("allow", False):
        rows = _allow(int(ix.row_ids.size))
        kw.update(allow=oracle.allow_bitmap(rows, int(ix.row_ids.size)), allow_bits=int(ix.row_ids.size))
    if kw.pop("lower", False):                            # a band inside the first query's unfiltered top 50
        d = oracle.OracleIndex.from_data(ix).search(q[:1], k=50, nprobes=kw["nprobes"], nthreads=8)[1][0]
        kw.update(lower=float(d[5]), upper=float(d[30]))
    if ixname == "sq":
        return ix, q, kw, lambda: sq_oracle.search(ix, q, **kw)
    return ix, q, kw, lambda: oracle.OracleIndex.from_data(ix).search(q, nthreads=8, **kw)


def _run(name):
    """the result of one host call and the kernel launches of a second one; the environment is the caller's"""
    ix, q, kw, want = _request(name)
    gpu = _native.GpuIvfSq(ix) if CASES[name][0] == "sq" else _native.GpuIvfPq(ix)
    try:
        got = gpu.search(q, **kw)
        n0 = _native.kernel_launch_count()
        again = gpu.search(q, **kw)
        launches = _native.kernel_launch_count() - n0
        _native.set_profiling(True)
        try:
            profiled = gpu.search(q, **kw)
            stage_ms = list(_native.last_stage_ms().values())
        finally:
            _native.set_profiling(False)
    finally:
        gpu.close()
    return got, [again, profiled], want(), launches, stage_ms


@pytest.mark.parametrize("name", sorted(CASES))
def test_ivf_path(name, monkeypatch):
    for var, value in CASES[name][3].items():
        monkeypatch.setenv(var, value)
    got, repeats, want, launches, stage_ms = _run(name)
    assert_same(got, want, name)
    for r in repeats:
        assert_same(r, got, f"{name} (repeated)")
    assert launches == LAUNCHES[name], (name, launches)
    assert len(stage_ms) == 7 and all(math.isfinite(t) and t >= 0 for t in stage_ms), stage_ms

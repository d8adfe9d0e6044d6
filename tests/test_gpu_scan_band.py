"""The filter scan's band on the GPU, on the constructions of tests/util.py (see tests/test_scan_band.py for the CPU
restatement): end-to-end results must be bit-identical to the oracle in candidate mode, dense mode, under a prefilter
and at k > 32, with the filter proving some queries itself where the data allows; the band must scale with the data
(l2); and a query whose |q|^2 overflows f32 must still get its k rows."""
import numpy as np
import pytest

import oracle
from lancedb_b200 import _native
from tests.util import (F32, cancellation_case, dot_cancellation_case, filter_bounds, full_lane_case, overflow_case,
                        quantiser_boundary_case, queries, random_index, row_consts, same_result, scaled)

pytestmark = pytest.mark.gpu

CASES = {
    "boundary-l2-m96": lambda: quantiser_boundary_case("l2", 96, rows=(600, 600, 600), B=64),
    "boundary-dot-m8": lambda: quantiser_boundary_case("dot", 8, rows=(600, 600, 600), B=64),
    "lanes-m255-d1": lambda: full_lane_case(255, 1, rows=800, B=64),
    "lanes-m3-d8": lambda: full_lane_case(3, 8, rows=800, B=64),
    "lanes-m17-d4": lambda: full_lane_case(17, 4, rows=800, B=64),
    "cancel-100": lambda: cancellation_case(100.0, n=6000, B=64),
    "dot-cancel": lambda: dot_cancellation_case(n=1500, B=64),
    "chain-dsub32-m96": lambda: _random(3072, 96, 4000, 32),
    "chain-m193": lambda: _random(386, 193, 4000, 32),
    "chain-m512": lambda: _random(512, 512, 3000, 32),
}


# constructions on which the filter proves no query in these modes, by design -- only the parity is checked there:
# a common offset of 100 widens W itself (the tables are on q, not on the residual); dot-cancel makes E large on
# purpose; m 512 multiplies E by ceil(512 / 96) = 6 against a 32-row shortlist; the dot boundary rows nearly tie
NO_PROOF = {"cancel-100": ("candidate", "dense", "prefilter", "k40"), "dot-cancel": ("candidate", "dense", "prefilter", "k40"),
            "chain-m512": ("dense", "prefilter"), "boundary-dot-m8": ("dense",)}


def _random(dim, m, n, B, seed=4):
    rng = np.random.default_rng(seed)
    ix = random_index(rng, dim=dim, nlist=4, m=m, n=n, scale=1 / np.sqrt(dim))
    return ix, queries(rng, B, dim, scale=1 / np.sqrt(dim))


def _search(ix, Q, k, nprobes, **kw):
    gpu = _native.GpuIvfPq(ix)
    _native.set_profiling(True)
    try:
        got = gpu.search(Q, k=k, nprobes=nprobes, **kw)
        st = _native.last_filter_stats()
    finally:
        _native.set_profiling(False)
        gpu.close()
    return got, st


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("case", sorted(CASES) + ["scale-2^-20", "scale-2^20", "overflow"])
def test_kernel_bounds_equal_the_restatement_and_bracket_the_oracle(case):
    """lgpu_debug_filter_bounds returns the L that scan3 wrote in dense mode for every probed row, and the W and E the
    consumers use.  They must equal tests/util.py's restatement (filter_bounds, scan_band) bit for bit -- so the CPU
    tests' constructions and non-vacuity checks speak about the kernels -- and bracket the oracle's d*:
    L - s E <= d* <= L + s (W + E)."""
    if case.startswith("scale"):
        ix, Q = scaled(*_random(768, 96, 20000, 16, seed=9), 2.0 ** int(case.split("^")[1]))
    elif case == "overflow":
        ix, Q = overflow_case(B=8)                                             # every query flagged (bad) by probe_terms
    else:
        ix, Q = CASES[case]()
    Q = Q[:8]
    ld = int(np.diff(ix.part_offsets.astype(np.int64)).max())
    gpu = _native.GpuIvfPq(ix)
    try:
        parts, L, W, E, bad = gpu.debug_filter_bounds(Q, ix.nlist, ld)
    finally:
        gpu.close()
    orc = oracle.OracleIndex.from_data(ix)
    R = None if ix.metric == "dot" else [row_consts(ix, p) for p in range(ix.nlist)]
    checked = 0
    for b, q in enumerate(Q):
        out, Wr, Er, s, bad_r = filter_bounds(ix, orc, q, R=R)
        assert bool(bad[b]) == bad_r, b
        if bad_r:
            continue
        assert _bits(W[b]) == _bits(Wr) and _bits(E[b]) == _bits(Er), (b, W[b], Wr, E[b], Er)
        assert sorted(parts[b].tolist()) == sorted(out), b
        for j, p in enumerate(parts[b]):
            Lr, d = out[int(p)]
            Lg = L[b, j, :len(Lr)]
            assert np.array_equal(_bits(Lg), _bits(Lr)), (b, int(p), int((_bits(Lg) != _bits(Lr)).sum()))
            assert (d >= (Lg - F32(s * E[b])).astype(F32)).all() and (d <= (Lg + F32(s * F32(W[b] + E[b]))).astype(F32)).all()
            checked += len(Lr)
    assert checked > 0 or case == "overflow"


@pytest.mark.parametrize("mode", ["candidate", "dense", "prefilter", "k40"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_constructions_match_the_oracle(case, mode, monkeypatch):
    ix, Q = CASES[case]()
    k, kw = (40 if mode == "k40" else 10), {}
    if mode == "dense":
        monkeypatch.setenv("LGPU_DENSE_FILTER", "1")
    if mode == "prefilter":
        rid = ix.row_ids[np.random.default_rng(1).random(ix.row_ids.size) < 0.7]
        kw = dict(allow=_native.allow_bitmap(rid, int(ix.row_ids.max()) + 1), allow_bits=int(ix.row_ids.max()) + 1)
    got, st = _search(ix, Q, k, ix.nlist, **kw)
    want = oracle.OracleIndex.from_data(ix).search(Q, k=k, nprobes=ix.nlist, nthreads=8, **kw)
    assert same_result(got, want)
    assert st["queries"] == len(Q), st
    if mode not in NO_PROOF.get(case, ()):
        assert st["flagged_queries"] < len(Q), st                              # the filter proved some queries itself


def test_scale_metamorphic_l2(monkeypatch):
    """Index and queries times 2^j: the oracle's distances scale by exactly 4^j, the GPU's ids stay and its distances
    scale by exactly 4^j, and the dense filter flags the same number of queries at every j (the band is homogeneous).
    Unit-norm data at 768 dims, m 96, like the flagship workload; j from 2^-20 to 2^20 (small-norm data included)."""
    monkeypatch.setenv("LGPU_DENSE_FILTER", "1")
    ix0, Q0 = _random(768, 96, 20000, 256, seed=9)
    base, flagged = None, set()
    for j in (0, -20, -10, -3, -1, 3, 10, 20):
        ix, Q = scaled(ix0, Q0, 2.0 ** j)
        (gi, gd, gc), st = _search(ix, Q, 10, 4)
        oi, od, oc = oracle.OracleIndex.from_data(ix).search(Q, k=10, nprobes=4, nthreads=8)
        f = np.float32(4.0 ** j)
        if base is None:
            base = (gi, gd, oi, od)
            assert st["flagged_queries"] < len(Q) // 2, st
        assert np.array_equal(od, (base[3] * f).astype(np.float32)) and np.array_equal(oi, base[2]), j
        assert np.array_equal(gi, base[0]) and np.array_equal(gd, (base[1] * f).astype(np.float32)), j
        flagged.add(st["flagged_queries"])
    assert len(flagged) == 1, flagged


@pytest.mark.parametrize("dense", [False, True])
def test_overflowing_query_norm(dense, monkeypatch):
    """|q|^2 > FLT_MAX with finite distances (overflow_case), B x nlist < 2^16 so the coarse step is the exact SIMT
    one: every query must get the oracle's k rows, bit for bit (through the exact fix-up)."""
    if dense:
        monkeypatch.setenv("LGPU_DENSE_FILTER", "1")
    ix, Q = overflow_case()
    (gi, gd, gc), st = _search(ix, Q, 10, ix.nlist)
    want = oracle.OracleIndex.from_data(ix).search(Q, k=10, nprobes=ix.nlist, nthreads=8)
    assert (want[2] == 10).all()
    assert same_result((gi, gd, gc), want), (int(gc.min()), int(gc.max()))

"""Host restatement of the filter scan's arithmetic (lancedb_b200/csrc/tables.cu + scan3.cu, restated bit for bit in
tests/util.py: filter_bounds) checked against the oracle on the CPU: the lower bound L built from the 16-bit per-query
tables, the per-probe scalar A and the per-row constant R must bracket the oracle's exact PQ distance d*:
L - E <= d* <= L + W + E (times 0.5 for cosine), with W and E of scan_band (kernels.cuh) -- exactly the band
`band_check3_kernel` uses to prove that a shortlist contains the exact top-k.  This pins the algebra
(|r - b|^2 = |q - b|^2 + (|c|^2 - 2 q.c) + 2 b.c), the quantiser and the error budget on random data without a GPU;
tests/test_scan_band.py attacks the same band with constructed data, and the GPU parity tests check the kernels
themselves."""
import numpy as np
import pytest

import oracle
from tests.util import candidate_appends, filter_bounds, queries, random_index, row_consts

F = np.float32


def _bounds(ix, orc, q, p, R=None):
    """(L, W, E, dstar) for every row of partition p, W and E scaled by the metric's scale"""
    out, W, E, scale, bad = filter_bounds(ix, orc, q, R=R)
    assert not bad
    L, d = out[p]
    return L, F(W * scale), F(E * scale), d


def _consts(ix):
    return None if ix.metric == "dot" else [row_consts(ix, p) for p in range(ix.nlist)]


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dim,m,scale", [(768, 96, 1.0), (64, 8, 1.0), (80, 10, 1.0), (32, 8, 1e-3), (64, 4, 300.0),
                                         (24, 24, 1.0)])
def test_lower_bound_brackets_the_oracle_distance(metric, dim, m, scale):
    rng = np.random.default_rng(5)
    ix = random_index(rng, dim=dim, nlist=6, m=m, metric=metric, sizes=[40, 700, 0, 1300, 5, 257], scale=scale)
    orc = oracle.OracleIndex.from_data(ix)
    R = _consts(ix)
    worst = 0.0
    for q in queries(rng, 5, dim, scale=scale):
        for p in (0, 1, 3, 4, 5):
            L, W, E, d = _bounds(ix, orc, q, p, R)
            lo, hi = L - E, L + W + E
            assert (d >= lo).all(), (metric, p, float((lo - d).max()), float(E))
            assert (d <= hi).all(), (metric, p, float((d - hi).max()), float(E), float(W))
            if W > 0 and E < 0.01 * W:        # where the fp slack is negligible the band is tight: d* within one W of L
                worst = max(worst, float(((d - L) / W).max()))
    assert worst <= 1.02


def test_band_is_narrow_relative_to_the_spread_of_distances():
    """What makes the filter useful: W (the quantisation band) is a small fraction of the spread of the
    candidates' distances, so a 32-row shortlist almost always proves a top-10."""
    rng = np.random.default_rng(6)
    ix = random_index(rng, dim=768, nlist=4, m=96, sizes=[3000, 10, 10, 10])
    orc = oracle.OracleIndex.from_data(ix)
    q = queries(rng, 1, 768)[0]
    L, W, E, d = _bounds(ix, orc, q, 0)
    assert W + 2 * E < 0.25 * d.std()
    order = np.argsort(L, kind="stable")
    assert L[order[31]] > L[order[9]] + W + 2 * E      # the proof condition of band_check3 for k=10, kp=32


def test_candidate_lists_hold_the_exact_topk_under_any_tile_order():
    """The scanners' threshold protocol (scan3.cu, candidate mode) restated on the host: tau_q may be ANY value such that
    at least k rows seen so far have L <= tau_q (a tile's own k-th smallest, found from above by bisection; the k-th
    smallest of the list so far; a stale copy read before another tile lowered it); a tile appends its rows with
    L <= tau + W + 2E, or every row while no threshold exists.  Whatever the tile order, the staleness and the mix of
    tightening rules, the union of the appended rows must contain the exact top-k by (d*, row) -- the property that lets
    the finalize step re-score only the list."""
    rng = np.random.default_rng(8)
    ix = random_index(rng, dim=64, nlist=5, m=8, sizes=[900, 1500, 40, 2300, 700])
    orc = oracle.OracleIndex.from_data(ix)
    R = _consts(ix)
    k = 10
    for q in queries(rng, 4, 64):
        rows = []                                             # (L, d*, partition, row), band per partition
        Wm, Em = F(0), F(0)
        for p in range(5):
            L, W, E, d = _bounds(ix, orc, q, p, R)
            Wm, Em = max(Wm, W), max(Em, E)
            rows += [(float(L[r]), float(d[r]), p, r) for r in range(len(L))]
        slack = float(Wm + 2 * Em)
        truth = set(map(lambda t: (t[2], t[3]), sorted(rows, key=lambda t: (t[1], t[2], t[3]))[:k]))
        for trial in range(6):
            got = {(rows[i][2], rows[i][3]) for i in candidate_appends(np.array([r[0] for r in rows]), k, slack, rng)}
            assert truth <= got, (trial, len(got))
            assert len(got) < len(rows)                       # and the filter does filter

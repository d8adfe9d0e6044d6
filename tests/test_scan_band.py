"""The filter scan's 16-bit band (scan_band in kernels.cuh) against constructed data, on the CPU.

tests/util.py restates the table arithmetic of tables.cu and scan3.cu bit for bit (filter_bounds: fmaf chains over
(even, odd) components, the quantiser, step / base / sbound in the kernels' reduction order, |q|^2, A, R and the fmaf
epilogue).  Every construction is checked three ways:
  - bracket: every row satisfies L - E <= d* <= L + W + E (times the metric scale), d* from the C oracle;
  - consumers: the dense proof (L_(kp) > L_(k) + W + 2E) and its proven prefix, the candidate lists under any tile
    order and stale thresholds, and cand_filter's k-th key each keep the exact top-k;
  - non-vacuity: each term of the band is removed in turn where a construction needs it.
Two terms cannot be shown necessary by data.  The 1 + 2^-10 on W: E >= 2^-15 sbound always exceeds the quantiser's
rounding (a few 2^-24 qmax steps per entry), so test_quantiser_floor_is_off_by_one only shows that the floor does
cross an integer.  The underflow floor: see test_band_holds_down_to_the_underflow_range."""
import numpy as np
import pytest

import oracle
from tests.util import (F32, candidate_appends, cancellation_case, dot_cancellation_case, filter_bounds,
                        filter_tables, full_lane_case, overflow_case, quantiser_boundary_case, quantiser_crossings,
                        query_norm2, queries, random_index, row_consts, scaled)


def _all(ix, Q, nq=None, **band):
    """per query: (L, d*, id) of every row of every partition, W, E, scale, bad"""
    orc = oracle.OracleIndex.from_data(ix)
    R = None if ix.metric == "dot" else [row_consts(ix, p) for p in range(ix.nlist)]
    res = []
    for q in Q[:nq]:
        out, W, E, scale, bad = filter_bounds(ix, orc, q, R=R, **band)
        L = np.concatenate([out[p][0] for p in sorted(out)])
        d = np.concatenate([out[p][1] for p in sorted(out)])
        ids = np.concatenate([ix.row_ids[int(ix.part_offsets[p]):int(ix.part_offsets[p + 1])] for p in sorted(out)])
        res.append((L, d, ids, W, E, scale, bad))
    return res


def _violations(res):
    """rows outside [L - E, L + W + E] over every unflagged query"""
    n = 0
    for L, d, _, W, E, s, bad in res:
        if not bad:
            with np.errstate(invalid="ignore", over="ignore"):
                lo, hi = (L - F32(s * E)).astype(F32), (L + F32(s * F32(W + E))).astype(F32)
            n += int(((d < lo) | (d > hi)).sum())
    return n


def _check_consumers(res, k=10, kp=32, seed=0):
    rng = np.random.default_rng(seed)
    proven = 0
    for L, d, ids, W, E, s, bad in res:
        if bad or len(L) <= kp:
            continue
        slack = F32(s * F32(W + F32(2) * E))
        truth = set(np.lexsort((ids, d))[:k].tolist())
        # dense mode: the kp smallest (L, id); proof L_(kp) > L_(k) + slack, proven prefix L <= L_(k) + slack
        order = np.lexsort((ids, L))
        Lk, Lkp = L[order[k - 1]], L[order[kp - 1]]
        if Lkp > F32(Lk + slack):
            proven += 1
            assert truth <= set(order[:kp].tolist())
            pre = [i for i in order[:kp] if L[i] <= F32(Lk + slack)]
            assert truth <= set(pre)
        # candidate mode: any tile order / staleness, then cand_filter's k-th key of the list
        for _ in range(2):
            app = np.array(candidate_appends(L, k, float(slack), rng))
            assert truth <= set(app.tolist())
            kth = np.sort(L[app])[k - 1]
            assert truth <= set(app[L[app] <= F32(kth + slack)].tolist())
    return proven


def _cases():
    c = {}
    for metric in ("l2", "dot"):
        for m in (8, 96):
            c[f"boundary-{metric}-m{m}"] = lambda metric=metric, m=m: quantiser_boundary_case(metric, m)
    for m, dsub in ((3, 8), (5, 4), (15, 2), (17, 1), (51, 2), (85, 1), (255, 1)):
        c[f"lanes-m{m}-d{dsub}"] = lambda m=m, dsub=dsub: full_lane_case(m, dsub, rows=60)
    for off in (10.0, 100.0, 1000.0):
        c[f"cancel-{off:g}"] = lambda off=off: cancellation_case(off, n=1500, B=6)
    for j in (-56, -40, 0, 40, 60):
        c[f"scale-2^{j}"] = lambda j=j: scaled(*_random("l2", 64, 8, 1500, 6), 2.0 ** j)
    for metric in ("cosine", "dot"):
        c[f"random-{metric}"] = lambda metric=metric: _random(metric, 64, 8, 1500, 6)
    c["chain-dsub32-m96"] = lambda: _random("l2", 3072, 96, 200, 3)
    for m in (97, 192, 193, 512):
        c[f"chain-m{m}"] = lambda m=m: _random("l2", m, m, 200, 3)
    c["dot-cancel"] = lambda: dot_cancellation_case()
    return c


def _random(metric, dim, m, n, B, seed=4):
    rng = np.random.default_rng(seed)
    ix = random_index(rng, dim=dim, nlist=4, m=m, n=n, metric=metric, scale=1 / np.sqrt(dim))
    return ix, queries(rng, B, dim, scale=1 / np.sqrt(dim))


CASES = _cases()


@pytest.mark.parametrize("case", sorted(CASES))
def test_band_brackets_the_oracle_and_keeps_the_topk(case):
    """Bracket and consumers on every construction (see the constructions' docstrings in tests/util.py)."""
    ix, Q = CASES[case]()
    res = _all(ix, Q, nq=6)
    assert not all(r[6] for r in res), "every query flagged: the construction tests nothing"
    assert _violations(res) == 0
    _check_consumers(res)


def test_band_holds_down_to_the_underflow_range():
    """Random data scaled towards the subnormal range.  At 2^-56 the tables' range is ~2^-118 and the band (floor
    included) still brackets d*; below it qmax / range overflows f32 and the quantiser flags every query for the exact
    path.  So the underflow floor 2^-126 of E is not shown necessary by data: an unflagged query has a range above
    qmax 2^-128, hence E >= 2^-15 sbound >= 2^-134, within a factor 4 of the worst-case underflow error (2^-132,
    tables.cu); the floor is kept as that margin."""
    ix, Q = scaled(*_random("l2", 64, 8, 1500, 6), 2.0 ** -56)
    res = _all(ix, Q)
    assert not any(r[6] for r in res) and _violations(res) == 0
    assert all(r[6] for r in _all(*scaled(*_random("l2", 64, 8, 1500, 6), 2.0 ** -60)))


def test_band_needs_the_query_and_codebook_term():
    """dot with large, nearly orthogonal q_i and codewords (dot_cancellation_case): each entry's rounding is ~2^-24 of
    |q_i||b|, far above sbound + m.  Without 2 (|q|^2 + CB2) the band fails.  For l2 and cosine the term is not shown
    necessary here: |q_i|^2 + |b|^2 <= 5 (T + |q_i|^2), and amax >= |q|^2, so sbound + amax nearly cover it."""
    ix, Q = dot_cancellation_case()
    assert _violations(_all(ix, Q)) == 0
    assert _violations(_all(ix, Q, q_term=False)) > 0


@pytest.mark.parametrize("m", [8, 96])
def test_quantiser_floor_is_off_by_one(m):
    """The quantiser's f32 product (T - min) * f32(qmax / range) does round across integers on the boundary data: some
    entries get a code one off the exact floor (with this range f32(qmax / R) rounds up, so the code is one above it and
    L lies above the entry; rounded down, the remainder would exceed one step -- what the 1 + 2^-10 on W is for).  The
    error is far below E, which is why W's factor cannot fail on its own."""
    R = 1000 ** 2 + 17 ** 2
    code, exact = quantiser_crossings(np.arange(R + 1), R, m)
    assert (code != exact).sum() >= 20
    assert np.abs(code - exact).max() == 1


def test_band_is_homogeneous_for_l2():
    """Scaling index and queries by 2^j scales every table entry, A, R, |q|^2, step and E by exactly 4^j in the normal
    range, so the proof decisions must not change.  An absolute term (the `+ m` the band had for l2) breaks it: at
    small norms it dominates E and no query is proven."""
    ix0, Q0 = _random("l2", 768, 96, 3000, 8, seed=5)
    ref = None
    for j in (-3, -1, 0, 2, 10):
        res = _all(*scaled(ix0, Q0, 2.0 ** j))
        E = [F32(r[4]) for r in res]
        dec = []
        for L, d, ids, W, Ej, s, bad in res:
            o = np.sort(L)
            dec.append(bool(o[31] > F32(o[9] + F32(s * F32(W + F32(2) * Ej)))))
        if ref is None:
            ref = (j, E, dec)
            assert sum(dec) >= len(dec) // 2, "the unscaled data proves too few queries to compare"
        else:
            f = F32(4.0 ** (j - ref[0]))
            assert all(e == F32(e0 * f) for e, e0 in zip(E, ref[1])), j
            assert dec == ref[2], j


def test_overflowing_query_norm_is_flagged():
    """|q|^2 above FLT_MAX with finite distances (overflow_case): A = -inf would make every L -inf; the query must be
    flagged bad (exact fix-up) while its tables stay finite."""
    ix, Q = overflow_case(B=2)
    orc = oracle.OracleIndex.from_data(ix)
    for q in Q:
        assert not filter_tables(q, ix.codebook, "l2")[5]                    # the tables alone look fine
        assert np.isinf(query_norm2(q))
        out, W, E, scale, bad = filter_bounds(ix, orc, q)
        assert bad                                                           # probe_terms' check flags it
        d = np.concatenate([v[1] for v in out.values()])
        assert np.isfinite(d).all()

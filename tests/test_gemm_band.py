"""The tensor-core shortlist's error band against adversarial bf16 rounding, checked on the CPU.

gemm.cu scores S[x] = |x|^2 - 2 bf16(q).bf16(x) and every consumer relies on |S[x] - (|q - x|^2 - |q|^2)| <= E_q
(tests/util.py tc_band).  Rounding BOTH operands can cost up to ~2^-6 |q||x| per score: here components sit one f32
ulp either side of a bf16 rounding midpoint, rounded in the direction that makes the errors add, so a band that
allows for one operand's rounding only (2^-7 |q| xmax, `_one_sided_band`) is exceeded -- per score and, on the
split-support rows of tests/util.py, in each consumer's decision.  For every consumer the decision is restated in
numpy and the true top-k (true probes) must be admitted, or the query handed to the exact fix-up:
  band_check_kernel            the kp shortlist is proven iff S_(kp) > S_(k) + 2E           (flat, N >= 4096)
  sample_threshold_kernel      admit S <= (k-th smallest S of the first Ns rows) + 2E       (flat, N >= 262144)
  coarse_finish_kernel         admit S <= (k-th smallest S, bisected to within E/4) + 2E     (IVF coarse step)
  sample_kth_threshold_kernel  list = S <= (k-th smallest S of every 8th centroid) + 2E, then the above on the list
"""
import numpy as np
import pytest

from tests.util import F32, bf16, bf16_midpoint_neighbours, split_support_case, tc_band, tc_scores

DIMS = [8, 64, 72, 768, 1536]
SCALES = [1.0, 2.0 ** -9, 64.0, 1.03, 33.0, 0.002]      # powers of two, and bf16 bases just above one


def _exact(q, X):
    """|q - x|^2 - |q|^2 = |x|^2 - 2 q.x in f64"""
    X64 = X.astype(np.float64)
    return (X64 ** 2).sum(1) - 2.0 * X64 @ q.astype(np.float64)


def _one_sided_band(q, X):
    """2^-7 (1 + 2^-8) |q| xmax + 4 d 2^-24 (|q| + xmax)^2: what rounding q alone (or x alone) can cost"""
    qn = float(np.sqrt((q.astype(np.float64) ** 2).sum()))
    xmax = float(np.sqrt((X.astype(np.float64) ** 2).sum(1).max())) * 1.0001
    return 2.0 ** -7 * (1 + 2.0 ** -8) * qn * xmax + 4.0 * q.shape[0] * 2.0 ** -24 * (qn + xmax) ** 2


def _truth(q, X, k):
    ex = _exact(q, X)
    return np.lexsort((np.arange(len(ex)), ex))[:k]


def _kth(S, k):
    return np.sort(S)[k - 1]


# ---- the four consumers: True = the true top-k is admitted or the query is flagged for the exact fix-up ----
def band_check_ok(S, truth, k, kp, E):
    order = np.lexsort((np.arange(len(S)), S))
    short = order[:kp]
    proven = len(S) <= kp or S[short[kp - 1]] > S[short[k - 1]] + 2 * E
    return (not proven) or np.isin(truth, short).all()


def sample_threshold_ok(S, truth, k, ns, cap, E):
    adm = S <= _kth(S[:ns], k) + 2 * E
    return adm.sum() > cap or adm[truth].all()


def coarse_finish_ok(S, truth, k, cap, E, cols=None):
    """the bisection leaves hi in [kth, kth + E/4]: hi = kth admits least.  cols: the list's columns (list mode)"""
    cols = np.arange(len(S)) if cols is None else cols
    adm = cols[S[cols] <= _kth(S[cols], k) + 2 * E]
    return len(adm) > cap or np.isin(truth, adm).all()


def coarse_list_ok(S, truth, k, lcap, cap, E, stride=8):
    ns = len(S) // stride
    lst = np.flatnonzero(S <= _kth(S[::stride][:ns], k) + 2 * E)
    return len(lst) > lcap or coarse_finish_ok(S, truth, k, cap, E, cols=lst)


def _consumers(S, truth, k, E):
    cap_cf = max(512, 1 << int(np.ceil(np.log2(4 * k))))             # coarse_finish's candidate capacity
    return {"band_check": band_check_ok(S, truth, k, 256, E),
            "sample_threshold": sample_threshold_ok(S, truth, k, len(S) // 4, 1024, E),
            "coarse_finish": coarse_finish_ok(S, truth, k, cap_cf, E),
            "coarse_list": coarse_list_ok(S, truth, k, 1024, cap_cf, E)}


def _adversarial_rows(rng, d, n, scale, q_exact):
    """q and n rows with bf16 mantissas near 1 (the largest relative rounding error), every component one f32 ulp from
    a rounding midpoint, with the direction chosen per component: q's at random, then the sign of x_i and its rounding
    direction so that both error terms of bf16(q_i) bf16(x_i) - q_i x_i have the row's sign s (alternating).
    q_exact: q is a bf16 value itself (only the rows round, x's signs are random)."""
    def base(shape):
        m = 1.0 + rng.integers(0, 3, shape) / 128.0
        return bf16(F32(scale) * (m * rng.choice([-1.0, 1.0], shape)).astype(F32))
    qb, Xb = base(d), np.abs(base((n, d)))
    s = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)[:, None]
    qlo, qhi = bf16_midpoint_neighbours(qb)
    q = qb.astype(F32) if q_exact else np.where(rng.random(d) < 0.5, qlo, qhi).astype(F32)
    dq = np.sign(bf16(q).astype(np.float64) - q)                       # 0 when q is exact
    xs = np.where(dq != 0, s * dq, rng.choice([-1.0, 1.0], (n, d)))    # (bf16(q_i) - q_i) x_i has sign s
    Xb = (Xb * xs).astype(F32)
    xlo, xhi = bf16_midpoint_neighbours(Xb)
    away = s * np.sign(q)[None, :] * xs > 0                             # q_i (bf16(x_i) - x_i) has sign s
    return q, np.where(away, xhi, xlo).astype(F32)


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("q_exact", [False, True])
def test_per_score_band_holds_under_adversarial_rounding(d, scale, q_exact):
    """claim (1): |S[x] - (|q - x|^2 - |q|^2)| <= E_q for every row; with q rounded too, the error is beyond what
    rounding one operand can cost (the construction is adversarial), and E_q stays within 2.1x of the error"""
    rng = np.random.default_rng(d * 7 + int(q_exact))
    q, X = _adversarial_rows(rng, d, 256, scale, q_exact)
    err = np.abs(tc_scores(q, X).astype(np.float64) - _exact(q, X)).max()
    E = tc_band(q, X)
    assert err <= E
    if q_exact:
        assert err <= _one_sided_band(q, X)
    else:
        assert err > _one_sided_band(q, X)
        assert E <= 2.1 * err


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("scale", SCALES)
def test_split_support_defeats_one_sided_band(d, scale):
    """the construction is adversarial: with the one-sided band every consumer drops the true nearest row without
    flagging the query (so its tests below are not vacuous)"""
    k = 10
    q, X = split_support_case(d, scale, 4096, k)
    truth = _truth(q, X, k)
    assert truth[0] == 4095
    S = tc_scores(q, X)
    assert not any(_consumers(S, truth, k, _one_sided_band(q, X)).values())


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("scale", SCALES)
def test_split_support_consumers_admit_true_top_k(d, scale):
    k = 10
    q, X = split_support_case(d, scale, 4096, k)
    S = tc_scores(q, X)
    E = tc_band(q, X)
    assert np.abs(S.astype(np.float64) - _exact(q, X)).max() <= E
    ok = _consumers(S, _truth(q, X, k), k, E)
    assert all(ok.values()), ok


@pytest.mark.parametrize("d", [64, 768])
def test_gaussian_band_not_wider_than_one_sided(d):
    """on ordinary data the data-dependent band is about as wide as the one-sided one (the rounding errors of random
    components do not all line up): the shortlists fall back about as often as they would with it"""
    rng = np.random.default_rng(d)
    X = rng.standard_normal((2000, d)).astype(F32)
    ratio = [tc_band(q, X) / _one_sided_band(q, X) for q in rng.standard_normal((16, d)).astype(F32)]
    assert np.median(ratio) <= 0.95 and max(ratio) <= 1.05

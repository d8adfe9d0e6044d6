"""Host restatement of the coarse step at many lists (api.cu: sampled bound -> list epilogue -> finishing kernel on the
list; gemm.cu, dist.cu) checked on the CPU: with S[x] = |c_x|^2 - 2 bf16(q).bf16(c_x) (f32 accumulation of bf16
products) and E_q = 2 ((|q| + r_q) r_C + r_q cmax)(1 + 2^-10) + 4 d 2^-24 (|q| + cmax)^2, r_q = |bf16(q) - q|,
r_C = max_x |bf16(c_x) - c_x| (kernels.cuh tc_band, tests/util.py),

  (1) |S[x] + |q|^2 - d*(q, x)| <= E_q for every centroid (the band the kernels rely on), d* the oracle's distance;
  (2) thr1 = (k-th smallest S over every 8th centroid) + 2 E_q admits every true probe into the list;
  (3) thr2 = (k-th smallest S of the LIST, found to within E_q / 4 from above) + 2 E_q still does, and the k-th
      smallest of the list equals the k-th smallest of the whole row;
  (4) the re-scored set is small: a few times k, not nlist / 8.

Random centroids, centroids in tight clusters with consecutive ids (what a hierarchical trainer leaves), queries on a
centroid, and scaled data.  The GPU tests (tests/test_gpu_tensorcore.py) check the kernels' results; this pins the
algebra they implement.  tests/test_gemm_band.py puts the same steps under adversarial rounding."""
import numpy as np
import pytest

import oracle
from tests.util import queries, random_index, tc_band, tc_scores

F = np.float32
STRIDE = 8


def _check(ix, q, k):
    C = ix.centroids
    orc = oracle.OracleIndex.from_data(ix)
    qn = oracle.normalize(q) if ix.metric == "cosine" else q.astype(F)
    dstar = orc.find_partitions(qn, ix.nlist)[2].astype(np.float64)      # exact distance to every centroid
    S = tc_scores(qn, C)
    qn2 = float((qn.astype(np.float64) ** 2).sum())
    E = tc_band(qn, C)
    assert np.abs(S.astype(np.float64) + qn2 - dstar).max() <= E                      # (1)
    truth = np.lexsort((np.arange(ix.nlist), dstar))[:k]
    sample = S[::STRIDE][: ix.nlist // STRIDE]
    thr1 = np.sort(sample)[k - 1] + 2 * E
    in_list = S <= thr1
    assert in_list[truth].all()                                                        # (2)
    lst = np.sort(S[in_list])
    assert lst[k - 1] == np.sort(S)[k - 1]
    hi = lst[k - 1] + 0.25 * E                                                         # bisection stops within E / 4
    cand = in_list & (S <= hi + 2 * E)
    assert cand[truth].all()                                                           # (3)
    return int(in_list.sum()), int(cand.sum())


@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("scale", [1.0, 1e-2, 40.0])
def test_sampled_bound_and_list_threshold_hold_the_true_probes(metric, scale):
    rng = np.random.default_rng(41)
    nlist, dim, k = 2048, 96, 20
    ix = random_index(rng, dim=dim, nlist=nlist, m=8, metric=metric, sizes=np.ones(nlist, np.int64), scale=scale)
    ix.centroids[:300] = ix.centroids[0] + F(0.01 * scale) * rng.standard_normal((300, dim)).astype(F)   # one tight blob
    if metric == "cosine":
        ix.centroids /= np.linalg.norm(ix.centroids, axis=1, keepdims=True)
    qs = queries(rng, 12, dim, scale=scale)
    qs[0] = ix.centroids[5]; qs[1] = ix.centroids[1000]; qs[2] = ix.centroids[7] * F(1.001)
    listed, rescored = zip(*[_check(ix, q, k) for q in qs])
    # the list is what the sample bound costs (about k * STRIDE + band), the re-scored set what the band costs
    assert max(rescored) <= max(listed)
    assert np.median(rescored[3:]) <= 12 * k                                            # (4) random queries

"""The exact training reference (tests/train_oracle.py) on the CPU: it equals Lloyd written straight from the definition,
its sums do not depend on row order for dyadic data, and every GPU case of tests/test_gpu_train.py reaches the kernel
branch it claims to.  Also the IVF build's refusal of an all-zero row under cosine, on the torch path."""
import numpy as np
import pytest

from lancedb_b200.index import IVF_KINDS
from tests import train_oracle as T
from tests.util import bf16


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _plain_lloyd(x, c, iters):
    """max(iters, 1) Lloyd iterations, one row at a time: exact f64 distances (small-integer data and centres that are
    means of them), the lowest centre on a tie, a mean in f64 rounded to f32, empty centres kept"""
    c = [[float(v) for v in row] for row in c]
    for _ in range(max(iters, 1)):
        groups = [[] for _ in c]
        for r, row in enumerate(x):
            d = [sum((float(a) - b) ** 2 for a, b in zip(row, cc)) for cc in c]
            groups[d.index(min(d))].append(r)
        for j, g in enumerate(groups):
            if g:
                c[j] = [float(np.float32(sum(float(x[r][t]) for r in g) / len(g))) for t in range(len(x[0]))]
    return np.array(c, np.float32)


def _plain_pq_lloyd(x, cb, iters):
    m, _, dsub = cb.shape
    cb = cb.astype(np.float64)
    for _ in range(max(iters, 1)):
        new = cb.copy()
        for i in range(m):
            groups = [[] for _ in range(256)]
            for r in range(len(x)):
                sub = x[r, i * dsub:(i + 1) * dsub].astype(np.float64)
                d = [float(((sub - cb[i, j]) ** 2).sum()) for j in range(256)]
                groups[d.index(min(d))].append(r)
            for j, g in enumerate(groups):
                if g:
                    s = [sum(float(x[r, i * dsub + t]) for r in g) for t in range(dsub)]
                    new[i, j] = np.float32(np.array(s) / len(g))
        cb = new
    return cb.astype(np.float32)


def test_lloyd_equals_the_definition():
    rng = np.random.default_rng(81)
    x = rng.integers(-6, 7, (40, 4)).astype(np.float32)
    init = x[[0, 1, 2]].copy()
    for iters in (0, 1, 2):
        assert np.array_equal(_bits(T.lloyd(x, init, iters)), _bits(_plain_lloyd(x, init, iters)))


def test_pq_lloyd_equals_the_definition():
    rng = np.random.default_rng(82)
    x = rng.integers(-6, 7, (40, 4)).astype(np.float32)
    init = (rng.integers(-6, 7, (2, 256, 2)) / 2).astype(np.float32)
    init[:, 5] = init[:, 3]                                     # a tie: code 5 stays unused
    for iters in (1, 2):
        assert np.array_equal(_bits(T.pq_lloyd(x, init, iters)), _bits(_plain_pq_lloyd(x, init, iters)))


def test_lloyd_keeps_empty_centres_and_skips_non_finite_rows():
    rng = np.random.default_rng(83)
    x = rng.standard_normal((200, 8)).astype(np.float32)
    init = x[:5].copy()
    init[3] = 1e4
    want = T.lloyd(x, init, 2)
    assert np.array_equal(_bits(want[3]), _bits(init[3]))
    bad = x.copy()
    bad[17, 2] = np.nan
    bad[18, 0] = np.inf
    assert np.array_equal(_bits(T.lloyd(bad, init, 2)), _bits(T.lloyd(np.delete(x, [17, 18], 0), init, 2)))


def test_sums_start_from_positive_zero():
    """The kernels accumulate from +0.0: a coordinate that is -0.0 in every row of a cluster averages to +0.0"""
    x = np.array([[-0.0, 1.0], [-0.0, 3.0], [5.0, 5.0]], np.float32)
    c = T.lloyd(x, x[[0, 2]], 1)
    assert _bits(c[0]).tolist() == _bits(np.array([0.0, 2.0], np.float32)).tolist()
    assert np.array_equal(_bits(c), _bits(_plain_lloyd(x, x[[0, 2]], 1)))
    cb = np.zeros((1, 256, 2), np.float32)
    cb[0, 1] = [-0.0, 9.0]
    got = T.pq_lloyd(np.array([[-0.0, 8.0], [-0.0, 9.0]], np.float32), cb, 1)
    assert _bits(got[0, 1]).tolist() == _bits(np.array([0.0, 8.5], np.float32)).tolist()


@pytest.mark.parametrize("name", ["chunks", "big_clusters", "dyadic_fine"])
def test_lloyd_on_dyadic_data_does_not_depend_on_row_order(name):
    """Permuting the rows changes no cluster (a row's centre does not depend on the other rows) but reorders every
    cluster's sum: on dyadic data not a bit changes, which is what lets the GPU sum large clusters in any order."""
    x, init, iters = T.kmeans_case(name)
    perm = np.random.default_rng(84).permutation(len(x))
    assert np.array_equal(_bits(T.lloyd(x[perm], init, iters)), _bits(T.lloyd(x, init, iters)))


@pytest.mark.parametrize("name", ["d64m16", "d768m96", "unused"])
def test_pq_lloyd_on_dyadic_data_does_not_depend_on_row_order(name):
    x, cb, iters, _ = T.pq_case(name)
    perm = np.random.default_rng(85).permutation(len(x))
    assert np.array_equal(_bits(T.pq_lloyd(x[perm], cb, iters)), _bits(T.pq_lloyd(x, cb, iters)))


def _is_dyadic(x):
    return bool(np.all(np.abs(x) <= 8) and np.all(np.round(x * 1024) == x * 1024))


@pytest.mark.parametrize("name", list(T.KMEANS_CASES))
def test_kmeans_case_reaches_its_branch(name):
    x, init, iters = T.kmeans_case(name)
    claims = T.KMEANS_CASES[name][1]
    n, dim = x.shape
    k = init.shape[0]
    trace = []
    out = T.lloyd(x, init, iters, trace)
    counts = np.stack([c for _, c in trace])                     # [iterations, k]
    assert len(trace) == max(iters, 1) and dim <= T.KM_MAX_DIM and np.isfinite(x).all()
    # bit-exactness: a cluster the GPU sums in atomic order needs dyadic data
    big = bool((counts > T.KM_SORT_MAX).any())
    assert big == ("big" in claims)
    if big:
        assert _is_dyadic(x)
    assert T.tensor_core_assignment(dim, k) == ("tc" in claims)
    if "exact" in claims:
        assert not T.tensor_core_assignment(dim, k)
    assert (dim > T.KM_THREADS) == ("dpt" in claims)
    assert (n > T.assign_chunk_rows(k)) == ("chunks" in claims)
    assert (k > 1024) == ("scan2" in claims)
    assert bool((counts == 0).any()) == ("empty" in claims)
    never = np.nonzero((counts == 0).all(axis=0))[0]
    assert np.array_equal(_bits(out[never]), _bits(init[never]))  # a centre no row reached is kept bit for bit
    if "tie" in claims:
        twins = [(i, j) for i in range(k) for j in range(i + 1, k) if np.array_equal(init[i], init[j])]
        assert twins and all(counts[0, i] > 0 and counts[0, j] == 0 for i, j in twins)
    assert (k > n) == ("k>n" in claims)
    assert (n == 1) == ("n=1" in claims)
    if "ragged" in claims:
        assert n % 256 != 0
    if "bf16" in claims:
        assert np.array_equal(bf16(x), x) and np.array_equal(bf16(init), init)
    if name == "dyadic_fine":
        assert _is_dyadic(x) and not np.array_equal(bf16(x), x)
    assert (iters == 0) == ("iters0" in claims)


@pytest.mark.parametrize("name", list(T.PQ_CASES))
def test_pq_case_reaches_its_branch(name):
    x, cb, iters, m = T.pq_case(name)
    n, dim = x.shape
    assert _is_dyadic(x) and cb.shape == (m, 256, dim // m) and dim // m in T.PQ_DSUB
    trace = []
    out = T.pq_lloyd(x, cb, iters, trace)
    used = np.zeros((m, 256), bool)
    for codes in trace:
        for i in range(m):
            used[i, codes[:, i]] = True
    assert np.array_equal(_bits(out[~used]), _bits(cb[~used]))
    if name == "unused":
        assert n < 256 and (~used).any()
    if name == "tie":
        assert np.array_equal(cb[:, 200], cb[:, 9])
        assert (trace[0] == 9).any(axis=0).all() and not (trace[0] == 200).any()


def test_pq_cases_cover_every_sub_vector_length():
    assert {T.pq_case(n)[0].shape[1] // T.pq_case(n)[3] for n in T.PQ_CASES} == set(T.PQ_DSUB)


@pytest.mark.parametrize("kind", [k for k, v in IVF_KINDS.items() if "cosine" in v.metrics])
def test_cosine_training_refuses_an_all_zero_row(kind):
    """An all-zero row has no direction: under cosine its distance to every centroid is NaN, so it has no partition.
    The torch build refuses it by index, as the accelerator build does (tests/test_gpu_train.py); l2 indexes it."""
    rng = np.random.default_rng(87)
    x = rng.standard_normal((300, 16)).astype(np.float32)
    x[11] = 0
    train = IVF_KINDS[kind].train
    with pytest.raises(ValueError, match=r"vector 11 has norm 0"):
        train(x, num_partitions=4, distance_type="cosine", max_iterations=2)
    x[11] = np.float32(1e-30)                                   # squares underflow to 0: no direction either
    with pytest.raises(ValueError, match=r"vector 11 has norm 0"):
        train(x, num_partitions=4, distance_type="cosine", max_iterations=2)
    x[11] = 0
    data = train(x, num_partitions=4, distance_type="l2", max_iterations=2)
    assert getattr(data, "sq", data).row_ids.size == 300

"""NaN, infinite and overflowing values in stored rows, centroids, codebooks, raw vectors and queries, on every float
search route, against the oracle run on the same arrays: ids and counts exact, distances bit for bit.

The contract (DESIGN.md section 0, rules a-d): a NaN _distance is never returned; +-inf distances are ordinary values,
ordered by (_distance, _rowid); a partition whose coarse distance is NaN is never probed; a tensor-core shortlist or
threshold whose bf16 error band is not finite gives way to the exact kernels (per operand at open time, per query at
search time).  Each case also checks which route ran, by kernel launch counts."""
import numpy as np
import pytest

import oracle
from lancedb_b200 import _native
from tests import pq4_oracle, rq_oracle, sq_oracle
from tests.pq4_oracle import random_pq4_index
from tests.rq_oracle import random_rq_index
from tests.sq_oracle import random_sq_index
from tests.util import queries, random_index

pytestmark = pytest.mark.gpu

FMAX = float(np.finfo(np.float32).max)
INF = float("inf")
# stored-row components: NaN, +inf, -inf, 2e19 (|x|^2 overflows, the row stays finite), +-FLT_MAX (bf16 rounds it to
# inf)
ROW_VALUES = [np.nan, INF, -INF, 2e19, FMAX, -FMAX]


def _same(got, want, what):
    gi, gd, gc = got
    oi, od, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ {gc} vs {oc}"
    assert np.array_equal(gi, oi), f"{what}: ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distance bits differ"


def _launches(fn):
    """the kernel launches of fn(), after a warm-up call of the same shape; returns (result, launches)"""
    fn()
    n0 = _native.kernel_launch_count()
    out = fn()
    return out, _native.kernel_launch_count() - n0


def _plant_rows(X, rows, col=1):
    """ROW_VALUES into component `col` of the given rows, in turn; the last row given is all zero (cosine: no norm)"""
    for i, r in enumerate(rows[:-1]):
        X[r, col] = ROW_VALUES[i % len(ROW_VALUES)]
    X[rows[-1]] = 0.0
    return X


def _queries(rng, B, dim):
    """B queries: random rows first, then the values that turn an infinite band into NaN (bf16-exact: zeros, small
    integers) and the non-finite ones"""
    q = queries(rng, B, dim)
    q[1] = 0.0
    q[2] = rng.integers(-3, 4, dim).astype(np.float32)
    q[3] = 0.5
    q[4, 2] = np.nan
    q[5, 2] = INF
    q[6, 2] = -INF
    q[7, 2] = 2e19
    if B > 8:
        q[8, 2] = FMAX
        q[9] = INF
    return q


# ------------------------------------------------------------------------------------------------ flat search
def _flat(X, q, metric, k=10, **kw):
    fl = _native.GpuFlat(X)
    try:
        got, launches = _launches(lambda: fl.search(q, k=k, metric=metric, **kw))
        simt = _launches(lambda: fl.search(q, k=k, metric=metric, lower=-INF))[1]   # a range: the exact kernels
    finally:
        fl.close()
    want = oracle.flat_search(X, q, k=k, metric=metric, nthreads=8, **kw)
    return got, want, launches, simt


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_flat_simt_nonfinite_rows_and_queries(metric):
    rng = np.random.default_rng(501)
    X = _plant_rows(queries(rng, 3000, 12), [0, 17, 18, 400, 1999, 2998, 2999])
    X[100:140] = X[17]                                     # ties at +inf: ordered by row id
    got, want, launches, simt = _flat(X, _queries(rng, 16, 12), metric)
    _same(got, want, f"flat simt {metric}")
    assert launches == simt


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_flat_tc_dense_nonfinite_rows_take_the_exact_kernels(metric):
    """N = 8192, B = 16, d = 64: the dense tensor-core shortlist for a finite column; a column with a non-finite or
    overflowing row has no finite error band, so the handle is served by the exact kernels"""
    rng = np.random.default_rng(502)
    X = queries(rng, 8192, 64)
    q = _queries(rng, 16, 64)
    got, want, tc, simt = _flat(X, q, metric)
    _same(got, want, f"flat tc dense finite {metric}")
    assert (tc != simt) == (metric == "l2"), (tc, simt)         # finite l2: the tensor-core route ran
    for value in ROW_VALUES:
        Xp = X.copy()
        Xp[[5, 4000], 9] = value
        got, want, launches, simt = _flat(Xp, q, metric)
        _same(got, want, f"flat tc dense {metric} row value {value}")
        assert launches == simt, (value, launches, simt)


def test_flat_tc_dense_mostly_nonfinite_column():
    """more than N - kp rows hold an inf: the shortlist select drops their NaN scores, so a count below kp proves
    nothing there (the column takes the exact kernels)"""
    rng = np.random.default_rng(503)
    X = queries(rng, 8192, 64)
    X[:8100, 0] = INF
    q = _queries(rng, 16, 64)
    q[:, 0] = 0.0                                          # 0 * inf = NaN scores, exact distance +inf
    got, want, launches, simt = _flat(X, q, "l2", k=100)   # 92 finite rows, then the inf rows by id
    _same(got, want, "flat tc dense, 8100 inf rows")
    assert launches == simt


def test_flat_tc_nonfinite_queries_take_the_fixup():
    """finite column, non-finite queries: the tensor-core route runs and flags those queries for the exact fix-up"""
    rng = np.random.default_rng(504)
    for N, d in ((8192, 64), (262144, 16)):
        X = queries(rng, N, d)
        q = _queries(rng, 16, d)
        got, want, launches, simt = _flat(X, q, "l2")
        _same(got, want, f"flat tc N={N} non-finite queries")
        finite = _flat(X, queries(rng, 16, d), "l2")
        assert launches == finite[2] != simt


@pytest.mark.parametrize("where", ["sample", "rest", "both"])
def test_flat_tc_filtered_one_inf_row(where):
    """N = 262144, d = 16, B = 16: the filtered tensor-core path samples the first 65536 rows.  One inf row made the
    band 0 * inf = NaN for a bf16-exact query (all zero, small integers), the threshold NaN and the result empty."""
    rng = np.random.default_rng(505)
    X = queries(rng, 262144, 16)
    rows = {"sample": [70], "rest": [200000], "both": [3, 65535, 65536, 262143]}[where]
    for i, r in enumerate(rows):
        X[r, 5] = [INF, np.nan, -INF, 2e19][i % 4]
    q = _queries(rng, 16, 16)
    q[10] = 0.0
    q[11] = 2.0
    got, want, launches, simt = _flat(X, q, "l2")
    _same(got, want, f"flat tc filtered, non-finite rows in {where}")
    assert launches == simt


def test_flat_distance_range_with_infinite_bounds():
    """[lower, upper) with infinite bounds applies as written: lower = -inf keeps every distance that is not NaN, upper =
    +inf drops the +inf distances"""
    rng = np.random.default_rng(506)
    X = _plant_rows(queries(rng, 2000, 12), [0, 10, 11, 12, 13, 14, 15])
    q = _queries(rng, 16, 12)
    for lower, upper in ((-INF, INF), (-INF, None), (None, INF), (0.5, INF), (INF, None), (-INF, -INF)):
        got, want, _, _ = _flat(X, q, "l2", k=20, lower=lower, upper=upper)
        _same(got, want, f"flat range [{lower}, {upper})")


def test_flat_finite_launch_counts_are_unchanged():
    """finite data: the routes and launch counts of the tensor-core paths (dense and filtered) and of the exact kernels"""
    rng = np.random.default_rng(507)
    counts = []
    for N, d in ((8192, 64), (262144, 16)):
        X = queries(rng, N, d)
        got, want, tc, simt = _flat(X, queries(rng, 16, d), "l2")
        _same(got, want, f"flat finite N={N}")
        counts += [tc, simt]
    assert counts == FLAT_LAUNCHES, counts


# kernel launches of one host call on finite data, as the code before non-finite inputs were handled made them:
# flat [tc dense, exact, tc filtered, exact]; IVF_PQ filter scan; IVF_SQ
FLAT_LAUNCHES = [8, 2, 10, 2]
IVF_PQ_LAUNCHES = 22
IVF_SQ_LAUNCHES = 10


# ------------------------------------------------------------------------------------------------ IVF_PQ
def _pq_index(metric, rng, nlist=64, n=20000, dim=64, m=8, bits=8):
    if bits == 4:
        ix = random_pq4_index(rng, n=n, dim=dim, nlist=nlist, m=m, metric=metric, with_vectors=True, empty=())
    else:
        ix = random_index(rng, dim=dim, nlist=nlist, m=m, n=n, metric=metric, with_vectors=True)
    return ix


def _plant_centroids(ix):
    ix.centroids[3, 7] = np.nan
    ix.centroids[5, 7] = INF
    ix.centroids[9, 1] = -INF
    return ix


def _pq_search(ix, q, env, monkeypatch, **kw):
    for var, value in env.items():
        monkeypatch.setenv(var, value)
    gpu = _native.GpuIvfPq(ix)
    try:
        got, launches = _launches(lambda: gpu.search(q, **kw))
    finally:
        gpu.close()
        for var in env:
            monkeypatch.delenv(var)
    if ix.num_bits == 4:
        want = pq4_oracle.search(ix, q, nthreads=8, **kw)
    else:
        want = oracle.OracleIndex.from_data(ix).search(q, nthreads=8, **kw)
    return got, want, launches


# scan: (batch, environment); the suite's conftest switches the small path off, "small" switches it back on
SCANS = {
    "filter_candidate": (64, {}),
    "filter_dense": (64, {"LGPU_DENSE_FILTER": "1"}),
    "exact": (64, {"LGPU_EXACT_SCAN": "1"}),
    "small": (2, {"LGPU_SMALL_SLOTS": "1024"}),
}
SMALL_MAX_LAUNCHES = 7          # coarse distances, select, small scan, select (+ refine: pair distances, select;
                                # + cosine: normalise); the batched pipeline makes 20 or more


def _pq_case(ix, q, scan, route, monkeypatch, what, **kw):
    """one request against the oracle, and the scan route it took: "filter" (the filter scan: a launch count unlike the
    exact scan's on the same request), "exact" (the exact scan's count) or "small" (at most SMALL_MAX_LAUNCHES)"""
    B, env = SCANS[scan]
    got, want, launches = _pq_search(ix, q, env, monkeypatch, **kw)
    _same(got, want, what)
    exact = _pq_search(ix, q, SCANS["exact"][1], monkeypatch, **kw)[2]
    if route == "small":
        assert launches <= SMALL_MAX_LAUNCHES, (what, launches)
    elif route == "exact":
        assert launches == exact, (what, launches, exact)
    else:
        assert launches != exact and launches > SMALL_MAX_LAUNCHES, (what, launches, exact)
    return got


def _scan_queries(rng, scan, dim):
    B = SCANS[scan][0]
    return _queries(rng, B, dim) if B >= 8 else np.stack([_queries(rng, 16, dim)[i] for i in (5, 10)])


KWS = (dict(k=10, nprobes=8), dict(k=5, nprobes=8, refine_factor=4))


@pytest.mark.parametrize("scan", sorted(SCANS))
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq_finite_index_nonfinite_queries(metric, scan, monkeypatch):
    """finite centroids and codebook, the non-finite and bf16-exact queries: every scan keeps its route (the filter
    scan hands a query whose tables are not finite to its exact fix-up)"""
    rng = np.random.default_rng(509)
    ix = _pq_index(metric, rng)
    q = _scan_queries(rng, scan, ix.dim)
    route = {"small": "small", "exact": "exact"}.get(scan, "filter")
    for kw in KWS:
        _pq_case(ix, q, scan, route, monkeypatch, f"IVF_PQ {metric} {scan} {kw}", **kw)


@pytest.mark.parametrize("scan", sorted(SCANS))
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq_nonfinite_centroids_and_codeword(metric, scan, monkeypatch):
    """a NaN centroid is never probed; +-inf centroids are (l2: every distance in them is inf; dot: the residual-free
    distances stay finite).  Under l2 / cosine such a centroid made the filter scan's band (max |2 b.c| over the rows)
    NaN for every query: no row was admitted and none was redone, so the index now takes the exact scan.  Dot has no
    such term and keeps the filter scan; an inf codeword (CB2 = inf) sends every metric to the exact scan.  The small
    path has no band and keeps its route."""
    rng = np.random.default_rng(510)
    ix = _plant_centroids(_pq_index(metric, rng))
    q = _scan_queries(rng, scan, ix.dim)
    q[0] = ix.centroids[5] if metric != "cosine" else q[0]        # a query whose nearest centroid is infinite
    for codeword in (False, True):
        if codeword:
            ix.codebook[1, 7, 2] = INF
        route = "small" if scan == "small" else ("filter" if scan != "exact" and metric == "dot" and not codeword
                                                 else "exact")
        for kw in KWS:
            _pq_case(ix, q, scan, route, monkeypatch, f"IVF_PQ {metric} {scan} {kw} inf codeword {codeword}", **kw)


@pytest.mark.parametrize("scan", ["filter_candidate", "filter_dense", "small"])
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_ivf_pq_overflowing_centroid(metric, scan, monkeypatch):
    """a finite centroid whose |c|^2 overflows (a 2e19 component): CB2 and max |2 b.c| stay finite, so the filter scan
    still runs, while a query near that centroid has residuals whose squares overflow"""
    rng = np.random.default_rng(516)
    ix = _pq_index(metric, rng)
    ix.centroids[11, 7] = 2e19
    q = _scan_queries(rng, scan, ix.dim)
    q[0, 7] = 1.5e19                                                # nearest to centroid 11, |q|^2 ~ 2.3e38
    q[-1] = ix.centroids[11]
    for kw in KWS:
        _pq_case(ix, q, scan, "small" if scan == "small" else "filter", monkeypatch,
                 f"IVF_PQ {metric} {scan} {kw} 2e19 centroid", **kw)


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq4_nonfinite_centroids_and_queries(metric, monkeypatch):
    """the 4-bit scan (its only route) with non-finite centroids and queries: the launches of the same request on the
    finite index"""
    rng = np.random.default_rng(511)
    ix = _pq_index(metric, rng, m=8, bits=4)
    q = _queries(rng, 32, ix.dim)
    finite = [_pq_search(ix, q, {}, monkeypatch, **kw)[2] for kw in KWS]
    _plant_centroids(ix)
    for kw, n in zip(KWS, finite):
        got, want, launches = _pq_search(ix, q, {}, monkeypatch, **kw)
        _same(got, want, f"4-bit IVF_PQ {metric} {kw}")
        assert launches == n, (kw, launches, n)


@pytest.mark.parametrize("variant", ["tc_dense", "tc_list"])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_tc_coarse_nonfinite(metric, variant, monkeypatch):
    """nlist = 1024: the tensor-core coarse step (dense scores, or the sampled-threshold list).  A non-finite query made
    its threshold NaN: no probe was admitted and no redo flagged.  A non-finite centroid, or one whose |c|^2 overflows,
    leaves the index on the exact coarse kernels."""
    rng = np.random.default_rng(512)
    ix = random_index(rng, dim=64, nlist=1024, m=8, n=60000, metric=metric, with_vectors=True)
    B = 16 if variant == "tc_dense" else 64
    env = {"LGPU_FORCE_TC_COARSE": "1"}
    if variant == "tc_list":
        env["LGPU_COARSE_LIST_MIN"] = "1024"
    kw = dict(k=10, nprobes=20)
    q = _queries(rng, B, 64)
    got, want, launches = _pq_search(ix, q, env, monkeypatch, **kw)
    _same(got, want, f"tc coarse {variant} {metric}, non-finite queries")
    finite = _pq_search(ix, queries(rng, B, 64), env, monkeypatch, **kw)
    exact = _pq_search(ix, queries(rng, B, 64), {}, monkeypatch, **kw)
    _same(*finite[:2], "finite control")
    assert launches == finite[2] != exact[2], (launches, finite[2], exact[2])     # the tensor-core coarse step ran
    base = ix.centroids.copy()
    for plant in ("nonfinite", "overflow"):
        ix.centroids[:] = base
        if plant == "nonfinite":
            _plant_centroids(ix)
        else:
            ix.centroids[11, 7] = 2e19
        got, want, launches = _pq_search(ix, q, env, monkeypatch, **kw)
        _same(got, want, f"tc coarse {variant} {metric}, {plant} centroids")
        assert launches == _pq_search(ix, q, {}, monkeypatch, **kw)[2], plant     # the exact coarse kernels


@pytest.mark.parametrize("scan", sorted(SCANS))
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_ivf_pq_refine_over_nonfinite_raw_vectors(metric, scan, monkeypatch):
    """refine_factor re-ranks on the raw vectors: a NaN exact distance is dropped, +-inf ones are ordered by id.  The raw
    vectors do not change the route: the scan's own, and refine's two launches on top of the request without it"""
    rng = np.random.default_rng(513)
    ix = _pq_index(metric, rng)
    bad = rng.choice(ix.vectors.shape[0], 3000, replace=False)
    for i, r in enumerate(bad):
        ix.vectors[r, i % ix.dim] = ROW_VALUES[i % len(ROW_VALUES)]
    B = SCANS[scan][0]
    q = _queries(rng, B, ix.dim) if B >= 8 else queries(rng, B, ix.dim)
    route = {"small": "small", "exact": "exact"}.get(scan, "filter")
    got = _pq_case(ix, q, scan, route, monkeypatch, f"refine {metric} {scan}", k=10, nprobes=16, refine_factor=8)
    assert not np.isnan(got[1]).any()
    plain = _pq_search(ix, q, SCANS[scan][1], monkeypatch, k=80, nprobes=16)[2]
    with_refine = _pq_search(ix, q, SCANS[scan][1], monkeypatch, k=10, nprobes=16, refine_factor=8)[2]
    assert with_refine > plain, (with_refine, plain)


def test_ivf_pq_widening_after_nan_probes(monkeypatch):
    """maximum_nprobes under a prefilter: a query whose NaN centroids leave it fewer than nprobes probes is widened
    over the partitions that have a distance (the widening pass runs: more launches than without it)"""
    rng = np.random.default_rng(514)
    ix = _pq_index("dot", rng, nlist=32, n=16000)
    ix.centroids[::3, 4] = np.nan                          # a third of the partitions is never probed
    n = int(ix.row_ids.size)
    allow = oracle.allow_bitmap(np.sort(rng.choice(n, n // 50, replace=False)), n)
    q = _queries(rng, 16, ix.dim)
    launches = {}
    for name, kw in (("narrow", dict(nprobes=2)), ("widened", dict(nprobes=2, max_nprobes=32)),
                     ("all", dict(nprobes=32))):
        got, want, launches[name] = _pq_search(ix, q, {}, monkeypatch, k=10, allow=allow, allow_bits=n, **kw)
        _same(got, want, f"widening {kw}")
    assert launches["widened"] > launches["narrow"], launches


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_inf_query_is_answered_as_the_oracle_answers_it(metric, monkeypatch):
    """the all-inf query of test_gpu_api's NaN / Inf test, asserted: l2 returns the k rows of the first probes by
    partition id at distance +inf; dot (inf - inf) and cosine (inf / inf) have no distance and return nothing"""
    rng = np.random.default_rng(31)
    ix = random_index(rng, dim=64, nlist=12, m=8, metric=metric, n=3000)
    q = queries(rng, 6, 64)
    q[4, :] = INF
    q[5, :] = -INF
    got, want, _ = _pq_search(ix, q, {}, monkeypatch, k=5, nprobes=4)
    _same(got, want, f"inf query {metric}")
    if metric == "l2":
        assert got[2][4] == 5 and np.all(np.isposinf(got[1][4]))


def test_ivf_finite_launch_counts_are_unchanged(monkeypatch):
    rng = np.random.default_rng(515)
    ix = _pq_index("l2", rng)
    got, want, launches = _pq_search(ix, queries(rng, 64, ix.dim), {}, monkeypatch, k=10, nprobes=8)
    _same(got, want, "finite IVF_PQ")
    assert launches == IVF_PQ_LAUNCHES, launches
    six = random_sq_index(rng, n=8000, dim=48, nlist=32)
    got, want, launches = _sq_search(six, queries(rng, 40, 48), k=10, nprobes=4)
    _same(got, want, "finite IVF_SQ")
    assert launches == IVF_SQ_LAUNCHES, launches


# ------------------------------------------------------------------------------------------------ IVF_SQ, IVF_RQ
def _sq_search(ix, q, **kw):
    gpu = _native.GpuIvfSq(ix)
    try:
        got, launches = _launches(lambda: gpu.search(q, **kw))
    finally:
        gpu.close()
    return got, sq_oracle.search(ix, q, nthreads=8, **kw), launches


def _rq_search(ix, q, **kw):
    gpu = _native.GpuIvfRq(ix)
    try:
        got, launches = _launches(lambda: gpu.search(q, **kw))
    finally:
        gpu.close()
    return got, rq_oracle.search(ix, q, nthreads=8, **kw), launches


@pytest.mark.parametrize("kind", ["sq", "rq"])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_ivf_sq_rq_nonfinite(kind, metric):
    rng = np.random.default_rng(520)
    make, search = (random_sq_index, _sq_search) if kind == "sq" else (random_rq_index, _rq_search)
    ix = make(rng, n=8000, dim=48, nlist=32, metric=metric, empty=())
    q = _queries(rng, 40, 48)
    kws = (dict(k=10, nprobes=6), dict(k=5, nprobes=6, refine_factor=4))
    finite = [search(ix, q, **kw)[2] for kw in kws]
    ix.centroids[3, 7] = np.nan
    ix.centroids[5, 7] = INF
    for i, r in enumerate(rng.choice(ix.vectors.shape[0], 800, replace=False)):
        ix.vectors[r, i % ix.dim] = ROW_VALUES[i % len(ROW_VALUES)]
    for kw, n in zip(kws, finite):                         # the kind's scan, as on the finite index
        got, want, launches = search(ix, q, **kw)
        _same(got, want, f"IVF_{kind.upper()} {metric} {kw}")
        assert launches == n, (kw, launches, n)


# ------------------------------------------------------------------------------------------------ multivector
def _mv(values, off, q, qoff, k=10):
    """(result, oracle, last_filter_stats) of a multivector search; stats[1] = rows scored exactly (B x nrows on the
    exact path)"""
    from tests.multivec_oracle import flat_search_mv
    mv = _native.GpuMultivec(values, off)
    _native.set_profiling(True)
    try:
        got = mv.search(q, k=k, q_offsets=qoff)
        st = _native.last_filter_stats()
    finally:
        _native.set_profiling(False)
        mv.close()
    return got, flat_search_mv(values, off, q, qoff, k=k, nthreads=8), st


def test_multivector_nonfinite_stored_vectors():
    """a column of >= 65536 stored vectors (dim 48) takes the tensor-core MaxSim shortlist when every vector is finite
    with a finite norm; a +-inf, +-FLT_MAX or 2e19 component (an infinite norm: cosine 0 * inf or inf / inf) sends the
    whole column to the exact kernels, which must then agree with the oracle bit for bit"""
    from tests.multivec_oracle import offsets_of
    rng = np.random.default_rng(540)
    lens = rng.integers(0, 9, 20000)
    off = offsets_of(lens)
    x = rng.standard_normal((int(off[-1]), 48)).astype(np.float32)
    assert x.shape[0] >= 65536
    qoff = offsets_of([1, 5, 32])
    q = rng.standard_normal((int(qoff[-1]), 48)).astype(np.float32)
    rows = lens.size
    got, want, st = _mv(x, off, q, qoff)
    _same(got, want, "multivector, finite")
    assert st["rescored"] < 3 * rows, st                    # the tensor-core shortlist ran
    near = int(off[int(np.argmax(lens > 0))])               # a vector of the first non-empty row, and one far on
    for value in [INF, -INF, FMAX, -FMAX, 2e19]:
        xp = x.copy()
        xp[[near, x.shape[0] - 3], 5] = value
        got, want, st = _mv(xp, off, q, qoff, k=30)
        _same(got, want, f"multivector, stored component {value}")
        assert st["rescored"] == 3 * rows, (value, st)      # the exact kernels scored every row


# ------------------------------------------------------------------------------------------------ index build
@pytest.mark.parametrize("index_type", ["IVF_PQ", "IVF_SQ", "IVF_RQ"])
def test_create_index_refuses_nonfinite_rows_on_the_gpu(index_type):
    import lancedb_b200 as lancedb
    rng = np.random.default_rng(530)
    x = rng.standard_normal((3000, 32)).astype(np.float32)
    x[1234, 5] = np.nan
    x[2000, 1] = INF
    t = lancedb.connect("memory://").create_table("t", {"vector": list(x), "id": np.arange(3000)})
    kw = dict(num_bits=1) if index_type == "IVF_RQ" else {}
    with pytest.raises(ValueError, match="vector 1234 "):
        t.create_index(metric="l2", num_partitions=8, num_sub_vectors=4, accelerator="cuda", index_type=index_type,
                       **kw)

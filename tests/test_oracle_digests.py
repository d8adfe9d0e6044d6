"""Every C oracle search entry point and every NumPy mirror, pinned by the SHA-256 of (ids, distance bits, counts)
over a seeded case matrix: every metric a kind serves; plain, refine_factor, distance_range (finite and +-inf bounds), a
prefilter with maximum_nprobes widening, k larger than the probed rows, an empty partition; 1 and 8 threads; and NaN /
+-inf / overflowing values in queries, centroids, codebooks, rows and raw vectors.  The oracles state the search
contract (DESIGN.md section 0), so a change to any of them that moves a single bit shows up here.

The cases use only integer draws and uniform doubles of the seeded generator and element-wise f32 arithmetic, so the
digests do not depend on the host's BLAS or SIMD dispatch.  Regenerate tests/golden/oracle_digests.json with
`python -m tests.test_oracle_digests` only when the contract itself changes."""
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from lancedb_b200.index import IvfPqIndexData, IvfRqIndexData, IvfSqIndexData
from oracle import oracle_np as onp
from tests import hamming_oracle, ivf_binary_oracle, multivec_oracle, pq4_oracle, rq_oracle, sq_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_digests.json")
INF = float("inf")
f32 = np.float32
pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")      # NaN / inf arithmetic is part of the matrix


def _digest(ids, dist, cnt):
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(ids, "<u8").tobytes())
    h.update(np.ascontiguousarray(np.asarray(dist, f32).view(np.uint32), "<u4").tobytes())
    h.update(np.ascontiguousarray(cnt, "<u4").tobytes())
    return h.hexdigest()


def _f(rng, *shape, s=1.0):
    """uniform in [-s, s) as f32: the generator's doubles, one multiply-add and one rounding, no libm"""
    return ((rng.random(shape) * 2.0 - 1.0) * s).astype(f32)


def _layout(rng, n, nlist, empty):
    """(part_offsets, row_ids): n rows over the partitions not in `empty`, ids non-contiguous, ascending inside each"""
    full = np.setdiff1d(np.arange(nlist), empty)
    sizes = np.bincount(full[rng.integers(0, full.size, n)], minlength=nlist)
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    perm = rng.permutation(n).astype(np.uint64) * 3 + 7
    ids = np.concatenate([np.sort(perm[int(off[p]):int(off[p + 1])]) for p in range(nlist)])
    return off, ids


def _queries(rng, B, dim, nonfinite):
    q = _f(rng, B, dim)
    if nonfinite:
        q[1] = 0.0
        q[2, 3] = np.nan
        q[3, 0] = INF
        q[4] = INF
        q[5, 1] = 2e19
    return q


def _plant(centroids, vectors):
    centroids[1, 3] = np.nan
    centroids[2, 0] = INF
    centroids[4, 5] = -INF
    vectors[::7, 1] = np.nan
    vectors[3::7, 2] = INF
    vectors[5::11, 0] = -2e19


N, NLIST, B = 420, 6, 7


def _pq(rng, metric, nonfinite, num_bits):
    dim, m = (32, 4) if num_bits == 8 else (32, 8)
    off, ids = _layout(rng, N, NLIST, empty=[1])
    cb = _f(rng, m, 1 << num_bits, dim // m, s=0.5)
    codes_t = rng.integers(0, 256, N * m * num_bits // 8, dtype=np.uint8)
    codes_t[:3 * m * num_bits // 8] = 0                 # partition 0 starts with tied rows, ordered by row id
    ix = IvfPqIndexData(dim, NLIST, m, metric, _f(rng, NLIST, dim), cb, off, codes_t, ids, _f(rng, N, dim),
                        num_bits=num_bits)
    if nonfinite:
        _plant(ix.centroids, ix.vectors)
        ix.codebook[1, 9, 2] = INF
    return ix


def _sq(rng, metric, nonfinite):
    dim = 24
    off, ids = _layout(rng, N, NLIST, empty=[1])
    x = _f(rng, N, dim)
    codes = rng.integers(0, 256, (N, dim), dtype=np.uint8)
    codes[1:4] = codes[0]
    ix = IvfSqIndexData(dim, NLIST, metric, _f(rng, NLIST, dim), off, codes, ids, -0.9, 0.8, x)
    if nonfinite:
        _plant(ix.centroids, ix.vectors)
    return ix


def _rq(rng, metric, nonfinite):
    dim = 24
    off, ids = _layout(rng, N, NLIST, empty=[1])
    codes = rng.integers(0, 256, (N, 3), dtype=np.uint8)
    codes[1:4] = codes[0]
    ix = IvfRqIndexData(dim, NLIST, metric, _f(rng, NLIST, dim), _f(rng, dim, dim, s=0.4), off, codes,
                        (rng.random(N) * 4).astype(f32), (-rng.random(N) * 2).astype(f32), ids, _f(rng, N, dim))
    if nonfinite:
        _plant(ix.centroids, ix.vectors)
        ix.add_factors[10] = INF
    return ix


def _modes(plain_dist, max_id, rng, nlist):
    """search keyword sets; the distance range comes from query 0's plain results so that it keeps some rows"""
    d = plain_dist[0][np.isfinite(plain_dist[0])]
    lo, hi = (float(d[2]), float(d[7])) if d.size > 7 else (-1.0, 1.0)
    return {
        "plain": dict(k=10, nprobes=3),
        "refine": dict(k=5, nprobes=3, refine_factor=3),
        "range": dict(k=10, nprobes=4, lower=lo, upper=hi),
        "range_inf": dict(k=10, nprobes=4, lower=-INF, upper=INF),
        "upper_only": dict(k=10, nprobes=4, upper=hi),
        "prefilter": dict(k=10, nprobes=2, allow=rng.random(max_id + 1) < 0.03, max_nprobes=nlist),
        "prefilter_no_widening": dict(k=10, nprobes=2, allow=rng.random(max_id + 1) < 0.3),
        "big_k": dict(k=200, nprobes=2),
    }


def _pad(k, ids, dist):
    out_i = np.full(k, np.iinfo(np.uint64).max, np.uint64)
    out_d = np.full(k, np.inf, f32)
    out_i[:len(ids)] = ids
    out_d[:len(ids)] = dist
    return out_i, out_d


def _ivfpq_c(ix, q, nthreads, allow=None, **kw):
    orc = oracle.OracleIndex.from_data(ix)
    if allow is not None:
        kw.update(allow=oracle.allow_bitmap(np.nonzero(allow)[0], allow.size), allow_bits=allow.size)
    return orc.search(q, nthreads=nthreads, **kw)


def _ivfpq_np(ix, q, k, nprobes, lower=None, upper=None, allow=None):
    allowed = None if allow is None else set(np.nonzero(allow)[0].tolist())
    res = [_pad(k, *onp.ivfpq_search_one(ix, q[b], k, nprobes, lower, upper, allowed)) for b in range(len(q))]
    ids = np.stack([r[0] for r in res])
    return ids, np.stack([r[1] for r in res]), (ids != np.iinfo(np.uint64).max).sum(1).astype(np.uint32)


IVF_KINDS = {
    # kind: (metrics, index builder, C search, NumPy mirror, keywords the mirror does not take)
    "pq8": (("l2", "cosine", "dot"), lambda rng, m, nf: _pq(rng, m, nf, 8), _ivfpq_c, _ivfpq_np,
            ("refine_factor", "max_nprobes")),
    "pq4": (("l2", "cosine", "dot"), lambda rng, m, nf: _pq(rng, m, nf, 4),
            lambda ix, q, t, **kw: pq4_oracle.search(ix, q, nthreads=t, **kw), pq4_oracle.pq4_search_np, ()),
    "sq": (("l2", "cosine"), _sq, lambda ix, q, t, **kw: sq_oracle.search(ix, q, nthreads=t, **kw),
           sq_oracle.sq_search_np, ()),
    "rq": (("l2", "cosine"), _rq, lambda ix, q, t, **kw: rq_oracle.search(ix, q, nthreads=t, **kw),
           rq_oracle.rq_search_np, ()),
}


def _ivf_cases(kind):
    metrics, make, c_search, np_search, np_skip = IVF_KINDS[kind]
    out = {}
    for metric in metrics:
        for nonfinite in (False, True):
            rng = np.random.default_rng([sum(map(ord, kind)), len(metric), int(nonfinite)])
            ix = make(rng, metric, nonfinite)
            q = _queries(rng, B, ix.dim, nonfinite)
            plain = c_search(ix, q, 1, k=10, nprobes=3)
            for mode, kw in _modes(plain[1], int(ix.row_ids.max()), rng, ix.nlist).items():
                name = f"{kind}/{metric}/{'nonfinite' if nonfinite else 'finite'}/{mode}"
                for t in (1, 8):
                    out[f"{name}/c{t}"] = _digest(*c_search(ix, q, t, **kw))
                if not any(kw.get(s) for s in np_skip):
                    out[f"{name}/np"] = _digest(*np_search(ix, q, **{a: v for a, v in kw.items() if a not in np_skip}))
    return out


def _binary_ivf_cases():
    out = {}
    for patterns in (0, 12):
        rng = np.random.default_rng([5, patterns])
        ix = ivf_binary_oracle.random_index(rng, N, 8, NLIST, empty=(2,), patterns=patterns)
        q = np.concatenate([ix.vectors[:3], rng.integers(0, 256, (B - 3, 8), dtype=np.uint8)])
        plain = ivf_binary_oracle.search(ix, q, 10, 3)
        for mode, kw in _modes(plain[1], int(ix.row_ids.max()), rng, ix.nlist).items():
            kw.pop("refine_factor", None)                # refine changes nothing for exact distances
            name = f"ivf_binary/patterns{patterns}/{mode}"
            for t in (1, 8):
                out[f"{name}/c{t}"] = _digest(*ivf_binary_oracle.search(ix, q, nthreads=t, **kw))
            out[f"{name}/np"] = _digest(*ivf_binary_oracle.search_np(ix, q, **kw))
    return out


def _flat_modes(plain_dist, n, rng, row_ids):
    kws = _modes(plain_dist, int(row_ids.max()), rng, 1)
    out = {}
    for mode in ("plain", "range", "range_inf", "upper_only", "prefilter_no_widening"):
        kw = dict(kws[mode])
        kw.pop("nprobes")
        out[mode] = kw
    out["big_k"] = dict(k=n + 5)
    return out


def _flat_cases():
    out = {}
    for metric in ("l2", "cosine", "dot"):
        for nonfinite in (False, True):
            rng = np.random.default_rng([7, len(metric), int(nonfinite)])
            x = _f(rng, 300, 20)
            x[1:4] = x[0]
            rid = (rng.permutation(300) * 2 + 5).astype(np.uint64)
            if nonfinite:
                _plant(np.zeros((6, 20), f32), x)
            q = _queries(rng, B, 20, nonfinite)
            plain = oracle.flat_search(x, q, k=10, metric=metric, row_ids=rid)
            for mode, kw in _flat_modes(plain[1], 300, rng, rid).items():
                allow = kw.pop("allow", None)
                if allow is not None:
                    kw.update(allow=oracle.allow_bitmap(np.nonzero(allow)[0], allow.size), allow_bits=allow.size)
                name = f"flat/{metric}/{'nonfinite' if nonfinite else 'finite'}/{mode}"
                for t in (1, 8):
                    out[f"{name}/c{t}"] = _digest(*oracle.flat_search(x, q, metric=metric, row_ids=rid, nthreads=t,
                                                                      **kw))
    return out


def _hamming_cases():
    out = {}
    for patterns in (0, 10):
        rng = np.random.default_rng([11, patterns])
        x = rng.integers(0, 256, (500, 12), dtype=np.uint8)
        if patterns:
            x = x[rng.integers(0, patterns, 500)]
        rid = (rng.permutation(500) * 3 + 1).astype(np.uint64)
        q = rng.integers(0, 256, (B, 12), dtype=np.uint8)
        plain = hamming_oracle.flat_search_u8(x, q, 10, row_ids=rid)
        for mode, kw in _flat_modes(plain[1], 500, rng, rid).items():
            name = f"hamming/patterns{patterns}/{mode}"
            for t in (1, 8):
                out[f"{name}/c{t}"] = _digest(*hamming_oracle.flat_search_u8(x, q, row_ids=rid, nthreads=t, **kw))
            out[f"{name}/np"] = _digest(*hamming_oracle.flat_search_u8_np(x, q, row_ids=rid, **kw))
    return out


def _multivec_cases():
    out = {}
    for nonfinite in (False, True):
        rng = np.random.default_rng([13, int(nonfinite)])
        off = multivec_oracle.offsets_of(rng.integers(0, 5, 200))
        v = _f(rng, int(off[-1]), 20)
        qoff = multivec_oracle.offsets_of([1, 3, 2, 4])
        qv = _f(rng, int(qoff[-1]), 20)
        if nonfinite:
            v[::9, 1] = np.nan
            v[4::9] = INF
            v[7::13] = 0.0
            qv[2, 3] = np.nan
            qv[5] = 0.0
        rid = (rng.permutation(200) * 2 + 3).astype(np.uint64)
        plain = multivec_oracle.flat_search_mv(v, off, qv, qoff, 10, row_ids=rid)
        for mode, kw in _flat_modes(plain[1], 200, rng, rid).items():
            name = f"multivec/{'nonfinite' if nonfinite else 'finite'}/{mode}"
            for t in (1, 8):
                out[f"{name}/c{t}"] = _digest(*multivec_oracle.flat_search_mv(v, off, qv, qoff, row_ids=rid,
                                                                              nthreads=t, **kw))
            out[f"{name}/np"] = _digest(*multivec_oracle.flat_search_mv_np(v, off, qv, qoff, row_ids=rid, **kw))
    return out


FAMILIES = {"pq8": lambda: _ivf_cases("pq8"), "pq4": lambda: _ivf_cases("pq4"), "sq": lambda: _ivf_cases("sq"),
            "rq": lambda: _ivf_cases("rq"), "ivf_binary": _binary_ivf_cases, "flat": _flat_cases,
            "hamming": _hamming_cases, "multivec": _multivec_cases}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_oracle_digests(family):
    with open(GOLDEN) as fh:
        want = {k: v for k, v in json.load(fh).items() if k.split("/")[0] == family}
    got = FAMILIES[family]()
    assert sorted(got) == sorted(want)
    bad = [k for k in got if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(got)} cases changed: {bad[:10]}"


if __name__ == "__main__":
    digests = {}
    for fam in sorted(FAMILIES):
        digests.update(FAMILIES[fam]())
    with open(GOLDEN, "w") as fh:
        json.dump(digests, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print(f"{len(digests)} cases -> {GOLDEN}")

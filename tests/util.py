"""Test helpers: synthetic IVF_PQ indexes with arbitrary (untrained) contents.  Parity does
not depend on index quality -- the CUDA path and the oracle consume the identical arrays --
so random centroids / codebooks / codes exercise the arithmetic just as well and let the
tests shape edge cases (empty, tiny and multi-tile partitions)."""
import numpy as np

import oracle
from lancedb_b200.index import IvfPqIndexData


def random_index(rng, *, dim, nlist, m, metric="l2", sizes=None, n=None, with_vectors=False, scale=1.0,
                 shuffle_ids=True):
    dsub = dim // m
    if sizes is None:
        w = rng.random(nlist) + 0.2
        sizes = np.floor(w / w.sum() * n).astype(np.int64)
        sizes[0] += n - sizes.sum()
    sizes = np.asarray(sizes, np.int64)
    n = int(sizes.sum())
    cent = (rng.standard_normal((nlist, dim)) * scale).astype(np.float32)
    if metric == "cosine":
        cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cb = (rng.standard_normal((m, 256, dsub)) * 0.5 * scale).astype(np.float32)
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    codes_t = rng.integers(0, 256, size=n * m, dtype=np.uint8)
    # ascending row ids inside each partition (lance scan order), interleaved across partitions
    ids = np.empty(n, np.uint64)
    perm = rng.permutation(n).astype(np.uint64) if shuffle_ids else np.arange(n, dtype=np.uint64)
    for p in range(nlist):
        a, b = int(off[p]), int(off[p + 1])
        ids[a:b] = np.sort(perm[a:b])
    vec = None
    if with_vectors:
        vec = (rng.standard_normal((n, dim)) * scale).astype(np.float32)
    ix = IvfPqIndexData(dim, nlist, m, metric, cent, cb, off, codes_t, ids, vec)
    ix.validate()
    return ix


def queries(rng, B, dim, scale=1.0):
    return (rng.standard_normal((B, dim)) * scale).astype(np.float32)


# ---- the tensor-core shortlist's arithmetic (gemm.cu), restated for CPU checks of its error band ----
F32 = np.float32


def bf16(x):
    """round-to-nearest-even f32 -> bf16 -> f32 (gemm.cu to_bf16_norm_kernel)"""
    u = np.ascontiguousarray(x, F32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(F32).reshape(np.shape(x))


def tc_scores(q, X):
    """S[x] = |x|^2 - 2 bf16(q).bf16(x): bf16 products are exact in f32, the sum is rounded once to f32"""
    qb, Xb = bf16(q).astype(np.float64), bf16(X).astype(np.float64)
    dot = (Xb @ qb).astype(F32)
    xn2 = (X.astype(np.float64) ** 2).sum(1).astype(F32)
    return (xn2 - F32(2) * dot).astype(F32)


def tc_band(q, X):
    """E_q of gemm.cu (tc_band): |S[x] - (|q - x|^2 - |q|^2)| <= E_q for every row x of X, with
    r_q = |bf16(q) - q|, r_X = max_x |bf16(x) - x|, xmax = max_x |x|:
        E_q = 2 ((|q| + r_q) r_X + r_q xmax)(1 + 2^-10) + 4 d 2^-24 (|q| + xmax)^2"""
    q64, X64 = q.astype(np.float64), X.astype(np.float64)
    qn = float(np.sqrt((q64 ** 2).sum()))
    xmax = float(np.sqrt((X64 ** 2).sum(1).max())) * 1.0001
    rq = float(np.sqrt(((bf16(q).astype(np.float64) - q64) ** 2).sum()))
    rx = float(np.sqrt(((bf16(X).astype(np.float64) - X64) ** 2).sum(1).max()))
    return 2.0 * ((qn + rq) * rx + rq * xmax) * (1.0 + 2.0 ** -10) + 4.0 * q.shape[0] * 2.0 ** -24 * (qn + xmax) ** 2


def bf16_midpoint_neighbours(b):
    """For nonzero bf16 values b: the two f32 values one ulp either side of the midpoint between |b| and the next bf16
    magnitude, signed like b -- round-to-nearest-even takes the first to b and the second away from zero, each with
    the largest rounding error a value near b can have"""
    b = np.asarray(b, np.float64)
    e = np.floor(np.log2(np.abs(b)))
    mid = (np.abs(b) + 2.0 ** (e - 8)).astype(F32)                     # 9 significant bits: exact in f32
    s = np.sign(b).astype(F32)
    return s * np.nextafter(mid, F32(0)), s * np.nextafter(mid, F32(np.inf))


def split_support_case(d, scale, n, k, stride=8):
    """Rows on which bf16 rounding pushes the true nearest row of q out of the shortlist a band of 2^-7 |q| xmax would
    prove complete.  b = bf16(scale), lo / hi the values either side of the midpoint above b (lo rounds to b, hi up):
      q       = [lo] * h + [hi] * (d - h)                     (h = d / 2)
      rows 0, stride, .. (k decoys): [0] * h + [hi] * (d - h), one of the first h set to -b 2^-10: scored low by
        ~2^-7 |q||x| (every 8th row: the coarse step's sample is)
      row n-1 (T, the true nearest): [lo] * h + [0] * (d - h): scored high by as much
      every other row (filler): [b] * h + [-c, 0, ...], bf16-exact, c chosen so that its score lies 3/4 of the way
      from the decoys' to T's -- just under T's, far above the decoys'
    Exact order: T, the decoys by id, then the fillers.  Returns (q, X)."""
    b = bf16(F32(scale))
    lo, hi = bf16_midpoint_neighbours(b)
    h = d // 2
    q = np.concatenate([np.full(h, lo, F32), np.full(d - h, hi, F32)])
    hb = float(bf16(hi))
    r = 1.5 * h * float(b) * (float(lo) - float(b))                   # 3/4 of T's excess over [b] * h + [0] * (d - h)
    c = bf16(F32(-hb + np.sqrt(hb * hb + r)))                          # c^2 + 2 bf16(hi) c = r
    X = np.zeros((n, d), F32)
    X[:, :h] = b
    X[:, h] = -c
    dec = np.arange(k) * stride
    X[dec] = 0
    X[dec, h:] = hi
    X[dec, np.arange(k) % h] = -b * F32(2.0 ** -10)
    X[n - 1] = 0
    X[n - 1, :h] = lo
    return q, X


GOLDEN_CASES = {"plain": dict(k=7, nprobes=3), "range": dict(k=7, nprobes=3, lower=2.0, upper=30.0),
                "refine": dict(k=5, nprobes=3, refine_factor=3), "prefilter": dict(k=7, nprobes=4)}


def load_golden(metric):
    """tests/golden/ivfpq_small.npz (made by tests/golden/make_golden.py): index, queries, and per case the
    search kwargs + the committed (ids, dist, cnt)."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ivfpq_small.npz"))
    g = lambda name: z[f"{metric}_{name}"]
    ix = IvfPqIndexData(32, 8, 4, metric, g("centroids"), g("codebook"), g("part_offsets"), g("codes_t"), g("row_ids"),
                        g("vectors"))
    ix.validate()
    cases = {}
    for name, kw in GOLDEN_CASES.items():
        kw = dict(kw)
        if name == "prefilter":
            kw.update(allow=g("allow"), allow_bits=600)
        cases[name] = (kw, (g(f"{name}_ids"), g(f"{name}_dist"), g(f"{name}_cnt")))
    flat = (g("flat_ids"), g("flat_dist"), g("flat_cnt"))
    return ix, g("queries"), cases, flat


def same_result(got, want):
    gi, gd, gc = got
    wi, wd, wc = want
    return (np.array_equal(gc, wc) and np.array_equal(gi, wi)
            and np.array_equal(np.asarray(gd, np.float32).view(np.uint32), np.asarray(wd, np.float32).view(np.uint32)))


# ---- the filter scan's arithmetic (tables.cu + scan3.cu), restated bit for bit for CPU checks of its band ----
def fmaf(a, b, c):
    """f32 fused multiply-add, correctly rounded (__fmaf_rn): the f64 product of two f32 values is exact; the f64 sum is
    rounded to odd (TwoSum gives its error; an inexact sum with an even last bit moves one f64 ulp towards the exact
    value), and rounding a round-to-odd value with 29 spare bits to f32 is the correct rounding of the exact sum --
    subnormal results included, as every f32 result lies far inside f64's normal range"""
    a, b, c = (np.asarray(x, F32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    s = np.array(s, np.float64, ndmin=1)
    e = np.broadcast_to(e, s.shape)
    fix = (e != 0) & ((s.view(np.uint64) & 1) == 0) & np.isfinite(s)
    s[fix] = np.nextafter(s[fix], np.where(e[fix] > 0, np.inf, -np.inf))
    return s.astype(F32).reshape(np.broadcast(a, b, c).shape)


def pair_dot(x, y):
    """SubVec::dot: over the last axis, one fmaf chain over the even and one over the odd components, then one add"""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    shape = np.broadcast(x[..., 0], y[..., 0]).shape
    ev, od = np.zeros(shape, F32), np.zeros(shape, F32)
    for t in range(x.shape[-1]):
        if t % 2 == 0:
            ev = fmaf(x[..., t], y[..., t], ev)
        else:
            od = fmaf(x[..., t], y[..., t], od)
    return (ev + od).astype(F32)


def _warp_sum(v, op):
    """lane l folds elements l, l + 32, ... in order, then a xor butterfly (16, 8, 4, 2, 1); lane 0's value"""
    lanes = [F32(0)] * 32
    for i, x in enumerate(np.asarray(v)):
        lanes[i % 32] = op(lanes[i % 32], x)
    lanes = np.array(lanes, dtype=np.asarray(v).dtype)
    for o in (16, 8, 4, 2, 1):
        lanes = op(lanes, lanes[np.arange(32) ^ o])
    return lanes[0]


def filter_tables(q, codebook, metric):
    """qtable_minmax / qtable_quant_kernel for one query q (normalised for cosine): the f32 entries T [m, 256] of
    filter_entry, and step, base, sbound, bad and the 16-bit codes n [m, 256] of the quantiser"""
    m, _, dsub = codebook.shape
    qs = np.asarray(q, F32).reshape(m, 1, dsub)
    cb = np.asarray(codebook, F32)
    d = pair_dot(qs, cb)
    if metric == "dot":
        T = (F32(1) - d).astype(F32)
    else:
        T = fmaf(F32(-2), d, (pair_dot(qs, qs) + pair_dot(cb, cb)).astype(F32))
    with np.errstate(invalid="ignore", over="ignore"):
        mn, mx = T.min(1), T.max(1)
        rng = F32(np.max(mx - mn))
        add = lambda a, b: (np.asarray(a, F32) + np.asarray(b, F32)).astype(F32)
        base = F32(_warp_sum(mn.astype(F32), add))
        sbound = F32(_warp_sum(np.maximum(np.abs(mn), np.abs(mx)).astype(F32), add))
        bad = not (np.isfinite(T).all() and np.isfinite(rng) and np.isfinite(base) and np.isfinite(sbound))
        qmax = F32(65535 // m)
        step = F32(rng / qmax) if (not bad and rng > 0) else F32(0)
        inv = F32(qmax / rng) if (step > 0 and np.isfinite(F32(qmax / rng))) else F32(0)
        if rng > 0 and inv == 0:
            bad = True
        if bad:
            step, inv = F32(0), F32(0)
        x = ((T - mn[:, None]).astype(F32) * inv).astype(F32)
        n = np.where(x >= 0, np.minimum(np.floor(x), qmax), F32(0)).astype(np.int64)
    if metric == "dot":
        base = F32(base - F32(m - 1))
    return T, n, step, base, sbound, bad


def query_norm2(q):
    """probe_terms_kernel's |q|^2: f64 sums per lane, butterfly, rounded once to f32"""
    v = np.asarray(q, F32).astype(np.float64)
    return F32(_warp_sum(v * v, lambda a, b: np.asarray(a, np.float64) + np.asarray(b, np.float64)))


def row_consts(ix, p):
    """row_const_kernel: R = f32(2 sum_i codeword_i . c_p,i), an f64 chain in (i, t) order, for partition p"""
    m, dsub = ix.m, ix.dim // ix.m
    codes = ix.partition_codes(p).astype(np.int64)
    cw = np.asarray(ix.codebook, F32).astype(np.float64)[np.arange(m)[:, None], codes]      # [m, n_p, dsub]
    cen = np.asarray(ix.centroids[p], F32).astype(np.float64).reshape(m, dsub)
    acc = np.zeros(codes.shape[1])
    for i in range(m):
        for t in range(dsub):
            acc = acc + cw[i, :, t] * cen[i, t]
    return (2.0 * acc).astype(F32)


def codebook_cb2(codebook):
    """CB2 of api.cu: f32(1.000001 sum_i max_c |codebook_i[c]|^2), in f64"""
    cb = np.asarray(codebook, F32).astype(np.float64)
    return F32((cb * cb).sum(2).max(1).sum() * 1.000001)


def scan_band(step, sbound, amax, rmax, qn2, cb2, m, metric, w_factor=True, q_term=True, floor=True, m_term=None):
    """scan_band (kernels.cuh) in the kernels' f32 order: (W, E).  The keywords weaken it for non-vacuity checks:
    w_factor=False drops 1 + 2^-10 from W, q_term=False drops 2 (|q|^2 + CB2), floor=False drops the underflow floor;
    m_term=True adds m for every metric (the band before it was made homogeneous), False for none"""
    if m_term is None:
        m_term = metric == "dot"
    with np.errstate(over="ignore", invalid="ignore"):
        mag = F32(F32(F32(sbound) + F32(amax)) + F32(rmax))
        if q_term:
            mag = F32(mag + F32(F32(2) * F32(F32(qn2) + F32(cb2))))
        if m_term:
            mag = F32(mag + F32(m))
        W = F32(F32(m) * F32(step))
        if w_factor:
            W = F32(W * F32(1.0009765625))
        E = F32(F32(F32(3.0517578125e-5) * F32((m + 95) // 96)) * mag)
        if floor:
            E = F32(E + F32(2.0 ** -126))
    return W, E


def filter_bounds(ix, orc, q, nprobes=None, R=None, **band):
    """The dense filter scan for one query, restated: ({partition: (L, d*)}, W, E, scale, bad) over the query's probes
    (all partitions by default), with L as scan3's epilogue writes it, d* the oracle's exact PQ distance, (W, E) of
    scan_band (unscaled: the band is [L - scale E, L + scale (W + E)]) and `bad` as the table and probe kernels set it.
    R: the row_consts of every partition, if already computed; `band` weakens scan_band."""
    metric = ix.metric
    if R is None and metric != "dot":
        R = [row_consts(ix, p) for p in range(ix.nlist)]
    qn = oracle.normalize(q) if metric == "cosine" else np.asarray(q, F32)
    T, n, step, base, sbound, bad = filter_tables(qn, ix.codebook, metric)
    nprobes = ix.nlist if nprobes is None else nprobes
    parts, cd, _ = orc.find_partitions(qn, nprobes)
    qn2 = query_norm2(qn)
    scale = F32(0.5) if metric == "cosine" else F32(1)
    with np.errstate(over="ignore", invalid="ignore"):
        if metric == "dot":
            A, amax, rmax = np.zeros(len(parts), F32), F32(0), F32(0)
        else:
            A = (cd - qn2).astype(F32)
            amax = F32(F32(np.abs(cd).max()) + qn2)
            rmax = F32(max(np.abs(r).max(initial=0) for r in R))
            bad = bad or not (np.isfinite(qn2) and np.isfinite(amax) and np.isfinite((base + A).astype(F32)).all())
        out = {}
        for j, p in enumerate(parts):
            codes = ix.partition_codes(int(p)).astype(np.int64)
            S = n[np.arange(ix.m)[:, None], codes].sum(0)
            assert S.max(initial=0) <= 65535
            Rp = np.zeros(codes.shape[1], F32) if metric == "dot" else R[int(p)]
            L = ((fmaf(step, S.astype(F32), F32(base + A[j])) + Rp).astype(F32) * scale).astype(F32)
            out[int(p)] = (L, orc.partition_distances(q, int(p)))
    W, E = scan_band(step, sbound, amax, rmax, qn2, codebook_cb2(ix.codebook), ix.m, metric, **band)
    return out, W, E, scale, bad


def candidate_appends(L, k, slack, rng):
    """The scanners' threshold protocol (scan3.cu, candidate mode) over rows with lower bounds L, in a random tile
    order: tau_q may be ANY value such that at least k rows seen so far have L <= tau_q (a tile's own k-th smallest,
    found from above by bisection; the k-th smallest of the list so far; a stale copy read before another tile lowered
    it); a tile appends its rows with L <= tau + slack, or every row while no threshold exists.  Returns the indices of
    the appended rows."""
    order = rng.permutation(len(L))
    tiles = np.array_split(order, rng.integers(3, 40))
    tau, stale, appended = None, None, []
    for tile in tiles:
        Ls = L[tile]
        use = stale if (stale is not None and rng.random() < 0.4) else tau      # a threshold read earlier
        rule = rng.integers(0, 3)
        if use is None or rule == 0:                  # tile-local: an upper bound of the tile's k-th smallest
            if len(Ls) >= k:
                kth = np.sort(Ls)[k - 1]
                cand = kth + rng.random() * 0.1 * abs(kth)              # bisection stops above it
                use = cand if use is None else min(use, cand)
        elif rule == 1 and len(appended) >= k:        # list-based: k-th smallest key of the list so far
            use = min(use, np.sort(L[appended])[k - 1])
        lim = np.inf if use is None else use + slack
        appended += [int(i) for i in tile if L[i] <= lim]
        stale = tau
        if use is not None:
            tau = use if tau is None else min(tau, use)
    return appended


# ---- adversarial data for the filter scan's band (tests/test_scan_band.py, tests/test_gpu_scan_band.py) ----
def make_index(centroids, codebook, part_codes, metric="l2"):
    """IvfPqIndexData from centroids [nlist, dim], codebook [m, 256, dsub] and per-partition codes [n_p, m]; row ids
    0, 1, .. in partition order"""
    cent, cb = np.asarray(centroids, F32), np.asarray(codebook, F32)
    nlist, dim = cent.shape
    m = cb.shape[0]
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum([len(c) for c in part_codes])
    codes_t = np.concatenate([np.asarray(c, np.uint8).reshape(-1, m).T.reshape(-1) for c in part_codes])
    ix = IvfPqIndexData(dim, nlist, m, metric, cent, cb, off, codes_t, np.arange(int(off[-1]), dtype=np.uint64), None)
    ix.validate()
    return ix


def quantiser_crossings(values, R, m):
    """For integer table offsets t = values (entries min + t ulps' worth of a common unit, range R units): the 16-bit
    code the quantiser gives (floor(f32(t * f32(qmax / R))), clamped) and the exact floor(t qmax / R).  Returns
    (code, exact) as int64 arrays."""
    t = np.asarray(values, np.int64)
    qmax = 65535 // m
    inv = F32(F32(qmax) / F32(R))
    x = (t.astype(F32) * inv).astype(F32)
    code = np.minimum(np.floor(x), qmax).astype(np.int64)
    return code, (t * qmax) // R


def quantiser_boundary_case(metric, m, rows=(96, 96, 96), nlist=3, B=8):
    """Attacks the quantiser: every table entry is exact (dyadic, few significant bits), the range R is not a power of
    two (so f32(qmax / R) is inexact), and the entries sit where the rounded (T - min) / step crosses an integer n:
    codes 2..129 of every sub-space are rounded DOWN across n or lie just under n + 1 (remainder >= one step: the
    row's d* is at or beyond L + m step, the top of the band), codes 130..255 are rounded UP across n (L above d*).
    Partition 0's rows take only codes 2..129, partition 1's only 130..255, partition 2's any code.
      l2 (dsub 2): q = centroids = 0, codeword (x, y) 2^-10, T = (x^2 + y^2) 2^-20 exactly (every sum of two squares).
      dot (dsub 1): q = 1, codeword 1 - t 2^-23, T = t 2^-23 exactly.
    Cosine: normalising the query moves it off the dyadic grid; not built."""
    R = 1000 ** 2 + 17 ** 2
    if metric == "l2":
        x = np.arange(0, 1001)
        xx, yy = np.meshgrid(x, x, indexing="ij")
        keep = (yy <= xx) & (xx * xx + yy * yy <= R)
        t_all, first = np.unique((xx * xx + yy * yy)[keep], return_index=True)
        xy = np.stack([xx[keep][first], yy[keep][first]], 1)
    else:
        t_all = np.arange(0, R + 1)
        xy = None
    code, exact = quantiser_crossings(t_all, R, m)
    qmax = 65535 // m
    frac = (t_all * qmax) % R / R                                            # exact fractional part of t / step
    hi_score = np.where(code < exact, 2.0, frac)                             # rounded down across n, or just under n + 1
    lo_score = np.where(code > exact, 1.0, 0.0) + (1 - frac) * (code > exact)
    sel_hi = np.argsort(-hi_score, kind="stable")[:128]
    sel_lo = np.argsort(-lo_score, kind="stable")[:126]
    pick = np.concatenate([[0, len(t_all) - 1], sel_hi, sel_lo])             # min (t = 0), max (t = R), high, low
    assert t_all[pick[1]] == R and t_all[0] == 0
    if metric == "l2":
        cw = (xy[pick] * 2.0 ** -10).astype(F32)                             # [256, 2]
        dim = 2 * m
        Q = np.zeros((B, dim), F32)
    else:
        cw = (1.0 - t_all[pick] * 2.0 ** -23).astype(F32)[:, None]
        dim = m
        Q = np.ones((B, dim), F32)
    cb = np.broadcast_to(cw, (m, 256, cw.shape[1])).copy()
    rng = np.random.default_rng(m)
    parts = [rng.integers(2, 130, (rows[0], m)), rng.integers(130, 256, (rows[1], m)), rng.integers(0, 256, (rows[2], m))]
    parts = (parts * nlist)[:nlist]
    return make_index(np.zeros((nlist, dim), F32), cb, parts, metric), Q


def full_lane_case(m, dsub, rows=200, nlist=2, B=16):
    """Full 16-bit lanes: m divides 65535, every sub-space's range is 1 (a power of two: f32(qmax / 1) is exact) and
    its arg-max entry (code 1, |b|^2 = 1) quantises to exactly qmax = 65535 / m, so the rows of partition 0, which take
    code 1 everywhere, sum to S = 65535 for query 0 (q = 0, centroids 0).  Any clamp or carry error would land in the
    neighbouring query's lane; the other queries are small random vectors."""
    rng = np.random.default_rng(m * 100 + dsub)
    cb = np.round(rng.uniform(-1, 1, (m, 256, dsub)) * 2 ** 5).astype(F32) * F32(2.0 ** -5 / np.sqrt(dsub + 1))
    cb[:, 0] = 0
    cb[:, 1] = 0
    cb[:, 1, 0] = 1
    parts = [np.ones((rows, m), np.int64), rng.integers(0, 256, (rows, m))][:nlist]
    Q = (rng.standard_normal((B, m * dsub)) * 0.05).astype(F32)
    Q[0] = 0
    return make_index(np.zeros((nlist, m * dsub), F32), cb, parts), Q


def cancellation_case(offset, dim=64, m=8, nlist=6, n=3000, B=12, seed=3):
    """A common offset `offset` times the residual scale on every centroid and query, the queries on their centroids:
    A = |q - c|^2 - |q|^2 ~ -|q|^2 cancels S ~ |q|^2, and the per-query tables (on q, not on the residual) hold
    entries ~ |q_i|^2 whose f32 rounding is large next to the distances (l2)"""
    rng = np.random.default_rng(seed)
    ix = random_index(rng, dim=dim, nlist=nlist, m=m, n=n, scale=1.0)
    mu = (rng.standard_normal(dim) * offset).astype(F32)
    ix.centroids = (ix.centroids + mu).astype(F32)
    Q = ix.centroids[rng.integers(0, nlist, B)].copy()
    return ix, Q


def scaled(ix, Q, s):
    """the index and queries multiplied by the power of two s (exact in f32 while nothing under- or overflows)"""
    s = F32(s)
    return IvfPqIndexData(ix.dim, ix.nlist, ix.m, ix.metric, (ix.centroids * s).astype(F32),
                          (ix.codebook * s).astype(F32), ix.part_offsets, ix.codes_t, ix.row_ids, None), (Q * s).astype(F32)


def dot_cancellation_case(m=16, n=400, nlist=2, B=4, big=2.0 ** 10):
    """dot, dsub 4: q_i = (X, X, X, X), codewords (Y1, Y2, -Y1 - r1 / X, -Y2 - r2 / X) with X, Y ~ `big`: q_i.b ~ r
    while the products are ~ big^2, so each table entry carries a rounding error ~ 2^-24 big^2 -- far above sbound + m
    when big^2 >> m -- and the filter's two fmaf chains round differently from the oracle's sum.  Only the
    2 (|q|^2 + CB2) term of E covers it."""
    rng = np.random.default_rng(7)
    X = (big * (1 + rng.random((B, m)))).astype(F32)
    Y = (big * (1 + rng.random((m, 256, 2)))).astype(F32)
    r = rng.uniform(-0.5, 0.5, (m, 256, 2))
    Xr = X[0].astype(np.float64)[:, None, None]
    cb = np.concatenate([Y, (-Y.astype(np.float64) - r / Xr).astype(F32)], 2).astype(F32)
    Q = np.repeat(X, 4, axis=1).astype(F32)
    parts = [rng.integers(0, 256, (n, m)) for _ in range(nlist)]
    return make_index(np.zeros((nlist, 4 * m), F32), cb, parts, "dot"), Q


def overflow_case(dim=64, m=8, nlist=4, per=300, B=1200, seed=11):
    """|q|^2 just above FLT_MAX with every distance finite: queries and centroids share a huge common vector mu
    (|mu|^2 = FLT_MAX (1 + 2^-12)), each query sits near its centroid, and every codeword points along mu with 2^-9..2^-7
    of its length, so that the table entries (|q_i - b|^2 ~ |q_i|^2 (1 - 2^-8)), their sums (base, sbound) and R stay
    finite while f32(|q|^2) = inf.  Then A = coarse - |q|^2 = -inf for every probe."""
    rng = np.random.default_rng(seed)
    dsub = dim // m
    u = rng.uniform(0.5, 1.0, dim)
    u /= np.sqrt((u * u).sum())
    mu = u * np.sqrt(float(np.finfo(F32).max) * (1 + 2.0 ** -12))
    assert np.isinf(F32(float((mu.astype(F32).astype(np.float64) ** 2).sum())))
    cent = (mu[None, :] + rng.standard_normal((nlist, dim)) * 1e15).astype(F32)
    s = rng.uniform(2.0 ** -9, 2.0 ** -7, (m, 256, 1))
    cb = (s * mu.reshape(m, 1, dsub)).astype(F32)
    parts = [rng.integers(0, 256, (per, m)) for _ in range(nlist)]
    ix = make_index(cent, cb, parts)
    Q = (cent[rng.integers(0, nlist, B)] + rng.standard_normal((B, dim)) * 1e15).astype(F32)
    return ix, Q

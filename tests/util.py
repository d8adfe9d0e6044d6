"""Test helpers: synthetic IVF_PQ indexes with arbitrary (untrained) contents.  Parity does
not depend on index quality -- the CUDA path and the oracle consume the identical arrays --
so random centroids / codebooks / codes exercise the arithmetic just as well and let the
tests shape edge cases (empty, tiny and multi-tile partitions)."""
import numpy as np

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

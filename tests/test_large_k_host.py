"""The large top-k select (csrc/select_large.cu) restated in NumPy, and the refusals above LGPU_K_MAX; no GPU needed.

The restatement follows the kernels step by step: the three key digits of 11 / 11 / 10 bits (each walk picks the digit
whose bin holds the r-th row of the prefix and stops early when that bin holds exactly the rows still needed), the
radix walk over the ids of the rows tied at the k-th key (relative to their minimum, 11 bits a digit), and the
compaction predicate key < t or (key == t and id <= u).  On adversarial key sets it must take exactly min(k, valid)
rows, and those rows sorted by (key, id) must be np.lexsort's first k."""
import ctypes as C
import zlib

import numpy as np
import pytest

from lancedb_b200 import _native
from lancedb_b200 import distributed

U64_MAX = np.iinfo(np.uint64).max
K_MAX = 65536


def f32_key(v: np.ndarray) -> np.ndarray:
    """the ordered key of common.cuh (NaN dropped by the caller, -0 folded into +0)"""
    b = np.ascontiguousarray(v, np.float32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def _digit(values: np.ndarray, r: int, nbins: int):
    """(digit, rows below it, rows in it) of the bin holding the r-th row (1-based)"""
    h = np.bincount(values.astype(np.int64), minlength=nbins)
    cum = np.cumsum(h)
    d = int(np.searchsorted(cum, r))
    return d, int(cum[d] - h[d]), int(h[d])


def threshold(keys: np.ndarray, ids: np.ndarray, k: int):
    """(t, u): the rows with key < t or (key == t and id <= u) are the k best, as the walk kernels find them"""
    n = len(keys)
    if n <= k:
        return 0xFFFFFFFF, int(U64_MAX)
    r, t = k, 0
    for shift, width in ((21, 11), (10, 11), (0, 10)):
        top = shift + width
        m = np.ones(n, bool) if top >= 32 else (keys >> np.uint32(top)) == np.uint32(t >> top)
        d, below, hd = _digit((keys[m] >> np.uint32(shift)) & np.uint32((1 << width) - 1), r, 1 << width)
        r -= below
        t |= d << shift
        if hd == r:
            return t | ((1 << shift) - 1), int(U64_MAX)
    tie = ids[keys == np.uint32(t)]
    lo, hi = int(tie.min()), int(tie.max())
    if lo == hi:
        return t, lo
    v = tie - np.uint64(lo)
    nbits = (hi - lo).bit_length()
    width = min(11, nbits)
    shift, pre = nbits - width, 0
    while True:
        top = shift + width
        m = np.ones(len(v), bool) if top >= 64 else (v >> np.uint64(top)) == np.uint64(pre >> top)
        d, below, hd = _digit((v[m] >> np.uint64(shift)) & np.uint64((1 << width) - 1), r, 1 << width)
        r -= below
        pre |= d << shift
        if hd == r or shift == 0:
            if hd == r:
                pre |= (1 << shift) - 1
            return t, lo + pre
        width = min(shift, 11)
        shift -= width


def check(vals: np.ndarray, ids: np.ndarray, k: int):
    keep = ~np.isnan(vals)
    v, i = vals[keep] + np.float32(0), ids[keep]                       # -0 + 0 = +0
    keys = f32_key(v)
    t, u = threshold(keys, i, k)
    sel = (keys < np.uint32(t)) | ((keys == np.uint32(t)) & (i <= np.uint64(u)))
    assert int(sel.sum()) == min(k, len(v)), (int(sel.sum()), k, len(v))
    got = np.lexsort((i[sel], keys[sel]))
    exp = np.lexsort((i, v))[:k]
    assert np.array_equal(i[sel][got], i[exp])
    assert np.array_equal(v[sel][got].view(np.uint32), v[exp].view(np.uint32))


def _values(kind: str, n: int, rng) -> np.ndarray:
    if kind == "equal":
        return np.full(n, 2.5, np.float32)
    if kind == "nan":
        return np.full(n, np.nan, np.float32)
    if kind == "inf":
        return rng.choice(np.array([np.inf, -np.inf, 1.0], np.float32), n)
    if kind == "zeros":
        return rng.choice(np.array([0.0, -0.0], np.float32), n)
    if kind == "few":                                                     # huge multiplicities, adjacent floats
        return rng.choice(np.array([-3.0, 0.5, np.nextafter(np.float32(0.5), np.float32(1)), 7.0], np.float32), n)
    if kind == "hamming":                                                 # integer distances 0..128
        return rng.integers(0, 129, n).astype(np.float32)
    if kind == "mixed":
        v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(np.float32)
        v[rng.random(n) < 0.1] = np.nan
        v[rng.random(n) < 0.05] = -0.0
        return v
    raise ValueError(kind)


def _ids(kind: str, n: int, rng) -> np.ndarray:
    if kind == "asc":
        return np.arange(n, dtype=np.uint64)
    if kind == "desc":
        return np.arange(n, dtype=np.uint64)[::-1] * np.uint64(7) + np.uint64(3)
    # the whole 64-bit range: the tie walk runs all six 11-bit id digits
    i = rng.integers(0, 1 << 62, n, dtype=np.uint64) * np.uint64(4)
    i[:2] = [0, U64_MAX - np.uint64(1)]
    return rng.permutation(np.unique(i))


@pytest.mark.parametrize("kind", ["equal", "nan", "inf", "zeros", "few", "hamming", "mixed"])
@pytest.mark.parametrize("idk", ["asc", "desc", "wide"])
def test_walk_takes_exactly_the_k_best(kind, idk):
    rng = np.random.default_rng(zlib.crc32(f"{kind}/{idk}".encode()))
    for n, k in ((5000, 2049), (5000, 4999), (5000, 5000), (5000, 5001), (20000, 4097), (150000, K_MAX),
                 (K_MAX, K_MAX), (K_MAX + 1, K_MAX)):
        ids = _ids(idk, n, rng)
        n = len(ids)                                       # (distinct wide ids: a few may collide)
        check(_values(kind, n, rng), ids, k)


def test_tie_walk_finishes_early_and_repeated_ids():
    """a tie run whose id digits split exactly at the needed count stops before the last digit, and one id repeated
    across the whole tie run (all rows identical) gives u = that id"""
    k = 3000
    vals = np.full(6000, 1.0, np.float32)
    check(vals, np.arange(6000, dtype=np.uint64) * np.uint64(1 << 20), k)
    keys = f32_key(vals)
    t, u = threshold(keys, np.full(6000, 42, np.uint64), k)
    assert t == int(keys[0]) and u == 42


# ---------------------------------------------------------------- refusals, before any device work
def test_debug_select_large_refuses_k_outside_2049_to_k_max():
    lib = _native.load()
    a = _native.DebugSelectArgs(mode=1, B=1, k=K_MAX + 1)
    assert lib.lgpu_debug_select_large(C.byref(a), -1, None) == _native.LGPU_INVALID_INPUT
    assert b"65536" in lib.lgpu_last_error()
    a.k = 2048
    assert lib.lgpu_debug_select_large(C.byref(a), -1, None) == _native.LGPU_INVALID_INPUT
    assert b"2049" in lib.lgpu_last_error()
    a.k = K_MAX                                             # in range: the next check (null buffers) is reached
    assert lib.lgpu_debug_select_large(C.byref(a), -1, None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"null output buffer"
    assert _native.K_MAX == K_MAX


def test_query_builder_refuses_k_above_k_max():
    import lancedb_b200 as lancedb
    db = lancedb.connect("memory://")
    t = db.create_table("t", {"vector": np.zeros((3, 4), np.float32), "id": np.arange(3)})
    q = np.zeros(4, np.float32)
    with pytest.raises(ValueError, match="65536"):
        t.search(q).limit(K_MAX + 1).to_arrow()
    with pytest.raises(ValueError, match="65536"):
        t.search(q).offset(K_MAX - 99).limit(100).to_arrow()


def test_sharded_search_refuses_k_above_2048():
    distributed.check_k(2048)
    with pytest.raises(ValueError, match="2048"):
        distributed.check_k(2049)

"""The top-k selection's restatement (tests/select_oracle.py) against a brute-force sort of Python tuples, the host
merge (distributed.merge_records) against both, and lgpu_debug_select's refusal of malformed arguments -- no GPU."""
import ctypes as C
import math

import numpy as np
import pytest

from lancedb_b200 import _native
from lancedb_b200.distributed import merge_records
from tests import select_oracle as so

MAX = 2 ** 64 - 1


def brute(a: dict):
    """per query: None (untouched) or the sorted list of (distance, id, pos) tuples it keeps"""
    res = []
    for q in range(a["B"]):
        if (a.get("gate") is not None and a["gate"][0] == 0) or (a.get("only") is not None and a["only"][q] == 0):
            res.append(None)
            continue
        cands = []
        if a["mode"] == 0:
            for j in range(a["nprobes"]):
                s = q * a["nprobes"] + j
                p = int(a["probes"][s])
                if p < a["nlist"]:
                    for r in range(int(a["part_n"][p])):
                        row = int(a["part_off"][p]) + r
                        rid = row if a.get("row_ids") is None else int(a["row_ids"][row])
                        cands.append((float(a["dist"][int(a["seg_off"][s]) + r]), rid, row))
        elif a["mode"] == 1:
            for c in range(a["ncols"]):
                cid = c if a.get("col_ids") is None else int(a["col_ids"][c])
                cands.append((float(a["dense"][q * a["row_stride"] + c]), cid, c))
        else:
            n = a["ncols"] if a.get("ncols_q") is None else min(a["ncols"], int(a["ncols_q"][q]))
            for c in range(n):
                addr = (c // a["inner"]) * a["outer_stride"] + q * a["row_stride"] + c % a["inner"]
                if a.get("cand_rec") is not None:
                    cid, v = int(a["cand_rec"][addr]["id"]), float(a["cand_rec"][addr]["dist"])
                else:
                    cid, v = int(a["cand_ids"][addr]), float(a["dense"][addr])
                if cid != MAX:
                    cands.append((v, cid, c if a.get("cand_pos") is None else int(a["cand_pos"][addr])))
        keep = []
        for v, i, p in cands:
            if math.isnan(v):
                continue
            if a.get("has_lower") and not v >= float(np.float32(a["lower"])):
                continue
            if a.get("has_upper") and not v < float(np.float32(a["upper"])):
                continue
            if a.get("allow") is not None and not (i < a["allow_bits"] and (int(a["allow"][i >> 5]) >> (i & 31)) & 1):
                continue
            keep.append((0.0 if v == 0 else v, i, p))
        res.append(sorted(keep)[:a["k"]])
    return res


def check_against_brute(a, pos, rec):
    out = so.select(a, so.outputs(a["B"], a["k"], pos, rec))
    fresh = so.outputs(a["B"], a["k"], pos, rec)
    for q, top in enumerate(brute(a)):
        ids = out["rec"][q]["id"] if rec else out["ids"][q]
        dist = out["rec"][q]["dist"] if rec else out["dist"][q]
        if top is None:
            assert out["count"][q] == fresh["count"][q] and np.array_equal(ids, (fresh["rec"][q]["id"] if rec else
                                                                                 fresh["ids"][q]))
            continue
        n = len(top)
        assert out["count"][q] == n
        assert ids[:n].tolist() == [t[1] for t in top] and np.all(ids[n:] == so.U64_MAX)
        want = np.array([t[0] for t in top] + [np.inf] * (a["k"] - n), np.float32)
        assert np.array_equal(dist.view(np.uint32), want.view(np.uint32))
        if rec:
            assert np.all(out["rec"][q]["pad"] == 0)
        if pos:
            assert out["pos"][q, :n].tolist() == [t[2] for t in top] and np.all(out["pos"][q, n:] == so.U64_MAX)


def random_case(rng, mode):
    B, k = int(rng.integers(1, 5)), int(rng.choice([1, 2, 5, 9, 33]))
    order = str(rng.choice(["mixed", "mixed", "two", "equal", "asc", "desc"]))
    kw = {}
    if mode == 0:
        nlist = int(rng.integers(1, 7))
        parts = [so.values(order, int(rng.choice([0, 1, 3, 4, 7, 20])), rng) for _ in range(nlist)]
        nrows = sum(len(p) for p in parts)
        nprobes = int(rng.integers(1, 5))
        probes = rng.integers(0, nlist + 2, (B, nprobes)).astype(np.uint64)
        probes[probes >= nlist] = so.U64_MAX
        a = so.segments_case(parts, probes, k, row_ids=rng.permutation(nrows).astype(np.uint64) * 3
                             if rng.random() < 0.7 else None)
    elif mode == 1:
        n = int(rng.choice([0, 1, 3, 8, 30]))
        V = np.stack([so.values(order, n, rng, shift=q) for q in range(B)])
        a = so.dense_case(V, k, col_ids=so.unique_ids(rng, n) if rng.random() < 0.6 else None,
                          stride=n + int(rng.integers(0, 3)))
    else:
        if rng.random() < 0.4:
            L, kk = int(rng.integers(1, 4)), int(rng.choice([1, 4, 9]))
            ids, dist = so.search_lists(rng, L, B, kk, rng.integers(0, kk + 1, (L, B)),
                                        so.values(order, 16, rng))
            a = so.merge_case(ids, dist, min(k, L * kk) if rng.random() < 0.5 else k, rec=rng.random() < 0.5)
        else:
            lens = rng.integers(0, 25, B)
            vals = [so.values(order, int(m), rng) for m in lens]
            a = so.cands_case(vals, [so.unique_ids(rng, int(m)) for m in lens], k,
                              pos=[rng.integers(0, 1 << 30, int(m)).astype(np.uint64) for m in lens]
                              if rng.random() < 0.5 else None, ncols_q=rng.random() < 0.5)
    if rng.random() < 0.4:
        present = [v for q in range(a["B"]) for v in so.candidates(a, q)[0].tolist() if not math.isnan(v)]
        pick = (lambda: float(rng.choice(present))) if present else (lambda: 0.0)
        kw["has_lower"], kw["lower"] = int(rng.random() < 0.7), float(rng.choice([pick(), -np.inf, np.inf]))
        kw["has_upper"], kw["upper"] = int(rng.random() < 0.7), float(rng.choice([pick(), np.inf, kw["lower"]]))
    if rng.random() < 0.3:
        kw["allow"] = rng.integers(0, 1 << 32, 16, dtype=np.uint64).astype(np.uint32)
        kw["allow_bits"] = int(rng.integers(0, 16 * 32 + 1))
    if rng.random() < 0.3:
        kw["only"] = rng.integers(0, 2, a["B"]).astype(np.uint32)
    if rng.random() < 0.1:
        kw["gate"] = np.array([rng.integers(0, 2)], np.uint32)
    a.update(kw)
    return a


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_reference_matches_a_brute_force_sort(mode):
    rng = np.random.default_rng(100 + mode)
    for _ in range(150):
        a = random_case(rng, mode)
        check_against_brute(a, pos=bool(rng.random() < 0.5), rec=bool(rng.random() < 0.3))


def test_reference_keeps_ids_in_the_allow_bitmap_only():
    """ids 0..63 over two words, allow_bits cutting the second word: the bits at and above allow_bits do not count"""
    a = so.dense_case(np.arange(64, dtype=np.float32)[None, :], 64, allow=np.array([0xF0F0F0F0, 0xFFFFFFFF], np.uint32),
                      allow_bits=40)
    ids, dist, _ = so.select_query(a, 0)
    want = [i for i in range(32) if (0xF0F0F0F0 >> i) & 1] + list(range(32, 40))
    assert ids.tolist() == want and dist.tolist() == [float(i) for i in want]
    check_against_brute(a, pos=True, rec=False)


def test_reference_range_bounds_as_written():
    """[lower, upper): a bound equal to a present value, lower == upper, and infinite bounds (+inf is outside
    [-inf, +inf), -inf inside it)"""
    v = np.array([-np.inf, -1.0, 0.0, -0.0, 1.0, 1.0, 2.0, np.inf, np.nan], np.float32)[None, :]
    for lo, hi, want in ((1.0, 2.0, [4, 5]), (1.0, 1.0, []), (-np.inf, np.inf, [0, 1, 2, 3, 4, 5, 6]),
                         (np.inf, None, [7]), (None, -np.inf, []), (0.0, None, [2, 3, 4, 5, 6, 7])):
        a = so.dense_case(v, 9, has_lower=lo is not None, lower=lo or 0.0, has_upper=hi is not None, upper=hi or 0.0)
        ids, dist, _ = so.select_query(a, 0)
        assert sorted(ids.tolist()) == want, (lo, hi)
        assert not np.any(np.signbit(dist[dist == 0]))                  # -0 is reported as +0
        check_against_brute(a, pos=False, rec=False)


def _gathered(ids, dist):
    g = np.zeros(ids.shape, _native.TOPK_RECORD)
    g["id"], g["dist"] = ids, dist
    return g


def test_merge_records_drops_nan_and_reports_minus_zero_as_plus_zero():
    """what the merge kernel does with a NaN and a -0 in a gathered list"""
    ids = np.array([[[5, 9, 2, MAX]], [[7, 3, 4, MAX]]], np.uint64)
    dist = np.array([[[-0.0, np.nan, 1.0, np.inf]], [[0.0, -0.0, np.nan, np.inf]]], np.float32)
    m_ids, m_dist, m_cnt = merge_records(_gathered(ids, dist), 4)
    assert m_cnt.tolist() == [4]
    assert m_ids.tolist() == [[3, 5, 7, 2]]
    assert m_dist.view(np.uint32).tolist() == [[0, 0, 0, np.float32(1.0).view(np.uint32)]]
    out = so.select(so.merge_case(ids, dist, 4, rec=True), so.outputs(1, 4, rec=True))
    assert np.array_equal(out["rec"]["id"], m_ids) and np.array_equal(out["rec"]["dist"].view(np.uint32),
                                                                       m_dist.view(np.uint32))


@pytest.mark.parametrize("L,k", [(1, 1), (2, 10), (3, 33), (8, 100), (8, 2048)])
def test_merge_records_restates_the_merge(L, k):
    rng = np.random.default_rng(L * 1000 + k)
    B = 3
    counts = rng.integers(0, k + 1, (L, B))
    counts[0, 0] = k
    pool = np.array([-2.5, -0.0, 0.0, 0.5, 1.0, 1.0, 3.0, np.inf], np.float32)
    ids, dist = so.search_lists(rng, L, B, k, counts, pool)
    dist[0, 1, 0] = np.nan if counts[0, 1] else dist[0, 1, 0]
    m_ids, m_dist, m_cnt = merge_records(_gathered(ids, dist), k)
    for rec in (False, True):
        out = so.select(so.merge_case(ids, dist, k, rec=rec), so.outputs(B, k, rec=rec))
        got_ids = out["rec"]["id"] if rec else out["ids"]
        got_dist = out["rec"]["dist"] if rec else out["dist"]
        assert np.array_equal(out["count"], m_cnt) and np.array_equal(got_ids, m_ids)
        assert np.array_equal(got_dist.view(np.uint32), m_dist.view(np.uint32))
    if k <= 100:
        check_against_brute(so.merge_case(ids, dist, k, rec=True), pos=True, rec=True)


# ---------------------------------------------------------------- lgpu_debug_select refuses before the device
FAKE = 0x10000          # never dereferenced: every call below is refused before the kernels run


def _valid(mode):
    a = dict(mode=mode, B=2, k=8, out_ids=FAKE, out_dist=FAKE, out_count=FAKE)
    if mode == 0:
        a.update(dist=FAKE, seg_off=FAKE, probes=FAKE, part_n=FAKE, part_off=FAKE, nprobes=1, nlist=1, dist_len=64)
    elif mode == 1:
        a.update(dense=FAKE, ncols=8, row_stride=8)
    else:
        a.update(dense=FAKE, cand_ids=FAKE, ncols=8, inner=8, row_stride=8)
    return a


def _refused(msg, **args):
    a = _native.DebugSelectArgs(**args)
    assert _native.load().lgpu_debug_select(C.byref(a), -1, None) == _native.LGPU_INVALID_INPUT
    assert msg in _native.load().lgpu_last_error().decode()


def test_debug_select_refuses_what_the_kernels_would_read_out_of_bounds_with():
    assert _native.load().lgpu_debug_select(None, 0, None) == _native.LGPU_INVALID_INPUT
    for mode in (-1, 3, 7):
        _refused("select mode", **{**_valid(1), "mode": mode})
    for k in (0, 2049, 1 << 31):
        _refused("k must be", **{**_valid(1), "k": k})
    for mode in (0, 1, 2):
        for drop in ("out_count", "out_ids", "out_dist"):
            _refused("null output buffer", **{**_valid(mode), drop: None})
        _refused("out_rec must be 16-byte aligned", **{**_valid(mode), "out_rec": FAKE + 8})
    for drop in ("dist", "seg_off", "probes", "part_n", "part_off"):
        _refused("null mode-0 buffer", **{**_valid(0), drop: None})
    _refused("dist must be 16-byte aligned", **{**_valid(0), "dist": FAKE + 4})
    _refused("null mode-1 buffer", **{**_valid(1), "dense": None})
    for drop in ("dense", "cand_ids"):
        _refused("null mode-2 buffer", **{**_valid(2), drop: None})
    _refused("cand_rec must be 16-byte aligned", **{**_valid(2), "cand_rec": FAKE + 8})
    _refused("inner must be at least 1", **{**_valid(2), "inner": 0})

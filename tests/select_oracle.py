"""Exact NumPy restatement of the top-k selection every search ends in (csrc/select.cu, run alone through
lgpu_debug_select), and the candidate layouts the library feeds it.

The selection is pure ordering, so the restatement is exact: per query, the valid candidates (probe < nlist in mode 0,
column < ncols_q[q] and id != UINT64_MAX in mode 2) without NaN, inside [lower, upper) as written (infinite bounds
included), with an id below allow_bits whose allow bit is 1; -0 folded into +0; ordered by (distance, id); the first k,
padded with UINT64_MAX / +inf.  A query with only[q] == 0, or every query when gate == 0, is left untouched.

A case is a dict keyed like lgpu_debug_select_args: host numpy arrays for the device buffers (None or absent = NULL),
plain numbers for the rest.  `outputs` gives the [B][k] / [B] buffers a call writes to."""
from __future__ import annotations

import numpy as np

U64_MAX = np.uint64(0xFFFF_FFFF_FFFF_FFFF)
RECORD = np.dtype([("id", "<u8"), ("dist", "<f4"), ("pad", "<u4")])       # TopkRecord, 16 bytes


def candidates(a: dict, q: int):
    """(values f32, ids u64, pos u64) of query q's valid candidates, in layout order"""
    get = a.get
    if a["mode"] == 0:
        vs, ids, pos = [], [], []
        for j in range(a["nprobes"]):
            s = q * a["nprobes"] + j
            p = int(a["probes"][s])
            if p >= a["nlist"]:
                continue
            n, off, base = int(a["part_n"][p]), int(a["seg_off"][s]), int(a["part_off"][p])
            r = np.arange(base, base + n, dtype=np.uint64)
            vs.append(a["dist"][off:off + n])
            ids.append(r if get("row_ids") is None else a["row_ids"][r])
            pos.append(r)
        if not vs:
            return np.zeros(0, np.float32), np.zeros(0, np.uint64), np.zeros(0, np.uint64)
        return np.concatenate(vs), np.concatenate(ids), np.concatenate(pos)
    if a["mode"] == 1:
        n, base = int(a["ncols"]), q * int(a["row_stride"])
        c = np.arange(n, dtype=np.uint64)
        return a["dense"][base:base + n], (c if get("col_ids") is None else a["col_ids"][:n]), c
    n = int(a["ncols"])
    if get("ncols_q") is not None:
        n = min(n, int(a["ncols_q"][q]))
    c = np.arange(n, dtype=np.uint64)
    addr = (c // np.uint64(a["inner"])) * np.uint64(a["outer_stride"]) + np.uint64(q * a["row_stride"]) + \
        c % np.uint64(a["inner"])
    if get("cand_rec") is not None:
        ids, v = a["cand_rec"]["id"][addr], a["cand_rec"]["dist"][addr]
    else:
        ids, v = a["cand_ids"][addr], a["dense"][addr]
    pos = c if get("cand_pos") is None else a["cand_pos"][addr]
    ok = ids != U64_MAX
    return v[ok], ids[ok], pos[ok]


def allowed(a: dict, ids: np.ndarray) -> np.ndarray:
    ok = ids < np.uint64(a["allow_bits"])
    w = np.where(ok, ids >> np.uint64(5), 0).astype(np.int64)
    return ok & (((a["allow"][w] >> (ids & np.uint64(31)).astype(np.uint32)) & 1) == 1)


def select_query(a: dict, q: int):
    """(ids, dist, pos) of query q's top-k, unpadded"""
    v, ids, pos = candidates(a, q)
    keep = ~np.isnan(v)
    if a.get("has_lower"):
        keep &= v >= np.float32(a["lower"])
    if a.get("has_upper"):
        keep &= v < np.float32(a["upper"])
    if a.get("allow") is not None:
        keep &= allowed(a, ids)
    v, ids, pos = v[keep] + np.float32(0), ids[keep], pos[keep]          # -0 + 0 = +0
    order = np.lexsort((ids, v))[:a["k"]]
    return ids[order], v[order], pos[order]


def outputs(B: int, k: int, pos: bool = False, rec: bool = False, fill: int = 0xA5) -> dict:
    """output buffers as a call sees them: every byte `fill`"""
    def buf(dt, n):
        return np.full(n * np.dtype(dt).itemsize, fill, np.uint8).view(dt)
    out = {"count": buf(np.uint32, B)}
    if rec:
        out["rec"] = buf(RECORD, B * k).reshape(B, k)
    else:
        out["ids"], out["dist"] = buf(np.uint64, B * k).reshape(B, k), buf(np.float32, B * k).reshape(B, k)
    if pos:
        out["pos"] = buf(np.uint64, B * k).reshape(B, k)
    return out


def select(a: dict, out: dict) -> dict:
    """what lgpu_debug_select leaves in `out` (modified in place and returned)"""
    B, k = a["B"], a["k"]
    if a.get("gate") is not None and a["gate"][0] == 0:
        return out
    for q in range(B):
        if a.get("only") is not None and a["only"][q] == 0:
            continue
        ids, dist, pos = select_query(a, q)
        n = len(ids)
        pid = np.full(k, U64_MAX, np.uint64); pid[:n] = ids
        pd = np.full(k, np.inf, np.float32); pd[:n] = dist
        if "rec" in out:
            out["rec"][q]["id"], out["rec"][q]["dist"], out["rec"][q]["pad"] = pid, pd, 0
        else:
            out["ids"][q], out["dist"][q] = pid, pd
        if "pos" in out:
            out["pos"][q] = U64_MAX
            out["pos"][q, :n] = pos
        out["count"][q] = n
    return out


# ---------------------------------------------------------------- candidate values
F32_TINY = np.float32(1.4e-45)                              # the smallest denormal


def values(order: str, n: int, rng: np.random.Generator, shift: float = 0.0) -> np.ndarray:
    """n candidate distances in one of the orders the tests use"""
    if order == "asc":
        return (np.arange(n) * 0.5 - n / 4 + shift).astype(np.float32)
    if order == "desc":
        return (np.arange(n)[::-1] * 0.5 - n / 4 + shift).astype(np.float32)
    if order == "equal":
        return np.full(n, 1.5 + shift, np.float32)
    if order == "two":
        return np.where(rng.random(n) < 0.5, 0.25, 0.75).astype(np.float32)
    if order == "mixed":
        # negative and positive values (some repeated) mixed with +-0, +-inf, denormals and NaNs of both signs
        v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(np.float32)
        rep = rng.random(n) < 0.2
        if n:
            v[rep] = rng.choice(v, int(rep.sum()))
        specials = np.array([0.0, -0.0, np.inf, -np.inf, F32_TINY, -F32_TINY, 3 * F32_TINY, -7 * F32_TINY],
                            np.float32)
        sel = rng.random(n) < 0.25
        v[sel] = rng.choice(specials, int(sel.sum()))
        nan = rng.random(n) < 0.08
        bits = rng.choice(np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFBFFFFF, 0x7FC0DEAD], np.uint32),
                          int(nan.sum()))
        v[nan] = bits.view(np.float32)
        return v
    raise ValueError(order)


# ---------------------------------------------------------------- the layouts the library hands the selection
def dense_case(V: np.ndarray, k: int, col_ids=None, stride: int | None = None, **kw) -> dict:
    """mode 1: row q of V [B][n] at q * stride of the dense block; the columns from n to stride hold -inf, which must
    never be read as candidates"""
    B, n = V.shape
    stride = n if stride is None else stride
    dense = np.full(max(B * stride, 1), -np.inf, np.float32)
    for q in range(B):
        dense[q * stride:q * stride + n] = V[q]
    return dict(mode=1, dense=dense, ncols=n, row_stride=stride, col_ids=col_ids, B=B, k=k, **kw)


def cands_case(vals, ids, k: int, pos=None, ncols_q: bool = False, **kw) -> dict:
    """mode 2 as select_cands lays it out: [B][ncols] values and ids, ncols the longest list.  A shorter list is padded
    with unused slots (id UINT64_MAX); with ncols_q the list is cut at ncols_q[q] = its length instead, and the slots
    behind the cut hold -inf entries with valid ids, which must never be read."""
    B = len(vals)
    n = max([len(v) for v in vals] + [1])
    dense = np.full((B, n), -np.inf, np.float32)
    cid = np.full((B, n), 7 if ncols_q else U64_MAX, np.uint64)
    cpos = np.full((B, n), 12345, np.uint64)
    for q in range(B):
        m = len(vals[q])
        dense[q, :m], cid[q, :m] = vals[q], ids[q]
        if pos is not None:
            cpos[q, :m] = pos[q]
    a = dict(mode=2, dense=dense.reshape(-1), cand_ids=cid.reshape(-1), ncols=n, inner=n, row_stride=n, outer_stride=0,
             B=B, k=k, cand_pos=None if pos is None else cpos.reshape(-1), **kw)
    if ncols_q:
        a["ncols_q"] = np.array([len(v) for v in vals], np.uint32)
    return a


def merge_case(ids: np.ndarray, dist: np.ndarray, k: int, rec: bool = False, **kw) -> dict:
    """mode 2 as the merge lays it out: nlists top-k lists [nlists][B][k] (list l of query q at l * B * k + q * k), as
    packed records or as ids + values"""
    L, B, kk = ids.shape
    a = dict(mode=2, ncols=L * kk, inner=kk, row_stride=kk, outer_stride=B * kk, B=B, k=k, **kw)
    if rec:
        r = np.zeros(ids.size, RECORD)
        r["id"], r["dist"] = ids.reshape(-1), dist.reshape(-1)
        a["cand_rec"] = r
    else:
        a["cand_ids"], a["dense"] = ids.reshape(-1).copy(), dist.reshape(-1).copy()
    return a


def unique_ids(rng: np.random.Generator, n: int) -> np.ndarray:
    """n distinct ids in no order, spread over 40 bits"""
    return (rng.permutation(n).astype(np.uint64) * np.uint64(1 << 20)) | rng.integers(0, 1 << 20, n).astype(np.uint64)


def search_lists(rng: np.random.Generator, L: int, B: int, k: int, counts: np.ndarray, pool: np.ndarray):
    """L top-k lists per query as a search emits them: list (l, q) holds counts[l, q] entries ascending by
    (distance, id), then UINT64_MAX / +inf.  Distances are drawn from `pool` (shared by the lists: ties across lists),
    ids are unique within a query."""
    ids = np.full((L, B, k), U64_MAX, np.uint64)
    dist = np.full((L, B, k), np.inf, np.float32)
    for q in range(B):
        qid = unique_ids(rng, int(counts[:, q].sum()))
        at = 0
        for l in range(L):
            c = int(counts[l, q])
            d = rng.choice(pool, c).astype(np.float32)
            i = qid[at:at + c]; at += c
            o = np.lexsort((i, d))
            ids[l, q, :c], dist[l, q, :c] = i[o], d[o]
    return ids, dist


def segments_case(part_vals, probes: np.ndarray, k: int, row_ids=None, gap: int = 4, **kw) -> dict:
    """mode 0: partition p holds part_vals[p] (stored rows part_off[p] ..); every used probe slot gets a segment of
    its own in `dist`, at a multiple of 4 floats, padded to 4 and followed by `gap` more floats, all -inf, which must
    never be read as candidates"""
    nlist = len(part_vals)
    part_n = np.array([len(v) for v in part_vals], np.uint32)
    part_off = np.concatenate([[0], np.cumsum(part_n)[:-1]]).astype(np.uint64)
    B, nprobes = probes.shape
    seg_off = np.zeros(B * nprobes, np.uint64)
    chunks, at = [], 0
    for s, p in enumerate(probes.reshape(-1)):
        seg_off[s] = at
        if p >= nlist:
            continue
        n = int(part_n[p])
        span = (n + 3) // 4 * 4 + gap
        c = np.full(span, -np.inf, np.float32)
        c[:n] = part_vals[p]
        chunks.append(c)
        at += span
    dist = np.concatenate(chunks + [np.zeros(4, np.float32)])
    return dict(mode=0, dist=dist, dist_len=dist.size, seg_off=seg_off, probes=probes.reshape(-1).astype(np.uint64),
                nprobes=nprobes, nlist=nlist, part_n=part_n, part_off=part_off, row_ids=row_ids, B=B, k=k, **kw)

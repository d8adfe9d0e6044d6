"""The union search's contract, composed from the existing oracles: the C oracle's search of the index (each kind's
own `search`), the exact flat top-k of the tail (float flat search under the index's metric, or Hamming), both under
the same distance_range and allow mask, merged by (_distance, _rowid) with NaN last (cand_less in oracle/oracle.c)."""
import numpy as np

import oracle
from tests import hamming_oracle, hnsw_sq_oracle, ivf_binary_oracle, pq4_oracle, rq_oracle, sq_oracle

U64_MAX = np.iinfo(np.uint64).max


def index_search(data, q, k, nprobes, refine_factor=0, lower=None, upper=None, allow=None, max_nprobes=0, ef=0):
    """The oracle's search of the index alone; allow: optional bool mask over row ids."""
    kw = dict(lower=lower, upper=upper, allow=allow, max_nprobes=max_nprobes)
    t = data.index_type
    if t == "IVF_FLAT":
        return ivf_binary_oracle.search(data, q, k, nprobes, **kw)
    if t == "IVF_PQ" and data.num_bits == 8:
        return oracle.OracleIndex.from_data(data).search(q, k, nprobes, refine_factor, nthreads=0, **kw)
    if t == "IVF_HNSW_SQ":
        return hnsw_sq_oracle.search(data, q, k, nprobes, ef, refine_factor, **kw)
    mod = {"IVF_PQ": pq4_oracle, "IVF_SQ": sq_oracle, "IVF_RQ": rq_oracle}[t]
    return mod.search(data, q, k, nprobes, refine_factor, **kw)


def tail_search(data, tail, tail_ids, q, k, lower=None, upper=None, allow=None):
    """The exact top-k of the tail rows (ids tail_ids) under the index's metric."""
    if data.index_type == "IVF_FLAT":
        return hamming_oracle.flat_search_u8(tail, q, k, row_ids=tail_ids, lower=lower, upper=upper, allow=allow)
    return oracle.flat_search(tail, q, k, metric=data.metric, row_ids=tail_ids, lower=lower, upper=upper, nthreads=0,
                              allow=allow)


def merge(a, b, k):
    """Top-k by (_distance, _rowid), NaN last, of the valid entries of two results."""
    B = len(a[2])
    ids = np.full((B, k), U64_MAX, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    for i in range(B):
        ci = np.concatenate([a[0][i, :a[2][i]], b[0][i, :b[2][i]]])
        cd = np.concatenate([a[1][i, :a[2][i]], b[1][i, :b[2][i]]])
        o = np.lexsort((ci, cd, np.isnan(cd)))[:k]
        n = o.size
        ids[i, :n], dist[i, :n], cnt[i] = ci[o], cd[o], n
    return ids, dist, cnt


def union_search(data, tail, tail_ids, q, k, nprobes, refine_factor=0, lower=None, upper=None, allow=None,
                 max_nprobes=0, ef=0):
    return merge(index_search(data, q, k, nprobes, refine_factor, lower, upper, allow, max_nprobes, ef),
                 tail_search(data, tail, tail_ids, q, k, lower, upper, allow), k)

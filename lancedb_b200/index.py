"""IVF_PQ, IVF_SQ, IVF_HNSW_SQ, IVF_RQ and binary IVF_FLAT index containers and trainers.

`IvfPqIndexData` is the plain-array form of a Lance IVF_PQ index: exactly the arrays
the reference's search path consumes after `prewarm_index`
(rust/lancedb/src/table.rs:3283-3286) -- IVF centroids, PQ codebook, per-partition
transposed PQ codes and row ids.  The same arrays are handed to the C-ABI
(`lgpu_index_open`, include/lancedb_b200.h) and to the CPU oracle.

`train_ivf_pq` mirrors the *parameters* of `Index::IvfPq`
(rust/lancedb/src/index/vector.rs:266-319, rust/lancedb/src/table/create_index.rs:68-102,
283-303): num_partitions, num_sub_vectors (default dim/16, else dim/8, else 1; rounded up to
even for 4 bits), num_bits = 8 or 4, sample_rate = 256, max_iterations = 50, distance_type.  Training itself
lives in the un-vendored lance crate; this is a plain k-means / PQ trainer written with
torch ops (CPU or CUDA), or, with `native_passes` (the `accelerator="cuda"` build), the library's own
training kernels (csrc/kmeans.cu) -- index *quality* is not on the hot path, and both the CUDA
path and the oracle consume the identical arrays it produces.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Optional, Tuple

import numpy as np

METRICS = ("l2", "cosine", "dot")


def suggested_num_sub_vectors(dim: int) -> int:
    """rust/lancedb/src/index/vector.rs:306-319"""
    if dim % 16 == 0:
        return dim // 16
    if dim % 8 == 0:
        return dim // 8
    return 1


def get_num_sub_vectors(provided: Optional[int], dim: int, num_bits: Optional[int]) -> int:
    """rust/lancedb/src/table/create_index.rs:86-102: the explicit value, else suggested_num_sub_vectors(dim) rounded up
    to an even number for 4-bit codes (two codes share a byte)."""
    if provided is not None:
        return int(provided)
    s = suggested_num_sub_vectors(dim)
    return s + 1 if num_bits == 4 and s % 2 else s


PQ4_MAX_M = 256             # LGPU_PQ4_MAX_M: a probe slot's quantised sum stays below 2^16


def suggested_num_partitions(num_rows: int, target_partition_size: int = 8192) -> int:
    """Default IVF sizing: 16384 rows => 2 partitions
    (rust/lancedb/src/table/create_index.rs:734-795)."""
    return max(1, num_rows // target_partition_size)


def _check_ivf_layout(d, width: int, dtype) -> None:
    """The layout every IVF index shares: centroids [nlist, width] of `dtype`, u64 part_offsets [nlist+1] running from
    0 to nrows, u64 row ids."""
    assert d.centroids.shape == (d.nlist, width) and d.centroids.dtype == dtype
    assert d.part_offsets.shape == (d.nlist + 1,) and d.part_offsets.dtype == np.uint64
    assert int(d.part_offsets[0]) == 0 and int(d.part_offsets[-1]) == d.nrows
    assert d.row_ids.dtype == np.uint64


def _partition_order(assign, nlist: int, row_ids):
    """Rows grouped by partition, ascending row id within each: (order, a torch tensor of row positions;
    part_offsets u64 [nlist+1]; the row ids (0..n-1 when row_ids is None) as u64 in that order)."""
    import torch
    assign = torch.as_tensor(assign)
    order = torch.argsort(assign, stable=True)
    part_offsets = np.zeros(nlist + 1, np.uint64)
    part_offsets[1:] = np.cumsum(torch.bincount(assign, minlength=nlist).cpu().numpy())
    rid = np.arange(assign.shape[0], dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    return order, part_offsets, rid[order.cpu().numpy()]


def _normalise(x):
    """Rows scaled to unit length, as a cosine index stores and encodes them (torch, any device)."""
    return x / x.norm(dim=1, keepdim=True).clamp(min=1e-30)


def _extend_order(part_offsets, assign, row_ids):
    """Where appended rows go: every partition keeps its rows in their order and takes its new rows after them, in
    row-id order.  Returns (order over [old rows, new rows] giving the extended partition order, the new part_offsets
    u64 [nlist+1], the new rows' ids u64)."""
    off = np.asarray(part_offsets, np.int64)
    nlist, n0 = off.size - 1, int(off[-1])
    rid = np.asarray(row_ids, np.uint64).reshape(-1)
    a = np.asarray(assign, np.int64).reshape(-1)
    by_id = np.argsort(rid, kind="stable")
    label = np.concatenate([np.repeat(np.arange(nlist), np.diff(off)), a[by_id]])
    order = np.argsort(label, kind="stable")
    order = np.where(order < n0, order, n0 + by_id[np.maximum(order - n0, 0)])
    new_off = np.zeros(nlist + 1, np.uint64)
    new_off[1:] = np.cumsum(np.bincount(label, minlength=nlist))
    return order, new_off, rid


def _compact_offsets(d, keep):
    """The rows `keep` (bool [n], True = kept) selects from an IVF index `d`, checked, and the part_offsets u64
    [nlist+1] once the others are dropped: every partition keeps its remaining rows in their order."""
    keep = np.asarray(keep, bool).reshape(-1)
    if keep.size != d.nrows:
        raise ValueError("keep must hold one flag per row of the index")
    off = np.asarray(d.part_offsets, np.int64)
    label = np.repeat(np.arange(off.size - 1), np.diff(off))
    new_off = np.zeros(off.size, np.uint64)
    new_off[1:] = np.cumsum(np.bincount(label[keep], minlength=off.size - 1))
    return keep, new_off


def _kept(a, keep):
    """Per-row array `a` (partition order) without the dropped rows (None stays None)."""
    return None if a is None else np.ascontiguousarray(np.asarray(a)[keep])


def _cat_rows(old, new, order):
    """Per-row arrays in the extended partition order (None stays None)."""
    if old is None:
        return None
    return np.ascontiguousarray(np.concatenate([np.asarray(old), np.asarray(new, old.dtype)])[order])


def _float_rows(d, vectors, row_ids, device: int):
    """(raw f32 rows [n, dim], rows as the index encodes them -- normalised for cosine --, partitions u32 [n] by the
    search's own coarse kernels on CUDA device `device`) of rows appended to the float IVF index `d`."""
    import torch
    from . import _native
    raw = np.ascontiguousarray(vectors, np.float32).reshape(-1, d.dim)
    if np.asarray(row_ids).size != raw.shape[0]:
        raise ValueError("row_ids must hold one id per appended row")
    x = torch.as_tensor(raw)
    if d.metric == "cosine":
        x = _normalise(x)
    parts = _native.ivf_assign(d.centroids, raw, d.metric, device) if raw.shape[0] else np.zeros(0, np.uint32)
    return raw, x, parts


def _transpose_codes(codes_sorted: np.ndarray, part_offsets) -> np.ndarray:
    """Row-major codes [n, w] in partition order -> the flat per-partition transposed layout ([w][n_p] each)."""
    n, w = codes_sorted.shape
    codes_t = np.empty(n * w, np.uint8)
    for p in range(len(part_offsets) - 1):
        a, b = int(part_offsets[p]), int(part_offsets[p + 1])
        if b > a:
            codes_t[a * w:b * w] = codes_sorted[a:b].T.reshape(-1)
    return codes_t


@dataclass
class IvfPqIndexData:
    index_type = "IVF_PQ"
    dim: int
    nlist: int
    m: int
    metric: str
    centroids: np.ndarray      # f32 [nlist, dim]
    codebook: np.ndarray       # f32 [m, 2**num_bits, dim/m]
    part_offsets: np.ndarray   # u64 [nlist+1]
    codes_t: np.ndarray        # u8 flat; partition p at [off[p]*w, off[p+1]*w) as [w][n_p], w = code_bytes
    row_ids: np.ndarray        # u64 [n] in partition order
    vectors: Optional[np.ndarray] = None   # f32 [n, dim] partition order (refine), optional
    num_bits: int = 8          # 8: one code per byte; 4: byte j holds sub-vector 2j (bits 0-3) and 2j+1 (bits 4-7)

    @property
    def nrows(self) -> int:
        return int(self.row_ids.size)

    @property
    def dsub(self) -> int:
        return self.dim // self.m

    @property
    def code_bytes(self) -> int:
        """Bytes of one row's codes: m (8-bit) or m / 2 (4-bit)."""
        return self.m if self.num_bits == 8 else self.m // 2

    def validate(self) -> None:
        assert self.metric in METRICS
        assert self.num_bits in (4, 8)
        assert self.dim % self.m == 0
        if self.num_bits == 4:
            assert self.m % 2 == 0 and self.m <= PQ4_MAX_M
        _check_ivf_layout(self, self.dim, np.float32)
        assert self.codebook.shape == (self.m, 1 << self.num_bits, self.dsub) and self.codebook.dtype == np.float32
        assert self.codes_t.dtype == np.uint8 and self.codes_t.size == self.nrows * self.code_bytes

    def partition_codes(self, p: int) -> np.ndarray:
        """[code_bytes, n_p] code bytes of partition p."""
        a, b = int(self.part_offsets[p]), int(self.part_offsets[p + 1])
        w = self.code_bytes
        return self.codes_t[a * w:b * w].reshape(w, b - a)

    def row_codes(self) -> np.ndarray:
        """[n, code_bytes] code bytes of every row, row-major in partition order."""
        return np.concatenate([self.partition_codes(p).T for p in range(self.nlist)]) if self.nrows else \
            np.zeros((0, self.code_bytes), np.uint8)

    def extend(self, vectors, row_ids, device: int = 0) -> "IvfPqIndexData":
        """The index with rows appended, without retraining: each row goes to the partition the search's coarse step
        ranks first (lgpu_ivf_assign) and is encoded against its centroid with the index's codebook -- lgpu_pq_encode
        for 8-bit codes, pq_codes for 4-bit ones -- and lands after the partition's rows (_extend_order)."""
        import torch
        from . import _native
        raw, x, parts = _float_rows(self, vectors, row_ids, device)
        if self.num_bits == 8:
            codes = (_native.pq_encode(self.centroids, self.codebook, raw, parts, self.metric, device) if raw.shape[0]
                     else np.zeros((0, self.m), np.uint8))
        else:
            codes = pack_pq4(pq_codes(x, torch.as_tensor(self.centroids), torch.as_tensor(parts.astype(np.int64)),
                                      torch.as_tensor(self.codebook), self.metric).numpy())
        order, off, rid = _extend_order(self.part_offsets, parts, row_ids)
        data = IvfPqIndexData(self.dim, self.nlist, self.m, self.metric, self.centroids, self.codebook, off,
                              _transpose_codes(_cat_rows(self.row_codes(), codes, order), off),
                              _cat_rows(self.row_ids, rid, order), _cat_rows(self.vectors, raw, order), self.num_bits)
        data.validate()
        return data

    def compact(self, keep) -> "IvfPqIndexData":
        """The index without the rows whose `keep` flag (bool [n], partition order) is False, without retraining: the
        other rows keep their partitions, order and ids; each partition's codes are transposed again (4-bit rows keep
        their packed bytes)."""
        keep, off = _compact_offsets(self, keep)
        data = IvfPqIndexData(self.dim, self.nlist, self.m, self.metric, self.centroids, self.codebook, off,
                              _transpose_codes(_kept(self.row_codes(), keep), off), _kept(self.row_ids, keep),
                              _kept(self.vectors, keep), self.num_bits)
        data.validate()
        return data

    def shard(self, rank: int, world: int) -> "IvfPqIndexData":
        """Partition-sharded view for multi-GPU search (SURVEY.md 8e): centroids and
        codebook replicated, each partition's codes/row ids owned by exactly one rank
        (greedy size-balanced); non-owned partitions become empty."""
        sizes = np.diff(self.part_offsets.astype(np.int64))
        owner = assign_partitions(sizes, world)
        keep = owner == rank
        new_sizes = np.where(keep, sizes, 0)
        new_off = np.zeros(self.nlist + 1, np.uint64)
        new_off[1:] = np.cumsum(new_sizes)
        codes, rids, vecs = [], [], []
        for p in np.nonzero(keep)[0]:
            a, b = int(self.part_offsets[p]), int(self.part_offsets[p + 1])
            codes.append(self.codes_t[a * self.code_bytes:b * self.code_bytes])
            rids.append(self.row_ids[a:b])
            if self.vectors is not None:
                vecs.append(self.vectors[a:b])
        cat = lambda xs, dt, shape: (np.concatenate(xs) if xs else np.zeros(shape, dt))
        return IvfPqIndexData(
            self.dim, self.nlist, self.m, self.metric, self.centroids, self.codebook, new_off,
            cat(codes, np.uint8, (0,)), cat(rids, np.uint64, (0,)),
            cat(vecs, np.float32, (0, self.dim)) if self.vectors is not None else None, self.num_bits)


def assign_partitions(sizes: np.ndarray, world: int) -> np.ndarray:
    """Greedy size-balanced bin packing of partitions onto ranks (largest first)."""
    owner = np.zeros(len(sizes), np.int64)
    load = np.zeros(world, np.int64)
    for p in np.argsort(-sizes, kind="stable"):
        r = int(np.argmin(load))
        owner[p] = r
        load[r] += int(sizes[p])
    return owner


# --------------------------------------------------------------------------------------
def _kmeans(x, k, iters, gen, chunk=1 << 16):
    """Lloyd k-means with torch ops; x [n, d] float32 (any device)."""
    import torch
    n = x.shape[0]
    perm = torch.randperm(n, generator=gen, device="cpu")[:k].to(x.device)
    c = x[perm].clone()
    if c.shape[0] < k:      # fewer points than centroids: pad with jittered copies
        extra = x[torch.randint(0, n, (k - c.shape[0],), generator=gen, device="cpu").to(x.device)]
        c = torch.cat([c, extra + 1e-3 * torch.randn(extra.shape, generator=gen).to(x.device)])
    assign = torch.empty(n, dtype=torch.long, device=x.device)
    for _ in range(max(1, iters)):
        cn = (c * c).sum(1)
        for s in range(0, n, chunk):
            xs = x[s:s + chunk]
            assign[s:s + chunk] = (cn[None, :] - 2.0 * (xs @ c.T)).argmin(1)
        sums = torch.zeros_like(c).index_add_(0, assign, x)
        cnt = torch.bincount(assign, minlength=k).to(x.dtype)
        empty = cnt == 0
        c = torch.where(empty[:, None], c, sums / cnt.clamp(min=1)[:, None])
        if empty.any():     # re-seed empty clusters from random points
            ne = int(empty.sum())
            idx = torch.randint(0, n, (ne,), generator=gen, device="cpu").to(x.device)
            c[empty] = x[idx]
    return c


def _init_rows(x, k, gen):
    """k initial centres: distinct random rows (jittered copies when there are fewer rows than centres)."""
    import torch
    n = x.shape[0]
    c = x[torch.randperm(n, generator=gen, device="cpu")[:k].to(x.device)].clone()
    if c.shape[0] < k:
        extra = x[torch.randint(0, n, (k - c.shape[0],), generator=gen, device="cpu").to(x.device)]
        c = torch.cat([c, extra + 1e-3 * torch.randn(extra.shape, generator=gen).to(x.device)])
    return c


def _assign(x, c, chunk=1 << 16, metric="l2"):
    """Partition of every row, ranked like the search's coarse step: L2 for l2/cosine, 1 - x.c for dot."""
    import torch
    n = x.shape[0]
    out = torch.empty(n, dtype=torch.long, device=x.device)
    cn = (c * c).sum(1)
    for s in range(0, n, chunk):
        xc = x[s:s + chunk] @ c.T
        out[s:s + chunk] = (-xc).argmin(1) if metric == "dot" else (cn[None, :] - 2.0 * xc).argmin(1)
    return out


def _batched_kmeans(x, k, iters, gen):
    """x [m, ns, dsub] -> centroids [m, k, dsub], all sub-spaces at once."""
    import torch
    m, ns, _ = x.shape
    idx = torch.stack([torch.randperm(ns, generator=gen, device="cpu")[:k] for _ in range(m)]).to(x.device)
    if idx.shape[1] < k:
        pad = torch.randint(0, ns, (m, k - idx.shape[1]), generator=gen, device="cpu").to(x.device)
        idx = torch.cat([idx, pad], 1)
    c = torch.gather(x, 1, idx[:, :, None].expand(-1, -1, x.shape[2])).clone()
    for _ in range(max(1, iters)):
        cn = (c * c).sum(2)                                       # [m, k]
        a = (cn[:, None, :] - 2.0 * torch.bmm(x, c.transpose(1, 2))).argmin(2)   # [m, ns]
        sums = torch.zeros_like(c).scatter_add_(1, a[:, :, None].expand(-1, -1, x.shape[2]), x)
        cnt = torch.zeros(m, k, device=x.device, dtype=x.dtype).scatter_add_(
            1, a, torch.ones_like(a, dtype=x.dtype))
        c = torch.where((cnt == 0)[:, :, None], c, sums / cnt.clamp(min=1)[:, :, None])
    return c


def _train_ivf(x, nlist, metric, sample_rate, max_iterations, gen, native_passes):
    """The IVF half of an index build: rows normalised for cosine (the index stores normalised vectors; search is L2 on
    them), a training sample of sample_rate rows per partition, k-means centroids and every row's partition.
    native_passes: the Lloyd loops and the assignment run in the library's kernels (lgpu_kmeans_train /
    lgpu_ivf_assign), so a row lands in the partition its own vector probes first.
    Returns (x normalised for cosine, sample, centroids, assign, device ordinal).
    A NaN or infinite component anywhere is refused: k-means would spread it into a centroid, and a row with no finite
    centroid distance has no partition.  So is an all-zero row under cosine (any row whose squared norm is 0 in f32): it
    has no direction, and its distance to every centroid is NaN."""
    import torch
    bad = ~torch.isfinite(x).all(dim=1)
    if bool(bad.any()):
        raise ValueError(f"vector {int(bad.nonzero()[0, 0])} holds a NaN or infinite value; IVF training needs finite "
                         f"vectors")
    if metric == "cosine":
        zero = (x * x).sum(dim=1) == 0
        if bool(zero.any()):
            raise ValueError(f"vector {int(zero.nonzero()[0, 0])} has norm 0; a cosine index needs vectors with a "
                             f"direction")
    n = x.shape[0]
    raw = x
    if metric == "cosine":
        x = _normalise(x)
    ns = min(n, sample_rate * nlist)
    samp = x[torch.randperm(n, generator=gen, device="cpu")[:ns].to(x.device)] if ns < n else x
    dev_index = x.device.index or 0 if x.device.type == "cuda" else 0
    if native_passes:
        # accelerator path: the Lloyd loops run in the library's own kernels (csrc/kmeans.cu through
        # lgpu_kmeans_train): no torch op inside the loop, only the random initial sample is drawn here
        from . import _native
        samp_np = samp.detach().cpu().numpy()
        init = _init_rows(samp, nlist, gen).cpu().numpy()
        centroids = torch.as_tensor(_native.kmeans_train(samp_np, init, max_iterations, dev_index), device=x.device)
        assign = torch.as_tensor(_native.ivf_assign(centroids.cpu().numpy(), raw.detach().cpu().numpy(), metric,
                                                    dev_index).astype(np.int64), device=x.device)
    else:
        centroids = _kmeans(samp, nlist, max_iterations, gen)
        assign = _assign(x, centroids, metric=metric)
    return x, samp, centroids, assign, dev_index


def train_ivf_pq(vectors, *, num_partitions: Optional[int] = None, num_sub_vectors: Optional[int] = None,
                 distance_type: str = "l2", sample_rate: int = 256, max_iterations: int = 50,
                 row_ids: Optional[np.ndarray] = None, keep_vectors: bool = False, seed: int = 45,
                 device: Optional[str] = None, encode_chunk: int = 1 << 16,
                 native_passes: bool = False, num_bits: int = 8) -> IvfPqIndexData:
    """Train IVF centroids + residual PQ codebooks and encode every row.

    vectors: [n, dim] float32 (numpy or torch).  Returns the plain-array index.
    native_passes: run the two passes over every row (IVF assignment, PQ encoding) through the C ABI
    (`lgpu_ivf_assign` / `lgpu_pq_encode`, csrc/build.cu) -- the search kernels' own arithmetic, so a row
    always lands in the partition its own vector probes first -- instead of torch's GEMM-form argmin.
    With native_passes the k-means training loops run in the library too (`lgpu_kmeans_train` / `lgpu_pq_train`,
    csrc/kmeans.cu); otherwise they are torch ops.
    num_bits = 4: 16-codeword codebooks and packed codes (byte j = code 2j | code 2j+1 << 4).  num_sub_vectors defaults
    to get_num_sub_vectors (even) and must be even.  The IVF passes follow native_passes as above; the PQ passes are
    torch ops on the training device either way (`lgpu_pq_train` / `lgpu_pq_encode` are 256-codeword kernels): k-means
    codebooks, and each code the argmin of |c|^2 - 2 r.c, ties to the lowest code.
    """
    import torch
    metric = distance_type.lower()
    if metric not in METRICS:
        raise ValueError(f"unknown distance_type {distance_type!r}")
    if num_bits not in (4, 8):
        raise ValueError(f"IVF_PQ supports num_bits 4 or 8, got num_bits={num_bits}")
    x = torch.as_tensor(vectors, dtype=torch.float32)
    if device is not None:
        x = x.to(device)
    if x.device.type == "cpu" and torch.get_num_threads() > 16:
        # many-core hosts with a small CPU quota: a 100+ thread OpenMP team spins instead of working
        prev = torch.get_num_threads()
        torch.set_num_threads(16)
        try:
            return train_ivf_pq(x, num_partitions=num_partitions, num_sub_vectors=num_sub_vectors,
                                distance_type=distance_type, sample_rate=sample_rate, max_iterations=max_iterations,
                                row_ids=row_ids, keep_vectors=keep_vectors, seed=seed, device=None,
                                encode_chunk=encode_chunk, native_passes=native_passes, num_bits=num_bits)
        finally:
            torch.set_num_threads(prev)
    n, dim = x.shape
    nlist = int(num_partitions or suggested_num_partitions(n))
    m = get_num_sub_vectors(num_sub_vectors or None, dim, num_bits)
    if dim % m:
        raise ValueError(f"num_sub_vectors {m} does not divide dimension {dim}")
    if num_bits == 4 and (m % 2 or m > PQ4_MAX_M):
        raise ValueError(f"4-bit PQ needs an even num_sub_vectors <= {PQ4_MAX_M}, got {m}")
    dsub = dim // m
    gen = torch.Generator(device="cpu").manual_seed(seed)
    raw = x
    x, samp, centroids, assign, dev_index = _train_ivf(x, nlist, metric, sample_rate, max_iterations, gen, native_passes)
    pq_native = native_passes and num_bits == 8       # the library's PQ kernels are 256-codeword
    if pq_native:
        from . import _native
        raw_np = raw.detach().cpu().numpy()

    # PQ codebooks: residuals for l2/cosine, raw vectors for dot
    nps = min(n, max(256, sample_rate) * 256)
    pidx = torch.randperm(n, generator=gen, device="cpu")[:nps].to(x.device)
    ps = x[pidx] - centroids[assign[pidx]] if metric != "dot" else x[pidx]
    if pq_native:
        init_cb = torch.stack([ps[torch.randperm(nps, generator=gen, device="cpu")[:256].to(x.device) if nps >= 256
                                  else torch.randint(0, nps, (256,), generator=gen, device="cpu").to(x.device)]
                               .reshape(256, m, dsub)[:, i, :] for i in range(m)])              # [m, 256, dsub]
        codebook = torch.as_tensor(_native.pq_train(ps.detach().cpu().numpy(), init_cb.cpu().numpy(), max_iterations,
                                                    dev_index), device=x.device)
    else:
        ps3 = ps.reshape(nps, m, dsub).transpose(0, 1).contiguous()      # [m, nps, dsub]
        codebook = _batched_kmeans(ps3, 1 << num_bits, max_iterations, gen)   # [m, 2**num_bits, dsub]

    if pq_native:
        codes = torch.as_tensor(_native.pq_encode(centroids.cpu().numpy(), codebook.cpu().numpy(), raw_np,
                                                  assign.cpu().numpy().astype(np.uint32), metric, dev_index),
                                device=x.device)
    else:
        codes = pq_codes(x, centroids, assign, codebook, metric, encode_chunk)

    order, part_offsets, rid = _partition_order(assign, nlist, row_ids)
    codes_sorted = codes[order].cpu().numpy()                              # [n, m] partition order
    if num_bits == 4:
        codes_sorted = pack_pq4(codes_sorted)                              # [n, m/2]
    codes_t = _transpose_codes(codes_sorted, part_offsets)
    data = IvfPqIndexData(
        dim=dim, nlist=nlist, m=m, metric=metric,
        centroids=centroids.cpu().numpy().astype(np.float32),
        codebook=codebook.cpu().numpy().astype(np.float32),
        part_offsets=part_offsets, codes_t=codes_t, row_ids=rid,
        vectors=(raw[order].cpu().numpy().astype(np.float32) if keep_vectors else None), num_bits=num_bits)
    data.validate()
    return data


def pq_codes(x, centroids, assign, codebook, metric: str, chunk: int = 1 << 16):
    """Codes [n, m] (torch u8) of rows x (normalised for cosine) in partitions `assign`: per sub-space the argmin over
    the codewords of |c|^2 - 2 r.c, r the residual (the row itself for dot), ties to the lowest code."""
    import torch
    m, _, dsub = codebook.shape
    cbn = (codebook * codebook).sum(2)                                     # [m, 2**num_bits]
    codes = torch.empty((x.shape[0], m), dtype=torch.uint8, device=x.device)
    for s in range(0, x.shape[0], chunk):
        xs = x[s:s + chunk]
        r = xs - centroids[assign[s:s + chunk]] if metric != "dot" else xs
        r = r.reshape(-1, m, dsub).transpose(0, 1)                         # [m, c, dsub]
        d = cbn[:, None, :] - 2.0 * torch.bmm(r, codebook.transpose(1, 2))
        codes[s:s + chunk] = d.argmin(2).transpose(0, 1).to(torch.uint8)
    return codes


def pack_pq4(codes) -> np.ndarray:
    """[n, m] 4-bit codes (m even) -> [n, m/2] bytes, byte j = code 2j | code 2j+1 << 4 (lance's packing, recalled)."""
    c = np.asarray(codes, np.uint8)
    if c.shape[-1] % 2 or (c.size and int(c.max()) > 15):
        raise ValueError("4-bit codes need an even number of sub-vectors and values below 16")
    return (c[..., 0::2] | (c[..., 1::2] << 4)).astype(np.uint8)


def unpack_pq4(packed) -> np.ndarray:
    """The inverse of pack_pq4: [n, m/2] bytes -> [n, m] codes."""
    b = np.asarray(packed, np.uint8)
    out = np.empty(b.shape[:-1] + (2 * b.shape[-1],), np.uint8)
    out[..., 0::2] = b & 15
    out[..., 1::2] = b >> 4
    return out


# --------------------------------------------------------------------------------------
SQ_METRICS = ("l2", "cosine")
SQ_MAX_DIM = 65536          # LGPU_SQ_MAX_DIM: the exact integer distance stays below 2^32


@dataclass
class IvfSqIndexData:
    """The plain-array form of an IVF_SQ index (lance `IvfSq`, rust/lancedb/src/index/vector.rs:216-256): IVF centroids,
    one global quantiser range [lo, hi] and one 8-bit code per dimension of every row, grouped by partition.  The same
    arrays go to `lgpu_ivf_sq_open` and to the CPU oracle (tests/sq_oracle.c)."""
    index_type = "IVF_SQ"
    dim: int
    nlist: int
    metric: str
    centroids: np.ndarray      # f32 [nlist, dim]
    part_offsets: np.ndarray   # u64 [nlist+1]
    codes: np.ndarray          # u8 [n, dim] partition order
    row_ids: np.ndarray        # u64 [n] in partition order
    lo: float                  # quantiser bounds (f64)
    hi: float
    vectors: Optional[np.ndarray] = None   # f32 [n, dim] partition order (refine), optional

    @property
    def nrows(self) -> int:
        return int(self.row_ids.size)

    def validate(self) -> None:
        assert self.metric in SQ_METRICS
        assert 1 <= self.dim <= SQ_MAX_DIM
        _check_ivf_layout(self, self.dim, np.float32)
        assert self.codes.shape == (self.nrows, self.dim) and self.codes.dtype == np.uint8
        assert np.isfinite(self.lo) and np.isfinite(self.hi) and self.lo <= self.hi

    def extend(self, vectors, row_ids, device: int = 0) -> "IvfSqIndexData":
        """The index with rows appended, without retraining: partitions from lgpu_ivf_assign, codes from sq_encode
        with the index's [lo, hi] (rows normalised for cosine); each partition's new rows follow its old ones."""
        raw, x, parts = _float_rows(self, vectors, row_ids, device)
        order, off, rid = _extend_order(self.part_offsets, parts, row_ids)
        data = IvfSqIndexData(self.dim, self.nlist, self.metric, self.centroids, off,
                              _cat_rows(self.codes, sq_encode(x.numpy(), self.lo, self.hi), order),
                              _cat_rows(self.row_ids, rid, order), self.lo, self.hi,
                              _cat_rows(self.vectors, raw, order))
        data.validate()
        return data

    def compact(self, keep) -> "IvfSqIndexData":
        """The index without the rows whose `keep` flag is False (IvfPqIndexData.compact)."""
        keep, off = _compact_offsets(self, keep)
        data = IvfSqIndexData(self.dim, self.nlist, self.metric, self.centroids, off, _kept(self.codes, keep),
                              _kept(self.row_ids, keep), self.lo, self.hi, _kept(self.vectors, keep))
        data.validate()
        return data


def sq_encode(x, lo: float, hi: float) -> np.ndarray:
    """lance's scale_to_u8 [lance, recalled]: sat_u8(((double)v - lo) * 255 / (hi - lo)), left to right in f64,
    truncated toward zero; below 0 -> 0, above 255 -> 255, NaN -> 0; every code 0 when lo == hi.  The clipping is
    explicit: a float -> uint8 cast is undefined outside [0, 256) and for NaN."""
    v = np.asarray(x, np.float32).astype(np.float64)
    lo, hi = float(lo), float(hi)
    if hi == lo:
        return np.zeros(v.shape, np.uint8)
    with np.errstate(invalid="ignore", over="ignore"):
        t = ((v - lo) * 255.0) / (hi - lo)
    t = np.where(np.isnan(t), 0.0, t)
    return np.trunc(np.clip(t, 0.0, 255.0)).astype(np.uint8)


def train_ivf_sq(vectors, *, num_partitions: Optional[int] = None, distance_type: str = "l2", sample_rate: int = 256,
                 max_iterations: int = 50, row_ids: Optional[np.ndarray] = None, keep_vectors: bool = False,
                 seed: int = 45, device: Optional[str] = None, native_passes: bool = False) -> IvfSqIndexData:
    """Train IVF centroids (the IVF half of train_ivf_pq), take [lo, hi] = the min and max over every component of the
    training sample (normalised for cosine), and encode every row (normalised for cosine) with sq_encode."""
    import torch
    metric = distance_type.lower()
    if metric not in SQ_METRICS:
        raise ValueError(f"IVF_SQ supports the l2 and cosine distance types, not {distance_type!r}")
    x = torch.as_tensor(vectors, dtype=torch.float32)
    if device is not None:
        x = x.to(device)
    n, dim = x.shape
    if not 1 <= dim <= SQ_MAX_DIM:
        raise ValueError(f"IVF_SQ supports dimensions 1..{SQ_MAX_DIM}, got {dim}")
    nlist = int(num_partitions or suggested_num_partitions(n))
    gen = torch.Generator(device="cpu").manual_seed(seed)
    raw = x
    x, samp, centroids, assign, _ = _train_ivf(x, nlist, metric, sample_rate, max_iterations, gen, native_passes)
    s = samp.detach().cpu().numpy()
    lo, hi = (float(np.min(s)), float(np.max(s))) if s.size else (0.0, 0.0)
    order, part_offsets, rid = _partition_order(assign, nlist, row_ids)
    data = IvfSqIndexData(
        dim=dim, nlist=nlist, metric=metric, centroids=centroids.cpu().numpy().astype(np.float32),
        part_offsets=part_offsets, codes=sq_encode(x[order].cpu().numpy(), lo, hi), row_ids=rid,
        lo=lo, hi=hi, vectors=(raw[order].cpu().numpy().astype(np.float32) if keep_vectors else None))
    data.validate()
    return data


# --------------------------------------------------------------------------------------
RQ_METRICS = ("l2", "cosine")
RQ_MAX_DIM = 4096           # LGPU_RQ_MAX_DIM: P is at most 64 MB, the scan's integers stay exact in f32


@dataclass
class IvfRqIndexData:
    """The plain-array form of an IVF_RQ index (lance `IvfRq`, RaBitQ with num_bits = 1; rust/lancedb/src/index/
    vector.rs:321-369): IVF centroids, one f32 orthogonal rotation P and, for every row of partition p with
    o = P (x - c_p), one sign bit per dimension (LSB first) and the factors add = |o|^2, scale = -2 |o|^2 / sum |o_i|,
    grouped by partition.  The same arrays go to `lgpu_ivf_rq_open` and to the CPU oracle (tests/rq_oracle.c)."""
    index_type = "IVF_RQ"
    dim: int
    nlist: int
    metric: str
    centroids: np.ndarray      # f32 [nlist, dim]
    rotation: np.ndarray       # f32 [dim, dim]
    part_offsets: np.ndarray   # u64 [nlist+1]
    codes: np.ndarray          # u8 [n, ceil(dim / 8)] partition order
    add_factors: np.ndarray    # f32 [n]
    scale_factors: np.ndarray  # f32 [n]
    row_ids: np.ndarray        # u64 [n] in partition order
    vectors: Optional[np.ndarray] = None   # f32 [n, dim] partition order (refine), optional
    num_bits: int = 1

    @property
    def nrows(self) -> int:
        return int(self.row_ids.size)

    def validate(self) -> None:
        assert self.metric in RQ_METRICS and self.num_bits == 1
        assert 1 <= self.dim <= RQ_MAX_DIM
        _check_ivf_layout(self, self.dim, np.float32)
        assert self.rotation.shape == (self.dim, self.dim) and self.rotation.dtype == np.float32
        assert self.codes.shape == (self.nrows, (self.dim + 7) // 8) and self.codes.dtype == np.uint8
        assert self.add_factors.shape == (self.nrows,) and self.add_factors.dtype == np.float32
        assert self.scale_factors.shape == (self.nrows,) and self.scale_factors.dtype == np.float32

    def extend(self, vectors, row_ids, device: int = 0) -> "IvfRqIndexData":
        """The index with rows appended, without retraining: partitions from lgpu_ivf_assign, sign bits and factors from
        rq_encode against the assigned centroid with the index's rotation; each partition's new rows follow its old
        ones."""
        raw, x, parts = _float_rows(self, vectors, row_ids, device)
        codes, add, scale = rq_encode(x, self.centroids, parts.astype(np.int64), self.rotation)
        order, off, rid = _extend_order(self.part_offsets, parts, row_ids)
        data = IvfRqIndexData(self.dim, self.nlist, self.metric, self.centroids, self.rotation, off,
                              _cat_rows(self.codes, codes, order), _cat_rows(self.add_factors, add, order),
                              _cat_rows(self.scale_factors, scale, order), _cat_rows(self.row_ids, rid, order),
                              _cat_rows(self.vectors, raw, order), self.num_bits)
        data.validate()
        return data

    def compact(self, keep) -> "IvfRqIndexData":
        """The index without the rows whose `keep` flag is False (IvfPqIndexData.compact)."""
        keep, off = _compact_offsets(self, keep)
        data = IvfRqIndexData(self.dim, self.nlist, self.metric, self.centroids, self.rotation, off,
                              _kept(self.codes, keep), _kept(self.add_factors, keep), _kept(self.scale_factors, keep),
                              _kept(self.row_ids, keep), _kept(self.vectors, keep), self.num_bits)
        data.validate()
        return data


def rq_rotation(dim: int, seed: int = 45, device=None) -> np.ndarray:
    """P: the Q of the QR of a seeded standard-normal f64 [dim, dim] matrix, its columns multiplied by sign(diag(R))
    (so P is Haar-distributed), cast to f32."""
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn((dim, dim), generator=g, dtype=torch.float64).to(device or "cpu")
    q, r = torch.linalg.qr(a)
    s = torch.sign(torch.diagonal(r))
    s = torch.where(s == 0, torch.ones_like(s), s)
    return (q * s[None, :]).to(torch.float32).cpu().numpy()


def rq_encode(x, centroids, assign, rotation, chunk: int = 1 << 16):
    """(codes [n, ceil(dim / 8)] u8, add [n] f32, scale [n] f32) of rows x (already normalised for cosine) in partitions
    `assign`: o = P (x - c_p) in f64 (from the f32 values), bit i = [o_i > 0] (bit i & 7 of byte i >> 3),
    add = f32(sum o_i^2), scale = f32(-2 sum o_i^2 / sum |o_i|), both 0 when sum |o_i| = 0.  torch ops on x's device."""
    import torch
    x = torch.as_tensor(x)
    dev = x.device
    c = torch.as_tensor(centroids, device=dev).to(torch.float64)
    P = torch.as_tensor(rotation, device=dev).to(torch.float64)
    a = torch.as_tensor(assign, device=dev).long()
    n, dim = x.shape
    nb = (dim + 7) // 8
    codes = np.zeros((n, nb), np.uint8)
    add = np.zeros(n, np.float32)
    scale = np.zeros(n, np.float32)
    w = (2 ** torch.arange(8, device=dev, dtype=torch.int64))
    for s in range(0, n, chunk):
        o = (x[s:s + chunk].to(torch.float64) - c[a[s:s + chunk]]) @ P.T
        bits = (o > 0).to(torch.int64)
        pad = nb * 8 - dim
        if pad:
            bits = torch.nn.functional.pad(bits, (0, pad))
        codes[s:s + chunk] = (bits.reshape(-1, nb, 8) * w).sum(2).to(torch.uint8).cpu().numpy()
        n2 = (o * o).sum(1)
        l1 = o.abs().sum(1)
        sc = torch.where(l1 > 0, -2.0 * n2 / torch.where(l1 > 0, l1, torch.ones_like(l1)), torch.zeros_like(l1))
        add[s:s + chunk] = torch.where(l1 > 0, n2, torch.zeros_like(n2)).to(torch.float32).cpu().numpy()
        scale[s:s + chunk] = sc.to(torch.float32).cpu().numpy()
    return codes, add, scale


def train_ivf_rq(vectors, *, num_partitions: Optional[int] = None, distance_type: str = "l2", num_bits: int = 1,
                 sample_rate: int = 256, max_iterations: int = 50, row_ids: Optional[np.ndarray] = None,
                 keep_vectors: bool = False, seed: int = 45, device: Optional[str] = None,
                 native_passes: bool = False) -> IvfRqIndexData:
    """Train IVF centroids (the IVF half of train_ivf_pq), draw the rotation P (rq_rotation) and encode every row
    (normalised for cosine) with rq_encode, in torch f64 on the given device."""
    import torch
    metric = distance_type.lower()
    if metric not in RQ_METRICS:
        raise ValueError(f"IVF_RQ supports the l2 and cosine distance types, not {distance_type!r}")
    if num_bits != 1:
        raise ValueError(f"IVF_RQ supports num_bits=1 only, got num_bits={num_bits}")
    x = torch.as_tensor(vectors, dtype=torch.float32)
    if device is not None:
        x = x.to(device)
    n, dim = x.shape
    if not 1 <= dim <= RQ_MAX_DIM:
        raise ValueError(f"IVF_RQ supports dimensions 1..{RQ_MAX_DIM}, got {dim}")
    nlist = int(num_partitions or suggested_num_partitions(n))
    gen = torch.Generator(device="cpu").manual_seed(seed)
    raw = x
    x, _, centroids, assign, _ = _train_ivf(x, nlist, metric, sample_rate, max_iterations, gen, native_passes)
    cent = centroids.cpu().numpy().astype(np.float32)
    P = rq_rotation(dim, seed, x.device)
    order, part_offsets, rid = _partition_order(assign, nlist, row_ids)
    codes, add, scale = rq_encode(x[order], cent, assign[order], P)
    data = IvfRqIndexData(
        dim=dim, nlist=nlist, metric=metric, centroids=cent, rotation=P, part_offsets=part_offsets, codes=codes,
        add_factors=add, scale_factors=scale, row_ids=rid,
        vectors=(raw[order].cpu().numpy().astype(np.float32) if keep_vectors else None))
    data.validate()
    return data


# --------------------------------------------------------------------------------------
HAMMING_MAX_BITS = 1 << 24  # binary vectors above 2^24 bits are rejected, as on the flat binary path


@dataclass
class IvfBinaryIndexData:
    """The plain-array form of a binary IVF_FLAT index (lance `IvfFlat` with distance_type "hamming",
    rust/lancedb/src/index/vector.rs:169-209): packed bit-vector centroids and the packed rows grouped by partition.  The
    same arrays go to `lgpu_ivf_binary_open` and to the CPU oracle (tests/ivf_binary_oracle.c)."""
    index_type = "IVF_FLAT"
    nbytes: int
    nlist: int
    centroids: np.ndarray      # u8 [nlist, nbytes] packed bits
    part_offsets: np.ndarray   # u64 [nlist+1]
    vectors: np.ndarray        # u8 [n, nbytes] partition order
    row_ids: np.ndarray        # u64 [n] in partition order
    metric: str = "hamming"

    @property
    def nrows(self) -> int:
        return int(self.row_ids.size)

    def validate(self) -> None:
        assert self.metric == "hamming"
        assert 1 <= self.nbytes and 8 * self.nbytes <= HAMMING_MAX_BITS
        _check_ivf_layout(self, self.nbytes, np.uint8)
        assert self.vectors.shape == (self.nrows, self.nbytes) and self.vectors.dtype == np.uint8

    def extend(self, vectors, row_ids, device: int = 0) -> "IvfBinaryIndexData":
        """The index with rows appended, without retraining: each row goes to its nearest centroid by Hamming distance
        (kmodes_assign, ties to the lower partition) after the partition's rows.  The assignment is exact integer work,
        so it runs on the host whatever `device` is."""
        x = np.ascontiguousarray(vectors, np.uint8).reshape(-1, self.nbytes)
        if np.asarray(row_ids).size != x.shape[0]:
            raise ValueError("row_ids must hold one id per appended row")
        parts = kmodes_assign(x, self.centroids) if x.shape[0] else np.zeros(0, np.int64)
        order, off, rid = _extend_order(self.part_offsets, parts, row_ids)
        data = IvfBinaryIndexData(self.nbytes, self.nlist, self.centroids, off, _cat_rows(self.vectors, x, order),
                                  _cat_rows(self.row_ids, rid, order))
        data.validate()
        return data

    def compact(self, keep) -> "IvfBinaryIndexData":
        """The index without the rows whose `keep` flag is False (IvfPqIndexData.compact)."""
        keep, off = _compact_offsets(self, keep)
        data = IvfBinaryIndexData(self.nbytes, self.nlist, self.centroids, off, _kept(self.vectors, keep),
                                  _kept(self.row_ids, keep))
        data.validate()
        return data


def _unpack_bits(x, device, dtype):
    """packed u8 rows [n, nbytes] -> 0/1 tensor [n, 8 nbytes] (bit i & 7 of byte i >> 3, the packing order)"""
    import torch
    t = torch.as_tensor(np.require(x, np.uint8, ["C", "W"]), device=device)
    shifts = torch.arange(8, device=device, dtype=torch.uint8)
    return ((t[:, :, None] >> shifts) & 1).reshape(t.shape[0], -1).to(dtype)


def kmodes_assign(x, centroids, device=None, chunk: int = 1 << 15) -> np.ndarray:
    """Index of the nearest centroid of every packed row by Hamming distance, ties to the lowest index:
    popc(x XOR c) = popc(x) + popc(c) - 2 x.c over the unpacked bits.  Operands and result are f32 on every device: 0
    and 1 are exact (also when TF32 rounds the operands), every product is exact, and the f32 sums stay exact integers
    below 2^24 bits per row.  (A bf16 result would round x.c above 256.)  The tie rule does not lean on argmin's
    choice among equal values: the key is d * nlist + index, an exact int64."""
    import torch
    dev = torch.device(device or "cpu")
    c = _unpack_bits(centroids, dev, torch.float32)
    k = c.shape[0]
    cpop = c.sum(1)
    idx = torch.arange(k, device=dev, dtype=torch.int64)
    x = np.ascontiguousarray(x, np.uint8)
    out = np.empty(x.shape[0], np.int64)
    chunk = max(1, min(chunk, (1 << 27) // max(8 * x.shape[1], k)))    # unpacked rows and keys: ~1 GB at most
    for s in range(0, x.shape[0], chunk):
        b = _unpack_bits(x[s:s + chunk], dev, torch.float32)
        d = b.sum(1)[:, None] + cpop[None, :] - 2.0 * (b @ c.T)
        key = d.to(torch.int64) * k + idx[None, :]
        out[s:s + chunk] = torch.argmin(key, dim=1).cpu().numpy()
    return out


def kmodes_update(x, assign, centroids, device=None) -> np.ndarray:
    """One k-modes centroid update [lance, recalled: KModeAlgo]: bit j of centroid c is set when 2 ones > members over
    the rows assigned to c (an exact half keeps 0, a project decision); a cluster with no rows keeps its previous
    centroid (a project decision)."""
    import torch
    dev = torch.device(device or "cpu")
    k = centroids.shape[0]
    a = torch.as_tensor(np.asarray(assign, np.int64), device=dev)
    ones = torch.zeros((k, 8 * centroids.shape[1]), dtype=torch.float32, device=dev)
    ones.index_add_(0, a, _unpack_bits(x, dev, torch.float32))
    members = torch.bincount(a, minlength=k).to(torch.float32)
    bits = (2.0 * ones > members[:, None]).to(torch.uint8).cpu().numpy()
    new = np.packbits(bits, axis=1, bitorder="little")
    empty = members.cpu().numpy() == 0
    new[empty] = np.asarray(centroids, np.uint8)[empty]
    return new


def train_ivf_binary(vectors, *, num_partitions: Optional[int] = None, distance_type: str = "hamming",
                     sample_rate: int = 256, max_iterations: int = 50, row_ids: Optional[np.ndarray] = None,
                     seed: int = 45, device: Optional[str] = None) -> IvfBinaryIndexData:
    """Binary IVF_FLAT (IvfFlat with distance_type "hamming"): k-modes over packed bit vectors [n, nbytes].  On a sample
    of min(n, sample_rate nlist) rows (seeded), the initial centroids are nlist distinct sample rows; each of
    max_iterations rounds assigns every sample row to its nearest centroid (kmodes_assign) and updates the centroids
    (kmodes_update).  Every row then lands in its nearest centroid.  All of it is integer work: the result does not
    depend on the device."""
    if distance_type.lower() != "hamming":
        raise ValueError(f"IVF_FLAT over binary vectors supports the hamming distance type only, not {distance_type!r}")
    x = np.ascontiguousarray(vectors, np.uint8)
    if x.ndim != 2 or x.shape[1] < 1:
        raise ValueError("binary vectors must be a [rows, bytes] uint8 array")
    n, nbytes = x.shape
    if 8 * nbytes > HAMMING_MAX_BITS:
        raise ValueError("binary vectors above 2^24 bits are not supported")
    nlist = int(num_partitions or suggested_num_partitions(n))
    if nlist < 1 or nlist > max(n, 1):
        raise ValueError(f"num_partitions must be in [1, {max(n, 1)}] for {n} rows, got {nlist}")
    rng = np.random.default_rng(seed)
    ns = min(n, int(sample_rate) * nlist)
    samp = x[np.sort(rng.choice(n, ns, replace=False))] if ns < n else x
    cent = samp[rng.choice(samp.shape[0], nlist, replace=False)] if n else np.zeros((nlist, nbytes), np.uint8)
    for _ in range(int(max_iterations) if n else 0):
        new = kmodes_update(samp, kmodes_assign(samp, cent, device), cent, device)
        if np.array_equal(new, cent):
            break
        cent = new
    assign = kmodes_assign(x, cent, device) if n else np.zeros(0, np.int64)
    order, part_offsets, rid = _partition_order(assign, nlist, row_ids)
    data = IvfBinaryIndexData(nbytes=nbytes, nlist=nlist, centroids=np.ascontiguousarray(cent, np.uint8),
                              part_offsets=part_offsets, vectors=np.ascontiguousarray(x[order.numpy()]), row_ids=rid)
    data.validate()
    return data


# --------------------------------------------------------------------------------------
HNSW_MAX_M = 64             # LGPU_HNSW_MAX_M: a level-0 list (2m entries) is at most 4 per lane of a warp
HNSW_MAX_LEVEL = 15         # LGPU_HNSW_MAX_LEVEL
HNSW_NONE = 0xFFFFFFFF      # an unused adjacency slot, an empty partition's entry, a level-0 row's upper_index
HNSW_BUILD_CAND_CAP = 128   # candidates the neighbour heuristic looks at, at most (ef_construction above it is capped)


@dataclass
class IvfHnswSqIndexData:
    """The plain-array form of an IVF_HNSW_SQ index (lance `HnswSq`, python/python/lancedb/index.py): an IVF_SQ index
    (`sq`) plus, in every partition, an HNSW graph over its rows.  Positions are row indices within the partition.
      levels       u8  [n]         the level of each row
      adj0         u32 [n, 2m]     level-0 neighbours, padded with HNSW_NONE
      upper_index  u32 [n]         first block of the row's upper adjacency (level L at upper_index + L - 1); HNSW_NONE
                                   for a level-0 row
      upper_adj    u32 [blocks, m] neighbours at levels >= 1, padded with HNSW_NONE
      entry        u32 [nlist]     the entry row of each partition (HNSW_NONE when empty); its level is top_level
      top_level    u8  [nlist]
    The same arrays go to `lgpu_ivf_hnsw_sq_open` and to the CPU oracle (tests/hnsw_sq_oracle.c)."""
    index_type = "IVF_HNSW_SQ"
    sq: IvfSqIndexData
    m: int
    levels: np.ndarray
    adj0: np.ndarray
    upper_index: np.ndarray
    upper_adj: np.ndarray
    entry: np.ndarray
    top_level: np.ndarray
    ef_construction: int = 300       # how the graphs were built: extend rebuilds a partition's graph the same way
    graph_device: Optional[str] = None

    dim = property(lambda self: self.sq.dim)
    nlist = property(lambda self: self.sq.nlist)
    metric = property(lambda self: self.sq.metric)
    nrows = property(lambda self: self.sq.nrows)
    part_offsets = property(lambda self: self.sq.part_offsets)
    row_ids = property(lambda self: self.sq.row_ids)
    vectors = property(lambda self: self.sq.vectors)

    def validate(self) -> None:
        """Every index in range and every degree bound held: what lgpu_ivf_hnsw_sq_open checks."""
        self.sq.validate()
        n, m = self.nrows, self.m
        assert 1 <= m <= HNSW_MAX_M
        assert self.levels.shape == (n,) and self.levels.dtype == np.uint8
        assert self.adj0.shape == (n, 2 * m) and self.adj0.dtype == np.uint32
        assert self.upper_index.shape == (n,) and self.upper_index.dtype == np.uint32
        assert self.upper_adj.ndim == 2 and self.upper_adj.shape[1] == m and self.upper_adj.dtype == np.uint32
        assert self.entry.shape == (self.nlist,) and self.entry.dtype == np.uint32
        assert self.top_level.shape == (self.nlist,) and self.top_level.dtype == np.uint8
        off = self.part_offsets.astype(np.int64)
        nb = self.upper_adj.shape[0]
        for p in range(self.nlist):
            a, b = off[p], off[p + 1]
            if a == b:
                continue
            lv = self.levels[a:b].astype(np.int64)
            top = int(self.top_level[p])
            assert top <= HNSW_MAX_LEVEL and int(self.entry[p]) < b - a and lv[self.entry[p]] == top
            assert lv.max() <= top
            adj = self.adj0[a:b]
            assert ((adj == HNSW_NONE) | (adj < b - a)).all()
            for r in np.nonzero(lv)[0]:
                u = int(self.upper_index[a + r])
                assert u != HNSW_NONE and u + lv[r] <= nb
                for L in range(1, lv[r] + 1):
                    blk = self.upper_adj[u + L - 1]
                    ok = blk == HNSW_NONE
                    ok[~ok] = (blk[~ok] < b - a)
                    assert ok.all() and (lv[blk[blk != HNSW_NONE].astype(np.int64)] >= L).all()


    def extend(self, vectors, row_ids, device: int = 0, seed: int = 45) -> "IvfHnswSqIndexData":
        """IvfSqIndexData.extend, then the graph of every partition that received rows is built again over all of its
        rows (build_hnsw_graph with the index's m, ef_construction and graph device); the other partitions keep their
        graphs."""
        return self._with_rows(self.sq.extend(vectors, row_ids, device), seed)

    def compact(self, keep, seed: int = 45) -> "IvfHnswSqIndexData":
        """IvfSqIndexData.compact, then the graph of every partition that lost rows is built again over the rows it
        keeps, as extend does; the other partitions keep their graphs."""
        return self._with_rows(self.sq.compact(keep), seed)

    def _with_rows(self, sq: IvfSqIndexData, seed: int) -> "IvfHnswSqIndexData":
        """This index's graphs over `sq`, whose partitions hold either this index's rows or a different number of
        rows: the graph of a partition whose row count changed is built again."""
        old, new = self.part_offsets.astype(np.int64), sq.part_offsets.astype(np.int64)
        entry, top = self.entry.copy(), self.top_level.copy()
        lvs, adjs, uas = [], [], []
        for p in range(self.nlist):
            a, b, a2, b2 = old[p], old[p + 1], new[p], new[p + 1]
            if b2 - a2 == b - a:
                lv, adj = self.levels[a:b], self.adj0[a:b]
                up = np.nonzero(lv)[0]
                first = int(self.upper_index[a + up[0]]) if up.size else 0
                ua = self.upper_adj[first:first + int(lv.astype(np.int64).sum())]
            else:
                lv, adj, _, ua, e, t = build_hnsw_graph(sq.codes[a2:b2], np.array([0, b2 - a2]), self.m,
                                                        self.ef_construction, seed, self.graph_device)
                entry[p], top[p] = e[0], t[0]
            lvs.append(lv); adjs.append(adj); uas.append(ua)
        levels = np.concatenate(lvs).astype(np.uint8)
        upper_index = np.full(levels.size, HNSW_NONE, np.uint32)
        up = np.nonzero(levels)[0]
        upper_index[up] = (np.cumsum(levels[up].astype(np.int64)) - levels[up]).astype(np.uint32)
        data = IvfHnswSqIndexData(sq, self.m, levels, np.concatenate(adjs).astype(np.uint32), upper_index,
                                  np.concatenate(uas).astype(np.uint32).reshape(-1, self.m), entry, top,
                                  self.ef_construction, self.graph_device)
        data.validate()
        return data


def _hnsw_candidates(xc, ncand, chunk):
    """The ncand nearest other rows of every row of xc [s, dim] (codes as floats), nearest first, ties to the lower
    position: ([s, C] positions, [s, C] f32 distances), C = min(ncand, s - 1)."""
    import torch
    s = xc.shape[0]
    c = min(ncand, s - 1)
    nx = (xc.float() * xc.float()).sum(1)
    pos = torch.arange(s, device=xc.device, dtype=torch.float64)
    out_i = torch.empty((s, c), dtype=torch.long, device=xc.device)
    out_d = torch.empty((s, c), dtype=torch.float32, device=xc.device)
    for a in range(0, s, chunk):
        b = min(s, a + chunk)
        d = (nx[a:b, None] + nx[None, :] - 2.0 * (xc[a:b] @ xc.T).float()).clamp(min=0)
        key = d.double() * s + pos                       # exact: ties fall to the lower position
        key[torch.arange(b - a, device=xc.device), torch.arange(a, b, device=xc.device)] = float("inf")
        _, idx = torch.topk(key, c, dim=1, largest=False, sorted=True)
        out_i[a:b] = idx
        out_d[a:b] = torch.gather(d, 1, idx)
    return out_i, out_d


def _hnsw_level_graph(xc, deg, ncand, chunk=1024):
    """Neighbour lists [s, deg] (local positions, -1 padded) of the rows xc [s, dim] at one level: the HNSW heuristic
    over each row's nearest candidates (a candidate is kept while fewer than deg are, unless a kept one is nearer to it
    than the row is), then reverse edges, every list pruned to its deg nearest (ties to the lower position)."""
    import torch
    s, dev = xc.shape[0], xc.device
    adj = torch.full((s, deg), -1, dtype=torch.long, device=dev)
    if s <= 1:
        return adj
    cand, cd = _hnsw_candidates(xc, min(ncand, HNSW_BUILD_CAND_CAP), chunk)
    c = cand.shape[1]
    nx = (xc.float() * xc.float()).sum(1)
    srcs, dsts, ds = [], [], []
    hb = max(1, (1 << 27) // max(1, c * xc.shape[1]))   # rows per heuristic batch (bounds the gathered codes)
    for a in range(0, s, hb):
        b = min(s, a + hb)
        ci, dv = cand[a:b], cd[a:b]
        g = xc[ci]                                                           # [b, c, dim]
        pair = (nx[ci][:, :, None] + nx[ci][:, None, :] - 2.0 * torch.bmm(g, g.transpose(1, 2)).float())
        sel = torch.zeros((b - a, c), dtype=torch.bool, device=dev)
        cnt = torch.zeros(b - a, dtype=torch.long, device=dev)
        for j in range(c):
            closer = ((pair[:, j, :] < dv[:, j:j + 1]) & sel).any(1)
            ok = ~closer & (cnt < deg)
            sel[:, j] = ok
            cnt += ok
        r, j = sel.nonzero(as_tuple=True)
        srcs.append(r + a); dsts.append(ci[r, j]); ds.append(dv[r, j])
    src, dst, d = torch.cat(srcs), torch.cat(dsts), torch.cat(ds)
    src, dst, d = torch.cat([src, dst]), torch.cat([dst, src]), torch.cat([d, d])     # reverse edges
    for i in (1, 2, 0):                                                               # sort by (src, d, dst)
        o = torch.sort((src, dst, d)[i], stable=True).indices
        src, dst, d = src[o], dst[o], d[o]
    keep = torch.ones_like(src, dtype=torch.bool)
    keep[1:] = (src[1:] != src[:-1]) | (dst[1:] != dst[:-1])
    src, dst = src[keep], dst[keep]
    first = torch.zeros(s + 1, dtype=torch.long, device=dev)
    first[1:] = torch.cumsum(torch.bincount(src, minlength=s), 0)
    rank = torch.arange(src.numel(), device=dev) - first[src]
    m = rank < deg
    adj[src[m], rank[m]] = dst[m]
    return adj


def build_hnsw_graph(codes, part_offsets, m: int = 20, ef_construction: int = 300, seed: int = 45, device=None):
    """The HNSW graphs of every partition of an IVF_SQ index over its codes [n, dim] (u8, partition order), in the
    IvfHnswSqIndexData layout: (levels, adj0, upper_index, upper_adj, entry, top_level).  Levels are a seeded geometric
    draw, floor(-ln(U) / ln m) capped at HNSW_MAX_LEVEL; each level's lists come from _hnsw_level_graph over the rows of
    that level in the partition (degree 2m at level 0, m above).  Deterministic for a seed on a given device."""
    import math
    import torch
    if not 1 <= m <= HNSW_MAX_M:
        raise ValueError(f"m must be in [1, {HNSW_MAX_M}], got {m}")
    if ef_construction < 1:
        raise ValueError(f"ef_construction must be positive, got {ef_construction}")
    codes = np.ascontiguousarray(codes, np.uint8)
    n = codes.shape[0]
    off = np.asarray(part_offsets, np.int64)
    nlist = off.size - 1
    gen = torch.Generator(device="cpu").manual_seed(seed)
    u = torch.rand(n, generator=gen, dtype=torch.float64).clamp(min=1e-300)
    lv = (-torch.log(u) / math.log(max(m, 2))).floor().clamp(max=HNSW_MAX_LEVEL).to(torch.uint8).numpy()
    dev = torch.device(device) if device is not None else torch.device("cpu")
    ftype = torch.float32          # codes are exact in f32 (and TF32); products and sums accumulate in f32
    adj0 = np.full((n, 2 * m), HNSW_NONE, np.uint32)
    upper_index = np.full(n, HNSW_NONE, np.uint32)
    up = np.nonzero(lv)[0]
    upper_index[up] = (np.cumsum(lv[up].astype(np.int64)) - lv[up]).astype(np.uint32)
    upper_adj = np.full((int(lv.astype(np.int64).sum()), m), HNSW_NONE, np.uint32)
    entry = np.full(nlist, HNSW_NONE, np.uint32)
    top = np.zeros(nlist, np.uint8)
    for p in range(nlist):
        a, b = int(off[p]), int(off[p + 1])
        if a == b:
            continue
        plv = lv[a:b]
        top[p] = plv.max()
        entry[p] = int(np.argmax(plv))                       # the first row of the top level
        xc = torch.as_tensor(codes[a:b], device=dev).to(ftype)
        for L in range(int(top[p]) + 1):
            rows = np.nonzero(plv >= L)[0]
            sub = _hnsw_level_graph(xc[torch.as_tensor(rows, device=dev)], 2 * m if L == 0 else m,
                                    ef_construction).cpu().numpy()
            g = np.where(sub >= 0, rows[np.maximum(sub, 0)], HNSW_NONE).astype(np.uint32)
            if L == 0:
                adj0[a:b] = g
            else:
                upper_adj[upper_index[a + rows].astype(np.int64) + L - 1] = g
    return lv, adj0, upper_index, upper_adj, entry, top


def train_ivf_hnsw_sq(vectors, *, num_partitions: Optional[int] = None, distance_type: str = "l2", m: int = 20,
                      ef_construction: int = 300, sample_rate: int = 256, max_iterations: int = 50,
                      row_ids: Optional[np.ndarray] = None, keep_vectors: bool = False, seed: int = 45,
                      device: Optional[str] = None, native_passes: bool = False) -> IvfHnswSqIndexData:
    """train_ivf_sq, then build_hnsw_graph over its codes (on `device`: torch on the GPU for "cuda", else the CPU)."""
    if not 1 <= m <= HNSW_MAX_M:
        raise ValueError(f"m must be in [1, {HNSW_MAX_M}], got {m}")
    sq = train_ivf_sq(vectors, num_partitions=num_partitions, distance_type=distance_type, sample_rate=sample_rate,
                      max_iterations=max_iterations, row_ids=row_ids, keep_vectors=keep_vectors, seed=seed,
                      device=device, native_passes=native_passes)
    g = build_hnsw_graph(sq.codes, sq.part_offsets, m, ef_construction, seed, device)
    data = IvfHnswSqIndexData(sq, m, *g, ef_construction=ef_construction, graph_device=device)
    data.validate()
    return data


# --------------------------------------------------------------------------------------
@dataclass(frozen=True)
class IvfKind:
    """One IVF index kind as `Table.create_index` builds it: what it accepts, how it is trained and which `_native`
    handle class opens its data.  The refusals are formatted with the value given (`kind`, `metric`, `num_bits`)."""
    index_type: str
    data: type                       # its IndexData class
    train: Callable
    handle: str
    metrics: Tuple[str, ...]
    metric_error: str
    num_bits: Tuple[int, ...] = ()   # () = any: the kind has no num_bits and create_index's is ignored
    num_bits_error: str = ""
    max_dim: Optional[int] = None    # a dimension bound checked before training
    params: Tuple[str, ...] = ()     # create_index arguments passed on to `train` besides the ones every kind takes
    column: str = "float"            # the vector column it indexes: "float" or "binary"


_L2_COSINE = "{kind} supports the l2 and cosine distance types, not {metric!r}"
IVF_KINDS = {k.index_type: k for k in (
    IvfKind("IVF_PQ", IvfPqIndexData, train_ivf_pq, "GpuIvfPq", METRICS, "unknown distance_type {metric!r}", (4, 8),
            "IVF_PQ supports num_bits 4 or 8, got num_bits={num_bits}", params=("num_sub_vectors", "num_bits")),
    IvfKind("IVF_SQ", IvfSqIndexData, train_ivf_sq, "GpuIvfSq", SQ_METRICS, _L2_COSINE, (8,),
            "only num_bits=8 is supported"),
    IvfKind("IVF_HNSW_SQ", IvfHnswSqIndexData, train_ivf_hnsw_sq, "GpuIvfHnswSq", SQ_METRICS, _L2_COSINE, (8,),
            "only num_bits=8 is supported", params=("m", "ef_construction")),
    # RaBitQ with 1 bit per dimension only (extended RaBitQ is not served): the legacy default of 8 is refused rather
    # than quietly building a 1-bit index
    IvfKind("IVF_RQ", IvfRqIndexData, train_ivf_rq, "GpuIvfRq", RQ_METRICS, _L2_COSINE, (1,),
            "IVF_RQ supports num_bits=1 only, got num_bits={num_bits}", max_dim=RQ_MAX_DIM, params=("num_bits",)),
    IvfKind("IVF_FLAT", IvfBinaryIndexData, train_ivf_binary, "GpuIvfBinary", ("hamming",),
            "IVF_FLAT over binary vectors supports the hamming distance type only, not {metric!r}", column="binary"),
)}

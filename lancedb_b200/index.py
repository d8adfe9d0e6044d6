"""IVF_PQ, IVF_SQ, IVF_RQ and binary IVF_FLAT index containers and trainers.

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
from typing import Optional

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


@dataclass
class IvfPqIndexData:
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
        assert self.centroids.shape == (self.nlist, self.dim) and self.centroids.dtype == np.float32
        assert self.codebook.shape == (self.m, 1 << self.num_bits, self.dsub) and self.codebook.dtype == np.float32
        assert self.part_offsets.shape == (self.nlist + 1,) and self.part_offsets.dtype == np.uint64
        assert int(self.part_offsets[-1]) == self.nrows
        assert self.codes_t.dtype == np.uint8 and self.codes_t.size == self.nrows * self.code_bytes
        assert self.row_ids.dtype == np.uint64

    def partition_codes(self, p: int) -> np.ndarray:
        """[code_bytes, n_p] code bytes of partition p."""
        a, b = int(self.part_offsets[p]), int(self.part_offsets[p + 1])
        w = self.code_bytes
        return self.codes_t[a * w:b * w].reshape(w, b - a)

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
    Returns (x normalised for cosine, sample, centroids, assign, device ordinal)."""
    import torch
    n = x.shape[0]
    raw = x
    if metric == "cosine":
        x = x / x.norm(dim=1, keepdim=True).clamp(min=1e-30)
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

    cbn = (codebook * codebook).sum(2)                                     # [m, 256]
    codes = torch.empty((n, m), dtype=torch.uint8, device=x.device)
    if pq_native:
        codes = torch.as_tensor(_native.pq_encode(centroids.cpu().numpy(), codebook.cpu().numpy(), raw_np,
                                                  assign.cpu().numpy().astype(np.uint32), metric, dev_index),
                                device=x.device)
    for s in range(0, n if not pq_native else 0, encode_chunk):
        xs = x[s:s + encode_chunk]
        r = xs - centroids[assign[s:s + encode_chunk]] if metric != "dot" else xs
        r = r.reshape(-1, m, dsub).transpose(0, 1)                         # [m, c, dsub]
        d = cbn[:, None, :] - 2.0 * torch.bmm(r, codebook.transpose(1, 2))
        codes[s:s + encode_chunk] = d.argmin(2).transpose(0, 1).to(torch.uint8)

    order = torch.argsort(assign, stable=True)                            # ascending row id per partition
    sizes = torch.bincount(assign, minlength=nlist).cpu().numpy().astype(np.int64)
    part_offsets = np.zeros(nlist + 1, np.uint64)
    part_offsets[1:] = np.cumsum(sizes)
    codes_sorted = codes[order].cpu().numpy()                              # [n, m] partition order
    if num_bits == 4:
        codes_sorted = pack_pq4(codes_sorted)                              # [n, m/2]
    w = codes_sorted.shape[1]
    codes_t = np.empty(n * w, np.uint8)
    for p in range(nlist):
        a, b = int(part_offsets[p]), int(part_offsets[p + 1])
        if b > a:
            codes_t[a * w:b * w] = codes_sorted[a:b].T.reshape(-1)
    order_np = order.cpu().numpy()
    rid = np.arange(n, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    data = IvfPqIndexData(
        dim=dim, nlist=nlist, m=m, metric=metric,
        centroids=centroids.cpu().numpy().astype(np.float32),
        codebook=codebook.cpu().numpy().astype(np.float32),
        part_offsets=part_offsets, codes_t=codes_t, row_ids=rid[order_np],
        vectors=(raw[order].cpu().numpy().astype(np.float32) if keep_vectors else None), num_bits=num_bits)
    data.validate()
    return data


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
        assert self.centroids.shape == (self.nlist, self.dim) and self.centroids.dtype == np.float32
        assert self.part_offsets.shape == (self.nlist + 1,) and self.part_offsets.dtype == np.uint64
        assert int(self.part_offsets[-1]) == self.nrows
        assert self.codes.shape == (self.nrows, self.dim) and self.codes.dtype == np.uint8
        assert self.row_ids.dtype == np.uint64
        assert np.isfinite(self.lo) and np.isfinite(self.hi) and self.lo <= self.hi


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
    order = torch.argsort(assign, stable=True)                            # ascending row id per partition
    sizes = torch.bincount(assign, minlength=nlist).cpu().numpy().astype(np.int64)
    part_offsets = np.zeros(nlist + 1, np.uint64)
    part_offsets[1:] = np.cumsum(sizes)
    order_np = order.cpu().numpy()
    rid = np.arange(n, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    data = IvfSqIndexData(
        dim=dim, nlist=nlist, metric=metric, centroids=centroids.cpu().numpy().astype(np.float32),
        part_offsets=part_offsets, codes=sq_encode(x[order].cpu().numpy(), lo, hi), row_ids=rid[order_np],
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
        assert self.centroids.shape == (self.nlist, self.dim) and self.centroids.dtype == np.float32
        assert self.rotation.shape == (self.dim, self.dim) and self.rotation.dtype == np.float32
        assert self.part_offsets.shape == (self.nlist + 1,) and self.part_offsets.dtype == np.uint64
        assert int(self.part_offsets[-1]) == self.nrows
        assert self.codes.shape == (self.nrows, (self.dim + 7) // 8) and self.codes.dtype == np.uint8
        assert self.add_factors.shape == (self.nrows,) and self.add_factors.dtype == np.float32
        assert self.scale_factors.shape == (self.nrows,) and self.scale_factors.dtype == np.float32
        assert self.row_ids.dtype == np.uint64


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
    order = torch.argsort(assign, stable=True)                            # ascending row id per partition
    sizes = torch.bincount(assign, minlength=nlist).cpu().numpy().astype(np.int64)
    part_offsets = np.zeros(nlist + 1, np.uint64)
    part_offsets[1:] = np.cumsum(sizes)
    codes, add, scale = rq_encode(x[order], cent, assign[order], P)
    order_np = order.cpu().numpy()
    rid = np.arange(n, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    data = IvfRqIndexData(
        dim=dim, nlist=nlist, metric=metric, centroids=cent, rotation=P, part_offsets=part_offsets, codes=codes,
        add_factors=add, scale_factors=scale, row_ids=rid[order_np],
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
        assert self.centroids.shape == (self.nlist, self.nbytes) and self.centroids.dtype == np.uint8
        assert self.part_offsets.shape == (self.nlist + 1,) and self.part_offsets.dtype == np.uint64
        assert int(self.part_offsets[0]) == 0 and int(self.part_offsets[-1]) == self.nrows
        assert self.vectors.shape == (self.nrows, self.nbytes) and self.vectors.dtype == np.uint8
        assert self.row_ids.dtype == np.uint64


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
    order = np.argsort(assign, kind="stable")                         # ascending row id per partition
    part_offsets = np.zeros(nlist + 1, np.uint64)
    part_offsets[1:] = np.cumsum(np.bincount(assign, minlength=nlist))
    rid = np.arange(n, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    data = IvfBinaryIndexData(nbytes=nbytes, nlist=nlist, centroids=np.ascontiguousarray(cent, np.uint8),
                              part_offsets=part_offsets, vectors=np.ascontiguousarray(x[order]), row_ids=rid[order])
    data.validate()
    return data

"""Partition-sharded IVF_PQ search across GPUs (SURVEY.md 8e): one process per GPU.

IVF partitions are the shardable unit: centroids and the PQ codebook are replicated, each
partition's codes + row ids live on exactly one rank (`IvfPqIndexData.shard`).  Every rank
gets the full query batch, runs the coarse step redundantly (so all ranks agree on the
probe set without communicating), scans only the probed partitions it owns, and produces a
local top-k.  The single exchange step happens INSIDE the library (`lgpu_search_sharded*`):
the local top-k is packed into `[B][k]` 16-byte (`_rowid` u64, `_distance` f32) records, one
`ncclAllGather` moves them over NVLink on the search stream, and the merge kernel re-selects
the global top-k by (_distance, _rowid) straight from the gather buffer.  A host needs no
torch for this: the only thing it has to do is hand rank 0's 128-byte group id
(`lgpu_comm_unique_id`) to every rank; this mirror uses torch.distributed for that.
The reference has no equivalent (LanceDB OSS is single-process; SURVEY.md 2a); it is only
needed where the index exceeds one GPU's HBM -- otherwise replicas with the batch split are
faster (zero communication), which is what bench.py reports as `value`.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from . import _native
from .index import IvfPqIndexData


def gather_shape(world: int, B: int, k: int):
    """Layout of the gathered candidate lists: [world][B][k] records (rank-major), which is what
    the merge (select mode 2: inner = k, outer stride = B*k) consumes."""
    return (world, B, k)


def pack_records(ids: np.ndarray, dist: np.ndarray) -> np.ndarray:
    """(ids [B,k] u64, dist [B,k] f32) -> [B,k] TopkRecord, the 16-byte wire format of the all-gather."""
    rec = np.zeros(ids.shape, _native.TOPK_RECORD)
    rec["id"] = ids
    rec["dist"] = dist
    return rec


def merge_records(gathered: np.ndarray, k: int):
    """Host restatement of the merge kernel: gathered [world][B][k] records -> global top-k per query by
    (_distance, _rowid); unused slots carry id UINT64_MAX.  Like the kernel it drops NaN distances and reports -0 as
    +0 (the two tie).  Used by the CPU (gloo) test of the exchange."""
    world, B, kk = gathered.shape
    ids = np.full((B, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((B, k), np.inf, np.float32)
    cnt = np.zeros(B, np.uint32)
    for b in range(B):
        c = gathered[:, b, :].reshape(-1)
        c = c[(c["id"] != np.iinfo(np.uint64).max) & ~np.isnan(c["dist"])]
        order = np.lexsort((c["id"], c["dist"]))[:k]
        n = len(order)
        ids[b, :n] = c["id"][order]; dist[b, :n] = c["dist"][order] + np.float32(0); cnt[b] = n     # -0 + 0 = +0
    return ids, dist, cnt


def exchange_unique_id(group=None) -> bytes:
    """rank 0 creates the NCCL unique id through the C ABI; torch.distributed carries the 128 bytes."""
    import torch.distributed as dist
    box = [_native.comm_unique_id() if dist.get_rank(group) == 0 else None]
    dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return box[0]


def check_k(k: int) -> None:
    """The sharded search serves k (limit + offset) up to SHARDED_K_MAX = 2048: its merge of world x k records per
    query stays on the shared-memory selects.  Refused here, before any device work."""
    if k > _native.SHARDED_K_MAX:
        raise ValueError(f"limit + offset = {k} is above {_native.SHARDED_K_MAX}, the largest k the sharded search "
                         "serves")


class ShardedIvfPq:
    def __init__(self, data: IvfPqIndexData, *, group=None, device: Optional[int] = None, presharded: bool = False):
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised (one process per GPU)")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device = torch.cuda.current_device() if device is None else device
        self.dim = data.dim
        shard = data if presharded else data.shard(self.rank, self.world)
        self.local = _native.GpuIvfPq(shard, device=self.device, with_vectors=False)
        self.comm = _native.Comm(exchange_unique_id(group), self.rank, self.world, self.device)

    def close(self):
        self.comm.close()
        self.local.close()

    def search_device(self, d_q, k: int = 10, nprobes: int = 20, lower=None, upper=None):
        """d_q: [B, dim] float32 CUDA tensor (identical on every rank).  Returns CUDA tensors
        (ids int64 holding the u64 row ids, dist float32, count int32), identical on every rank."""
        check_k(k)
        import torch
        B = d_q.shape[0]
        dev = d_q.device
        stream = torch.cuda.current_stream().cuda_stream
        ids = torch.empty(B, k, dtype=torch.int64, device=dev)
        dst = torch.empty(B, k, dtype=torch.float32, device=dev)
        cnt = torch.empty(B, dtype=torch.int32, device=dev)
        p = _native.make_params(k=k, nprobes=nprobes, lower=lower, upper=upper)
        self.comm.search_device(self.local, d_q.data_ptr(), B, p, ids.data_ptr(), dst.data_ptr(), cnt.data_ptr(), stream)
        return ids, dst, cnt

    def search(self, queries, k: int = 10, nprobes: int = 20, lower=None, upper=None):
        """Host-buffer collective search through lgpu_search_sharded."""
        check_k(k)
        return self.comm.search(self.local, queries, k=k, nprobes=nprobes, lower=lower, upper=upper)

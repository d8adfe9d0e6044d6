#!/usr/bin/env python
"""Rows added after an index was built: the union search (lgpu_search_unindexed_device: the IVF step and the tail's
exact scan on forked streams, merged by one select) against the index alone (fast_search), one JSON line per tail size.

Index: C2-shaped IVF_PQ (1M x 768, nlist 1024, m 96, l2; nprobes 20, k 10, B 1024), synthetic like bench_large_k.py's
(random centroids, codebook and codes: time and exactness do not depend on index quality).  Tails of 10k, 100k and 1M
random rows.

Per line: device name and power limit (read in the same run); step ms of the union and of the index alone (CUDA events
around the device entry point, median of --steps after --warmup); the tail's exact scan alone (the same device entry of
a flat handle over the tail, timed the same way) and its share of the union step; append rows/s (the tail grown by
GpuFlat.append in 10k-row chunks from 10k rows, host clock around calls that synchronise); optimize seconds (what
Table.optimize does: IvfPqIndexData.extend of the index by the tail, then the index handle opened again); and a
bit-exact check of 16 queries against the union oracle (tests/unindexed_oracle.py)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from bench_binary import device_info  # noqa: E402
from bench_large_k import exact, host, outputs, pq_index, time_steps  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from tests import unindexed_oracle as U  # noqa: E402

B, K, NP = 1024, 10, 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tails", default="10000,100000,1000000")
    a = ap.parse_args()
    ix = pq_index(False)
    n0 = ix.nrows
    gpu = _native.GpuIvfPq(ix, with_vectors=False)
    q = torch.randn(B, ix.dim, generator=torch.Generator().manual_seed(3))
    dq = q.cuda()
    st = torch.cuda.current_stream().cuda_stream
    p = _native.make_params(k=K, nprobes=NP)
    o = outputs(B, K)
    dev, power = device_info()

    def index_only():
        gpu.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    t_index = time_steps(index_only, a.steps, a.warmup)
    for n in (int(s) for s in a.tails.split(",")):
        x = torch.randn(n, ix.dim, generator=torch.Generator(device="cuda").manual_seed(n), device="cuda").cpu().numpy()
        ids = np.arange(n0, n0 + n, dtype=np.uint64)
        chunk = min(10000, n)
        tail = _native.GpuFlat(x[:chunk], row_ids=ids[:chunk])
        t0 = time.perf_counter()
        for s in range(chunk, n, chunk):
            tail.append(x[s:s + chunk], ids[s:s + chunk])
        append_s = time.perf_counter() - t0
        append_rate = (n - chunk) / append_s if n > chunk else None

        def union():
            gpu.search_unindexed_device(tail, dq.data_ptr(), B, p, 0, 0, o[0].data_ptr(), o[1].data_ptr(),
                                        o[2].data_ptr(), st)

        def tail_only():
            tail.search_device("l2", dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
        t_tail = time_steps(tail_only, a.steps, a.warmup)
        t_union = time_steps(union, a.steps, a.warmup)
        union()
        torch.cuda.synchronize()
        ok = exact(host(o, 16), U.union_search(ix, x, ids, q[:16].numpy(), K, NP))
        t0 = time.perf_counter()
        ext = ix.extend(x, ids)
        reopened = _native.GpuIvfPq(ext, with_vectors=False)
        optimize_s = time.perf_counter() - t0
        reopened.close()
        tail.close()
        del ext
        print(json.dumps(dict(workload=f"tail_{n}", device=dev, power_limit=power, index_rows=n0, tail_rows=n, B=B,
                              k=K, nprobes=NP, step_ms_union=round(t_union, 4), step_ms_fast_search=round(t_index, 4),
                              tail_scan_ms=round(t_tail, 4), tail_scan_share=round(t_tail / t_union, 4),
                              append_rows_per_s=float(f"{append_rate:.4g}") if append_rate else None,
                              optimize_s=round(optimize_s, 3), oracle_ok=ok)), flush=True)
    gpu.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""IVF_HNSW_SQ (per-partition HNSW graphs over 8-bit scalar codes) against the IVF_SQ scan on the SAME partitions and
codes, so the comparison isolates the graph: one JSON line per (nlist, nprobes, batch, ef).

Data: 1M x 768 clustered rows, l2, generated as scripts/bench_ivf_sq.py does (row = centre of its partition + 0.5 N(0,1)
noise, stored in the partition it was drawn around; quantiser range from a sample).  The graphs are built on the GPU by
lancedb_b200.index.build_hnsw_graph (m 20, ef_construction 300, the reference's defaults) and the build time is
reported per nlist.  nlist 16, 64 and 1024 -- HNSW variants are built with few, large partitions, IVF_SQ with many.

Per line: device name and power limit (read in the same run), ms per step and QPS of the device entry point (CUDA events,
median over the timed steps), recall@10 against exact f32 flat search (256 queries) for both kinds; per (nlist, nprobes)
the CPU oracle's QPS (all threads) and a bit-exact check of 16 queries against it."""
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

from bench_ivf_sq import device_info, exact_topk, make_index  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import IvfHnswSqIndexData, build_hnsw_graph  # noqa: E402
from tests import hnsw_sq_oracle  # noqa: E402

NPROBES = {16: (1, 4, 16), 64: (4, 16, 64), 1024: (20, 100, 1024)}
RECALL_QUERIES = 256


def timed(gpu, q, B, p, steps, warmup):
    k = p.k
    ids = torch.empty(B, k, dtype=torch.int64, device="cuda"); dist = torch.empty(B, k, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def step():
        gpu.search_device(q.data_ptr(), B, p, ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(), st)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for s, e in ev:
        s.record(); step(); e.record()
    torch.cuda.synchronize()
    return float(np.median([s.elapsed_time(e) for s, e in ev])), ids.cpu().numpy().view(np.uint64)


def recall(truth, got, k):
    return float(np.mean([len(set(t.tolist()) & set(g.tolist())) / k for t, g in zip(truth, got)]))


def run(nlist, n, k, m, ef_construction, batches, efs, steps, warmup, check, gpu_name, power):
    cfg = dict(n=n, dim=768, nlist=nlist, metric="l2")
    sq, x, queries = make_index(cfg)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    graph = build_hnsw_graph(sq.codes, sq.part_offsets, m, ef_construction, device="cuda")
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    data = IvfHnswSqIndexData(sq, m, *graph)
    g, s = _native.GpuIvfHnswSq(data, with_vectors=False), _native.GpuIvfSq(sq, with_vectors=False)
    print(json.dumps({"nlist": nlist, "device": gpu_name, "power_limit": power, "rows": n, "dim": 768, "m": m,
                      "ef_construction": ef_construction, "graph_build_s": build_s,
                      "upper_blocks": int(data.upper_adj.shape[0])}), flush=True)
    qall = queries(max(batches), 7)
    truth = exact_topk(x, qall[:RECALL_QUERIES], k, "l2")
    for nprobes in NPROBES[nlist]:
        for B in batches:
            q = qall[:B].contiguous()
            nr = min(B, RECALL_QUERIES)
            ms_s, ids_s = timed(s, q, B, _native.make_params(k, nprobes), steps, warmup)
            base = {"nlist": nlist, "nprobes": nprobes, "batch": B, "k": k, "device": gpu_name, "power_limit": power,
                    "ivf_sq_ms": ms_s, "ivf_sq_qps": B / (ms_s / 1e3), "ivf_sq_recall": recall(truth[:nr], ids_s[:nr], k)}
            for ef in efs:
                ms_h, ids_h = timed(g, q, B, _native.make_params(k, nprobes, ef=ef), steps, warmup)
                print(json.dumps(dict(base, ef=ef, hnsw_ms=ms_h, hnsw_qps=B / (ms_h / 1e3),
                                      hnsw_recall=recall(truth[:nr], ids_h[:nr], k),
                                      hnsw_over_sq=(B / (ms_h / 1e3)) / (B / (ms_s / 1e3)))), flush=True)
        qh = qall[:check].cpu().numpy()
        gi, gd, gc = g.search(qh, k=k, nprobes=nprobes, ef=64)
        t0 = time.perf_counter()
        oi, od, oc = hnsw_sq_oracle.search(data, qh, k=k, nprobes=nprobes, ef=64, nthreads=os.cpu_count())
        cpu_qps = check / (time.perf_counter() - t0)
        print(json.dumps({"nlist": nlist, "nprobes": nprobes, "ef": 64, "oracle_qps_cpu_all_threads": cpu_qps,
                          "cpu_threads": os.cpu_count(),
                          "oracle_check": bool(np.array_equal(gi, oi) and np.array_equal(gc, oc) and
                                               np.array_equal(gd.view(np.uint32), od.view(np.uint32)))}), flush=True)
    g.close(); s.close()
    del x
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nlist", default="16,64,1024")
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--m", type=int, default=20)
    ap.add_argument("--ef-construction", type=int, default=300)
    ap.add_argument("--batches", default="1,64,1024")
    ap.add_argument("--efs", default="16,64,512")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=16, help="queries verified against the CPU oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_hnsw_sq.py measures the GPU path and needs a CUDA device")
    gpu_name, power = device_info()
    for nl in a.nlist.split(","):
        run(int(nl), a.n, a.k, a.m, a.ef_construction, [int(b) for b in a.batches.split(",")],
            [int(e) for e in a.efs.split(",")], a.steps, a.warmup, a.check, gpu_name, power)


if __name__ == "__main__":
    main()

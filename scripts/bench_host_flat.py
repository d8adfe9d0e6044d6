#!/usr/bin/env python
"""Flat search from rows kept in pinned host memory (LGPU_FLAT_HBM_BYTES=0) against rows in HBM, in one run.

Column: the C4 shape, 1M x 1536 (6.1 GB of f32 rows), random normal rows, opened with both placements as f32 and again
as float16.  Queries: B 1, 64 and 1024, k 10, under l2, cosine and dot.

Prints one JSON line each for
  device        the card's name and power limit, read in this run
  memcpy        pinned host -> device cudaMemcpy bandwidth (1 GiB, CUDA events), the PCIe yardstick
  open          open time of the two placements (host clock), host and device bytes of each
  case          per row type, metric and B: ms per call of each placement (CUDA events around lgpu_flat_search_device,
                median of --steps, the two handles alternated call by call), the streamed rate (row bytes over the host
                call's time) and its share of the memcpy rate, the copy time of the rows at the memcpy rate, and
                whether both placements returned the same ids, counts and distance bits on the timed calls.  A host
                call overlaps the copy of each chunk with the scoring of the one before, so its time is about the
                larger of the copy time and the HBM call's time (the scoring of the same rows) plus one chunk
  oversized     a column larger than free HBM: not measured by this script
"""
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
from bench_host_vectors import emit, memcpy_gbs  # noqa: E402
from lancedb_b200 import _native  # noqa: E402

N, DIM, K = 1_000_000, 1536, 10


def open_both(x):
    os.environ.pop("LGPU_FLAT_HBM_BYTES", None)
    t0 = time.time()
    hbm = _native.GpuFlat(x)
    t_hbm = time.time() - t0
    os.environ["LGPU_FLAT_HBM_BYTES"] = "0"
    t0 = time.time()
    host = _native.GpuFlat(x)
    t_host = time.time() - t0
    del os.environ["LGPU_FLAT_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host
    emit(line="open", rows=str(x.dtype), hbm_s=round(t_hbm, 3), host_s=round(t_host, 3), host_bytes=host.host_bytes(),
         device_bytes_hbm=hbm.device_bytes, device_bytes_host=host.device_bytes)
    return hbm, host


def run(hbm, host, rows, bw, a):
    st = torch.cuda.current_stream().cuda_stream
    row_bytes = N * DIM * (2 if rows == "float16" else 4)
    for metric in ("l2", "cosine", "dot"):
        for B in (1, 64, 1024):
            dq = torch.randn(B, DIM, generator=torch.Generator().manual_seed(B)).cuda()
            p = _native.make_params(k=K, nprobes=0, refine_factor=0)
            outs = {name: (h, torch.empty(B, K, dtype=torch.int64, device="cuda"), torch.empty(B, K, device="cuda"),
                           torch.empty(B, dtype=torch.int32, device="cuda")) for name, h in (("hbm", hbm), ("host", host))}
            ms = {"hbm": [], "host": []}
            same = True
            for i in range(a.warmup + a.steps):
                for name, (h, oi, od, oc) in outs.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    h.search_device(metric, dq.data_ptr(), B, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
                    e.record()
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        ms[name].append(s.elapsed_time(e))
                if i >= a.warmup:
                    same &= all(torch.equal(outs["hbm"][j], outs["host"][j]) for j in (1, 3)) and \
                        torch.equal(outs["hbm"][2].view(torch.int32), outs["host"][2].view(torch.int32))
            t_hbm, t_host = float(np.median(ms["hbm"])), float(np.median(ms["host"]))
            rate = row_bytes / (t_host / 1e3) / 1e9
            emit(line="case", rows=rows, metric=metric, B=B, k=K, ms_hbm=round(t_hbm, 3), ms_host=round(t_host, 3),
                 streamed_GBps=round(rate, 2), share_of_memcpy=round(rate / bw, 3),
                 copy_ms_at_memcpy_rate=round(row_bytes / bw / 1e6, 3), same_results=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    bw = memcpy_gbs()
    emit(line="memcpy", h2d_pinned_GBps=round(bw, 2))
    x = torch.randn(N, DIM, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    x32 = x.cpu().numpy()
    hbm, host = open_both(x32)
    run(hbm, host, "float32", bw, a)
    hbm.close(); host.close()
    x16 = x.half().cpu().numpy()
    del x, x32
    hbm, host = open_both(x16)
    run(hbm, host, "float16", bw, a)
    hbm.close(); host.close()
    emit(line="oversized", status="not measured")


if __name__ == "__main__":
    main()

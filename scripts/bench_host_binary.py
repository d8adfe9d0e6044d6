#!/usr/bin/env python
"""Binary (Hamming) search from packed rows kept in pinned host memory (LGPU_BINARY_HBM_BYTES=0) against rows in HBM,
in one run.

Shapes: W1 of bench_binary.py, 10M x 1024 bits (1.28 GB of packed rows), at B 1 and 1024; and 1M x 256 bits at B 1024.
k 10, random rows and queries.  Every shape takes the list route (N above the 65536-row threshold sample): one sample
pass in HBM, then one filtering b1 GEMM per streamed chunk of a host handle.

Prints one JSON line each for
  device        the card's name and power limit, read in this run
  memcpy        pinned host -> device cudaMemcpy bandwidth (1 GiB, CUDA events), the PCIe yardstick
  open          per shape: open time of the two placements (host clock), host and device bytes of each
  case          per shape and B: ms per call of each placement (CUDA events around lgpu_binary_search_device, median of
                --steps, the two handles alternated call by call), the PCIe bytes of a host call (its packed rows, each
                crossing once; the fix-up streams nothing when no list overflowed, which `flagged` reports), their rate
                over the host call's time and its share of the memcpy rate, and whether both placements returned the
                same ids, counts and distance bits on the timed calls
"""
import argparse
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

K = 10
SHAPES = [("W1", 10_000_000, 128, (1, 1024)), ("1Mx256", 1_000_000, 32, (1024,))]


def open_both(name, x):
    os.environ.pop("LGPU_BINARY_HBM_BYTES", None)
    t0 = time.time()
    hbm = _native.GpuBinary(x)
    t_hbm = time.time() - t0
    os.environ["LGPU_BINARY_HBM_BYTES"] = "0"
    t0 = time.time()
    host = _native.GpuBinary(x)
    t_host = time.time() - t0
    del os.environ["LGPU_BINARY_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host
    emit(line="open", shape=name, hbm_s=round(t_hbm, 3), host_s=round(t_host, 3), host_bytes=host.host_bytes(),
         device_bytes_hbm=hbm.device_bytes, device_bytes_host=host.device_bytes)
    return hbm, host


def flagged(h, dq, B):
    _native.set_profiling(True)
    try:
        q = dq.cpu().numpy()
        h.search(q, k=K)
        return _native.last_filter_stats()["flagged_queries"]
    finally:
        _native.set_profiling(False)


def run(name, n, nb, bs, hbm, host, bw, a):
    st = torch.cuda.current_stream().cuda_stream
    row_bytes = n * ((nb + 31) // 32 * 32)
    for B in bs:
        dq = torch.randint(0, 256, (B, nb), dtype=torch.uint8, generator=torch.Generator().manual_seed(B)).cuda()
        p = _native.make_params(k=K, nprobes=0, refine_factor=0)
        outs = {nm: (h, torch.empty(B, K, dtype=torch.int64, device="cuda"), torch.empty(B, K, device="cuda"),
                     torch.empty(B, dtype=torch.int32, device="cuda")) for nm, h in (("hbm", hbm), ("host", host))}
        ms = {"hbm": [], "host": []}
        same = True
        for i in range(a.warmup + a.steps):
            for nm, (h, oi, od, oc) in outs.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                h.search_device(dq.data_ptr(), B, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
                e.record()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    ms[nm].append(s.elapsed_time(e))
            if i >= a.warmup:
                same &= all(torch.equal(outs["hbm"][j], outs["host"][j]) for j in (1, 3)) and \
                    torch.equal(outs["hbm"][2].view(torch.int32), outs["host"][2].view(torch.int32))
        t_hbm, t_host = float(np.median(ms["hbm"])), float(np.median(ms["host"]))
        rate = row_bytes / (t_host / 1e3) / 1e9
        emit(line="case", shape=name, rows=n, bits=nb * 8, B=B, k=K, ms_hbm=round(t_hbm, 3), ms_host=round(t_host, 3),
             ms_hbm_spread=[round(min(ms["hbm"]), 3), round(max(ms["hbm"]), 3)],
             ms_host_spread=[round(min(ms["host"]), 3), round(max(ms["host"]), 3)],
             pcie_bytes_per_call=row_bytes, streamed_GBps=round(rate, 2), share_of_memcpy=round(rate / bw, 3),
             flagged=flagged(host, dq, B), same_results=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    bw = memcpy_gbs()
    emit(line="memcpy", h2d_pinned_GBps=round(bw, 2))
    for name, n, nb, bs in SHAPES:
        x = torch.randint(0, 256, (n, nb), dtype=torch.uint8, generator=torch.Generator().manual_seed(n)).numpy()
        hbm, host = open_both(name, x)
        del x
        run(name, n, nb, bs, hbm, host, bw, a)
        hbm.close(); host.close()


if __name__ == "__main__":
    main()

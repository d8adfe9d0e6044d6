#!/usr/bin/env python
"""Refine from raw vectors kept in pinned host memory (LGPU_VECTORS_HBM_BYTES=0) against refine from HBM, in one run.

Index: C2-shaped IVF_PQ (1M x 768, nlist 1024, m 96, l2), synthetic as scripts/bench_config.py builds it (time and
exactness do not depend on index quality), with raw vectors.  Queries: B 1024, nprobes 20, k 10.

Prints one JSON line each for
  device        the card's name and power limit, read in this run
  memcpy        pinned host -> device cudaMemcpy bandwidth (1 GiB, CUDA events), the PCIe yardstick
  open          open time of the two placements (host clock around lgpu_index_open)
  rf<R>         for refine_factor 1, 10 and 50: step ms of each placement (CUDA events around lgpu_search_device,
                median of --steps, the two handles alternated step by step), refine-stage ms of each (the library's
                stage marks, lgpu_last_stage_ms, mean of --steps profiled host calls), the bytes refine reads from
                host memory (k x rf rows of round_up(768, 4) floats per query), their rate over the host refine
                stage and its share of the memcpy rate, and whether both placements returned the same ids and
                distance bits
  oversized     an index whose raw vectors exceed free HBM: not measured by this script
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
from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import IvfPqIndexData  # noqa: E402

B, NPROBES, K = 1024, 20, 10


def c2_index():
    rng = np.random.default_rng(7)
    n, dim, nlist, m = 1_000_000, 768, 1024, 96
    base = n // nlist
    sizes = rng.integers(int(base * 0.7), int(base * 1.3) + 1, nlist).astype(np.int64)
    n = int(sizes.sum())
    cent = rng.standard_normal((nlist, dim), dtype=np.float32)
    cb = (rng.standard_normal((m, 256, dim // m), dtype=np.float32) * 0.3).astype(np.float32)
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    codes = rng.integers(0, 256, size=n * m, dtype=np.uint8)
    vec = torch.randn(n, dim, generator=torch.Generator(device="cuda").manual_seed(9), device="cuda").cpu().numpy()
    return IvfPqIndexData(dim, nlist, m, "l2", cent, cb, off, codes, np.arange(n, dtype=np.uint64), vec)


def memcpy_gbs(reps=10):
    src = torch.empty(1 << 28, dtype=torch.float32).pin_memory()        # 1 GiB
    dst = torch.empty(1 << 28, dtype=torch.float32, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    e.record()
    torch.cuda.synchronize()
    return reps * src.numel() * 4 / (s.elapsed_time(e) / 1e3) / 1e9


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    bw = memcpy_gbs()
    emit(line="memcpy", h2d_pinned_GBps=round(bw, 2))
    ix = c2_index()
    os.environ.pop("LGPU_VECTORS_HBM_BYTES", None)
    t0 = time.time()
    hbm = _native.GpuIvfPq(ix)
    t_hbm = time.time() - t0
    os.environ["LGPU_VECTORS_HBM_BYTES"] = "0"
    t0 = time.time()
    host = _native.GpuIvfPq(ix)
    t_host = time.time() - t0
    del os.environ["LGPU_VECTORS_HBM_BYTES"]
    assert not hbm.vectors_on_host and host.vectors_on_host
    emit(line="open", hbm_s=round(t_hbm, 3), host_s=round(t_host, 3), host_bytes=host.host_bytes(),
         device_bytes_hbm=hbm.device_bytes(), device_bytes_host=host.device_bytes())
    q = torch.randn(B, ix.dim, generator=torch.Generator().manual_seed(3))
    qn = q.numpy()
    dq = q.cuda()
    st = torch.cuda.current_stream().cuda_stream
    stride = (ix.dim + 3) // 4 * 4
    for rf in (1, 10, 50):
        p = _native.make_params(k=K, nprobes=NPROBES, refine_factor=rf)
        outs = {}
        for name, h in (("hbm", hbm), ("host", host)):
            oi = torch.empty(B, K, dtype=torch.int64, device="cuda")
            od = torch.empty(B, K, device="cuda")
            oc = torch.empty(B, dtype=torch.int32, device="cuda")
            outs[name] = (h, oi, od, oc)
        ms = {"hbm": [], "host": []}
        for i in range(a.warmup + a.steps):
            for name, (h, oi, od, oc) in outs.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                h.search_device(dq.data_ptr(), B, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
                e.record()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    ms[name].append(s.elapsed_time(e))
        same = all(torch.equal(outs["hbm"][j], outs["host"][j]) for j in (1, 3)) and \
            torch.equal(outs["hbm"][2].view(torch.int32), outs["host"][2].view(torch.int32))
        refine = {}
        for name, h in (("hbm", hbm), ("host", host)):
            _native.set_profiling(True)
            r = []
            for _ in range(a.steps):
                h.search(qn, k=K, nprobes=NPROBES, refine_factor=rf)
                r.append(_native.last_stage_ms()["refine"])
            _native.set_profiling(False)
            refine[name] = float(np.mean(r))
        read = B * K * rf * stride * 4
        rate = read / (refine["host"] / 1e3) / 1e9
        emit(line=f"rf{rf}", refine_factor=rf, step_ms_hbm=round(float(np.median(ms["hbm"])), 4),
             step_ms_host=round(float(np.median(ms["host"])), 4), refine_ms_hbm=round(refine["hbm"], 4),
             refine_ms_host=round(refine["host"], 4), host_bytes_read=read, host_read_GBps=round(rate, 2),
             share_of_memcpy=round(rate / bw, 3), same_results=bool(same))
    emit(line="oversized", status="not measured")
    hbm.close()
    host.close()


if __name__ == "__main__":
    main()

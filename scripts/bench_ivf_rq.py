#!/usr/bin/env python
"""IVF_RQ (1-bit RaBitQ partitions, binary tensor-core scan): search throughput on the GPU, one JSON line per workload.

Workloads: R2 = 1M x 768, nlist 1024, nprobes 20, k 10, batch 1024, l2; R2r = R2 with refine_factor 10; R3 = 4M x 768,
nlist 4096, nprobes 50, k 100, batch 4096, cosine; R1 = R2 at batch 1.  The rows are clustered (row = centre of its
partition + 0.5 N(0, 1) noise, centres N(0, 1)) and stored in the partition they were drawn around, so no k-means runs
here; the rotation and the codes come from the trainer's own functions (rq_rotation, rq_encode).

Per line: device name and power limit (read in the same run), ms per step and QPS (CUDA events around the device entry
point, median over the timed steps), the per-kernel device ms of one profiled step (torch.profiler), the scan kernel's
time against the compulsory HBM bytes (the codes and the 12 bytes of factors of every probed partition read once) at
3.35 TB/s (H100 SXM data sheet), recall@k against exact f32 flat search (256 queries) without and with refine_factor 10,
the CPU oracle's QPS on all threads and a bit-exact check of the first 16 queries against it."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import IvfRqIndexData, rq_encode, rq_rotation  # noqa: E402
from tests import rq_oracle  # noqa: E402

WORKLOADS = {
    "R2": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1024, metric="l2", refine=0),
    "R2r": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1024, metric="l2", refine=10),
    "R3": dict(n=4_000_000, dim=768, nlist=4096, nprobes=50, k=100, batch=4096, metric="cosine", refine=0),
    "R1": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1, metric="l2", refine=0),
}
HBM_BYTES_PER_S = 3.35e12
RECALL_QUERIES = 256
RECALL_REFINE = 10


def device_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, power


def kernels_of(fn):
    """{kernel: device ms} of one profiled call (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0.0)
        if us <= 0 or "Memcpy" in e.key or "Memset" in e.key:
            continue
        m = re.search(r"(\w+_kernel)", e.key)
        name = m.group(1) if m else e.key
        out[name] = round(out.get(name, 0.0) + us / 1e3, 4)
    return out


def make_index(cfg, seed=1):
    """(IvfRqIndexData with the raw vectors, rows on the GPU (normalised for cosine), query generator)."""
    n, dim, nlist = cfg["n"], cfg["dim"], cfg["nlist"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    cent = torch.randn(nlist, dim, generator=g, device="cuda")
    part = torch.randint(0, nlist, (n,), generator=g, device="cuda").sort().values
    x = torch.empty(n, dim, device="cuda")
    for s in range(0, n, 1 << 18):
        e = min(n, s + (1 << 18))
        x[s:e] = cent[part[s:e]] + 0.5 * torch.randn(e - s, dim, generator=g, device="cuda")
    raw = x.cpu().numpy()
    if cfg["metric"] == "cosine":
        x /= x.norm(dim=1, keepdim=True)
        cent /= cent.norm(dim=1, keepdim=True)
    P = rq_rotation(dim)
    codes, add, scale = rq_encode(x, cent.cpu().numpy(), part, P)
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(torch.bincount(part, minlength=nlist).cpu().numpy())
    data = IvfRqIndexData(dim=dim, nlist=nlist, metric=cfg["metric"], centroids=cent.cpu().numpy(), rotation=P,
                          part_offsets=off, codes=codes, add_factors=add, scale_factors=scale,
                          row_ids=np.arange(n, dtype=np.uint64), vectors=raw)

    def queries(B, qseed):
        gq = torch.Generator(device="cuda").manual_seed(qseed)
        c = torch.randint(0, nlist, (B,), generator=gq, device="cuda")
        return (cent[c] + 0.5 * torch.randn(B, dim, generator=gq, device="cuda")).contiguous()
    return data, x, queries


def exact_topk(x, q, k, metric):
    """ids [B, k] of exact f32 flat search on the GPU (l2, or cosine on normalised rows)."""
    if metric == "cosine":
        q = q / q.norm(dim=1, keepdim=True)
    best_d = best_i = None
    for s in range(0, x.shape[0], 1 << 20):
        xs = x[s:s + (1 << 20)]
        d = (xs * xs).sum(1)[None, :] - 2.0 * (q @ xs.T)
        dv, di = d.topk(k, dim=1, largest=False)
        di = di + s
        if best_d is None:
            best_d, best_i = dv, di
        else:
            cd, ci = torch.cat([best_d, dv], 1), torch.cat([best_i, di], 1)
            best_d, j = cd.topk(k, dim=1, largest=False)
            best_i = ci.gather(1, j)
    return best_i.cpu().numpy()


def run(name, cfg, steps, warmup, check, gpu_name, power):
    B, k, nprobes = cfg["batch"], cfg["k"], cfg["nprobes"]
    data, x, queries = make_index(cfg)
    gpu = _native.GpuIvfRq(data)
    qs = [queries(B, 100 + i) for i in range(4)]
    ids = torch.empty(B, k, dtype=torch.int64, device="cuda"); dist = torch.empty(B, k, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    p = _native.make_params(k=k, nprobes=nprobes, refine_factor=cfg["refine"])
    st = torch.cuda.current_stream().cuda_stream

    def step(i):
        gpu.search_device(qs[i % 4].data_ptr(), B, p, ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(), st)

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for i in range(steps):
        ev[i][0].record()
        step(i)
        ev[i][1].record()
    torch.cuda.synchronize()
    ms = float(np.median([s.elapsed_time(e) for s, e in ev]))
    last = (steps - 1) % 4
    gi, gd, gc = ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
    _native.set_profiling(True)
    step(last)
    torch.cuda.synchronize()
    row_bytes = (cfg["dim"] + 255) // 256 * 32                 # codes padded to 256 bits
    scanned_rows = _native.last_scanned_code_bytes() // row_bytes
    _native.set_profiling(False)
    path = kernels_of(lambda: step(last))
    qh = qs[last].cpu().numpy()
    parts, _ = gpu.debug_coarse(qh, nprobes)
    sizes = np.diff(data.part_offsets.astype(np.int64))
    compulsory = int(sizes[np.unique(parts[parts < cfg["nlist"]])].sum()) * (row_bytes + 12)
    scan_ms = path.get("rq_scan_kernel", float("nan"))
    out = {"workload": name, "device": gpu_name, "power_limit": power,
           "config": f"{cfg['n']} x {cfg['dim']}, nlist {cfg['nlist']}, nprobes {nprobes}, k {k}, batch {B}, "
                     f"{cfg['metric']}, refine_factor {cfg['refine']}",
           "ms_per_step": ms, "qps": B / (ms / 1e3), "kernel_ms": path,
           "scan_ms": scan_ms, "compulsory_code_bytes": compulsory,
           "scan_hbm_lower_bound_ms": compulsory / HBM_BYTES_PER_S * 1e3,
           "scan_share_of_hbm_bound": (compulsory / HBM_BYTES_PER_S * 1e3) / scan_ms,
           "scanned_pairs_code_bytes": scanned_rows * row_bytes}
    nr = min(RECALL_QUERIES, B)
    truth = exact_topk(x, qs[last][:nr], k, cfg["metric"])
    recall = lambda ri, rc: float(np.mean([len(set(truth[b].tolist()) & set(ri[b, :rc[b]].tolist())) / k
                                           for b in range(nr)]))
    for key, rf in (("recall_at_k", 0), ("recall_at_k_refine10", RECALL_REFINE)):
        ri, _, rc = gpu.search(qh[:nr], k=k, nprobes=nprobes, refine_factor=rf)
        out[key] = recall(ri, rc)
    c = min(check, B)
    t0 = time.perf_counter()
    oi, od, oc = rq_oracle.search(data, qh[:c], k=k, nprobes=nprobes, refine_factor=cfg["refine"],
                                  nthreads=os.cpu_count())
    out["oracle_qps_cpu_all_threads"] = c / (time.perf_counter() - t0)
    out["oracle_check"] = bool(np.array_equal(gi[:c], oi) and np.array_equal(gc[:c], oc) and
                               np.array_equal(np.ascontiguousarray(gd[:c]).view(np.uint32), od.view(np.uint32)))
    gpu.close()
    del x
    torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="R2,R2r,R3,R1")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="queries verified against the CPU oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_rq.py measures the GPU path and needs a CUDA device")
    gpu_name, power = device_info()
    for w in a.workloads.split(","):
        run(w, WORKLOADS[w], a.steps, a.warmup, a.check, gpu_name, power)


if __name__ == "__main__":
    main()

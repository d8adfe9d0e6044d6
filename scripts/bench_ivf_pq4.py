#!/usr/bin/env python
"""4-bit IVF_PQ (packed nibble codes, pair-table scan over quantised per-probe tables): search throughput on the GPU,
one JSON line per workload, each 4-bit line followed by the 8-bit IVF_PQ at m 96 on the same rows (the comparison a user
makes when choosing num_bits).

Workloads: Q2 = 1M x 768, nlist 1024, nprobes 20, k 10, batch 1024, l2, 4-bit at m 48 (Q2) and at m 96 (Q2m96);
Q3 = 4M x 768, nlist 4096, nprobes 50, k 100, batch 4096, cosine, m 48; Q1 = Q2 at batch 1.  The rows are clustered
(row = centre of its partition + 0.5 N(0, 1) noise, centres N(0, 1)) and stored in the partition they were drawn around;
no k-means runs: each sub-space's codewords are that sub-vector of randomly sampled rows' residuals (training quality is
not what is measured), and every row is encoded by argmin (ties to the lowest code) on the GPU.

Per line: device name and power limit (read in the same run), ms per step and QPS (CUDA events around the device entry
point, median over the timed steps), the per-kernel device ms of one profiled step (torch.profiler, a separate run), the
scan kernel's time against the compulsory HBM bytes (the code bytes of every probed partition read once: m/2 per row
for 4 bits, m for 8) at 3.35 TB/s (H100 SXM data sheet), recall@k against exact f32 flat search (256 queries), the CPU
oracle's QPS on all threads and a bit-exact check of the first 16 queries against it."""
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

import oracle  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import IvfPqIndexData  # noqa: E402
from tests import pq4_oracle  # noqa: E402

WORKLOADS = {
    "Q2": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1024, metric="l2", m=48, pq8=True),
    "Q2m96": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1024, metric="l2", m=96, pq8=False),
    "Q3": dict(n=4_000_000, dim=768, nlist=4096, nprobes=50, k=100, batch=4096, metric="cosine", m=48, pq8=True),
    "Q1": dict(n=1_000_000, dim=768, nlist=1024, nprobes=20, k=10, batch=1, metric="l2", m=48, pq8=False),
}
PQ8_M = 96
HBM_BYTES_PER_S = 3.35e12
RECALL_QUERIES = 256


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


def make_rows(cfg, seed=1):
    """(rows on the GPU (normalised for cosine), centroids, partition of every row (sorted), query generator)."""
    n, dim, nlist = cfg["n"], cfg["dim"], cfg["nlist"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    cent = torch.randn(nlist, dim, generator=g, device="cuda")
    part = torch.randint(0, nlist, (n,), generator=g, device="cuda").sort().values
    x = torch.empty(n, dim, device="cuda")
    for s in range(0, n, 1 << 18):
        e = min(n, s + (1 << 18))
        x[s:e] = cent[part[s:e]] + 0.5 * torch.randn(e - s, dim, generator=g, device="cuda")
    if cfg["metric"] == "cosine":
        x /= x.norm(dim=1, keepdim=True)
        cent /= cent.norm(dim=1, keepdim=True)

    def queries(B, qseed):
        gq = torch.Generator(device="cuda").manual_seed(qseed)
        c = torch.randint(0, nlist, (B,), generator=gq, device="cuda")
        return (cent[c] + 0.5 * torch.randn(B, dim, generator=gq, device="cuda")).contiguous()
    return x, cent, part, queries


def make_index(cfg, x, cent, part, m, num_bits, seed=2):
    """IvfPqIndexData over the rows: sampled codewords, argmin codes (packed for 4 bits), partition-transposed."""
    n, dim, nlist = x.shape[0], cfg["dim"], cfg["nlist"]
    K, dsub = 1 << num_bits, dim // m
    g = torch.Generator(device="cuda").manual_seed(seed)
    pick = torch.randint(0, n, (m, K), generator=g, device="cuda")
    cb = torch.empty(m, K, dsub, device="cuda")
    for i in range(m):
        r = x[pick[i]] - cent[part[pick[i]]]
        cb[i] = r[:, i * dsub:(i + 1) * dsub]
    cbn = (cb * cb).sum(2)
    codes = np.empty((n, m), np.uint8)
    chunk = max(4096, (1 << 20) // K)                   # the [m, chunk, K] distance block stays near 4 GB or less
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        r = (x[s:e] - cent[part[s:e]]).reshape(e - s, m, dsub).transpose(0, 1)
        d = cbn[:, None, :] - 2.0 * torch.bmm(r, cb.transpose(1, 2))
        codes[s:e] = d.argmin(2).transpose(0, 1).to(torch.uint8).cpu().numpy()
    if num_bits == 4:
        codes = codes[:, 0::2] | (codes[:, 1::2] << 4)
    w = codes.shape[1]
    off = np.zeros(nlist + 1, np.uint64)
    off[1:] = np.cumsum(torch.bincount(part, minlength=nlist).cpu().numpy())
    codes_t = np.empty(n * w, np.uint8)
    for p in range(nlist):
        a, b = int(off[p]), int(off[p + 1])
        codes_t[a * w:b * w] = codes[a:b].T.reshape(-1)
    return IvfPqIndexData(dim=dim, nlist=nlist, m=m, metric=cfg["metric"], centroids=cent.cpu().numpy(),
                          codebook=cb.cpu().numpy(), part_offsets=off, codes_t=codes_t,
                          row_ids=np.arange(n, dtype=np.uint64), num_bits=num_bits)


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


def run(name, cfg, data, x, queries, steps, warmup, check, gpu_name, power):
    B, k, nprobes = cfg["batch"], cfg["k"], cfg["nprobes"]
    gpu = _native.GpuIvfPq(data, with_vectors=False)
    qs = [queries(B, 100 + i) for i in range(4)]
    ids = torch.empty(B, k, dtype=torch.int64, device="cuda"); dist = torch.empty(B, k, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    p = _native.make_params(k=k, nprobes=nprobes)
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
    path = kernels_of(lambda: step(last))
    qh = qs[last].cpu().numpy()
    parts, _ = gpu.debug_coarse(qh, nprobes)
    sizes = np.diff(data.part_offsets.astype(np.int64))
    compulsory = int(sizes[np.unique(parts[parts < cfg["nlist"]])].sum()) * data.code_bytes
    scan_ms = path.get("pq4_scan_kernel") if data.num_bits == 4 else sum(
        v for kname, v in path.items() if kname.startswith("scan"))
    out = {"workload": name, "device": gpu_name, "power_limit": power, "num_bits": data.num_bits, "m": data.m,
           "config": f"{cfg['n']} x {cfg['dim']}, nlist {cfg['nlist']}, nprobes {nprobes}, k {k}, batch {B}, "
                     f"{cfg['metric']}, {data.num_bits}-bit m {data.m}",
           "ms_per_step": ms, "qps": B / (ms / 1e3), "kernel_ms": path,
           "scan_ms": scan_ms, "compulsory_code_bytes": compulsory,
           "scan_hbm_lower_bound_ms": compulsory / HBM_BYTES_PER_S * 1e3,
           "scan_share_of_hbm_bound": (compulsory / HBM_BYTES_PER_S * 1e3) / scan_ms if scan_ms else None}
    nr = min(RECALL_QUERIES, B)
    truth = exact_topk(x, qs[last][:nr], k, cfg["metric"])
    out["recall_at_k"] = float(np.mean([len(set(truth[b].tolist()) & set(gi[b, :gc[b]].tolist())) / k
                                        for b in range(nr)]))
    c = min(check, B)
    t0 = time.perf_counter()
    if data.num_bits == 4:
        oi, od, oc = pq4_oracle.search(data, qh[:c], k=k, nprobes=nprobes, nthreads=os.cpu_count())
    else:
        oi, od, oc = oracle.OracleIndex.from_data(data).search(qh[:c], k=k, nprobes=nprobes, nthreads=os.cpu_count())
    out["oracle_qps_cpu_all_threads"] = c / (time.perf_counter() - t0)
    out["oracle_check"] = bool(np.array_equal(gi[:c], oi) and np.array_equal(gc[:c], oc) and
                               np.array_equal(np.ascontiguousarray(gd[:c]).view(np.uint32), od.view(np.uint32)))
    gpu.close()
    torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="Q2,Q2m96,Q3,Q1")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="queries verified against the CPU oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_pq4.py measures the GPU path and needs a CUDA device")
    gpu_name, power = device_info()
    for w in a.workloads.split(","):
        cfg = WORKLOADS[w]
        x, cent, part, queries = make_rows(cfg)
        run(w, cfg, make_index(cfg, x, cent, part, cfg["m"], 4), x, queries, a.steps, a.warmup, a.check, gpu_name,
            power)
        if cfg["pq8"]:
            run(w, cfg, make_index(cfg, x, cent, part, PQ8_M, 8), x, queries, a.steps, a.warmup, a.check, gpu_name,
                power)
        del x, cent, part
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

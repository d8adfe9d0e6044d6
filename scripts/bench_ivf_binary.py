#!/usr/bin/env python
"""Binary IVF_FLAT (Hamming partitions, b1 MMA scan): search throughput on the GPU against the flat binary path on the
same rows, one JSON line per workload.

Workloads: IB1 = 10M x 1024 bits, nlist 4096, nprobes 20, B 1024, k 10 (the flat path's W1 rows); IB2 = 1M x 256 bits,
nlist 1024, nprobes 20, B 1024; IB3 = IB1 at B 1; IB4 = IB1 under a 10 % prefilter (host-buffer filtered calls for both
paths, which include their copies).  Rows are bench_binary.py's `latent` data (sign bits of rank-32 latent Gaussian
vectors); queries are rows with 5 % of their bits flipped.  The index is trained by train_ivf_binary (k-modes on the
GPU, --iters rounds) and the training time is reported, not counted.

Per line: device name and power limit (read in the same run), ms per step and QPS (CUDA events around the device entry
point, median of the timed steps), the stage split of one profiled call (lgpu_last_stage_ms), the probed rows x nbytes
(a partition counted once per query that probes it) and their time at 3.35 TB/s (H100 SXM data sheet) against the scan
stage, recall@k against the flat binary path and the flat path's ms / QPS on the same queries, and a bit-exact check of
16 queries against the C oracle.  Recall counts a returned row as a hit when its distance is at or below the flat
path's k-th distance for that query (Hamming distances tie in runs, so which of the tied rows an exact top-k keeps is
decided by row id, and id overlap would under-count).  The batched workloads without a prefilter also sweep nprobes
(--sweep): ms and recall at each value."""
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

from bench_binary import device_info, packed  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import train_ivf_binary  # noqa: E402
from tests import ivf_binary_oracle  # noqa: E402

WORKLOADS = {
    "IB1": dict(n=10_000_000, bits=1024, nlist=4096, nprobes=20, batch=1024, k=10, filt=0.0),
    "IB2": dict(n=1_000_000, bits=256, nlist=1024, nprobes=20, batch=1024, k=10, filt=0.0),
    "IB3": dict(n=10_000_000, bits=1024, nlist=4096, nprobes=20, batch=1, k=10, filt=0.0),
    "IB4": dict(n=10_000_000, bits=1024, nlist=4096, nprobes=20, batch=1024, k=10, filt=0.1),
}
HBM_BYTES_PER_S = 3.35e12


def time_steps(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


_cache = {}


def index_for(cfg, iters):
    key = (cfg["n"], cfg["bits"], cfg["nlist"])
    if key not in _cache:
        x = packed(cfg["n"], cfg["bits"], "latent", 7)
        t0 = time.time()
        data = train_ivf_binary(x, num_partitions=cfg["nlist"], max_iterations=iters, device="cuda")
        _cache.clear()
        _cache[key] = (x, data, time.time() - t0)
    return _cache[key]


def recall_at_k(got, want, k):
    """hits: returned rows with distance <= the flat k-th distance of their query (all of them when the flat search
    found fewer than k rows), over min(k, rows the flat search found)"""
    gd, gc = got[1], got[2]
    wd, wc = want[1], want[2]
    kth = np.where(wc >= k, wd[:, k - 1], np.inf)
    hits = sum(min(k, int(np.sum(gd[b, :gc[b]] <= kth[b]))) for b in range(len(gc)))
    return hits / max(1, int(np.minimum(wc, k).sum()))


def run(name, cfg, steps, warmup, iters, sweep, gpu_name, power):
    x, data, train_s = index_for(cfg, iters)
    rng = np.random.default_rng(3)
    B, k, nb = cfg["batch"], cfg["k"], cfg["bits"] // 8
    flips = np.packbits(rng.random((B, cfg["bits"])) < 0.05, axis=1)
    q = np.ascontiguousarray(x[rng.integers(0, cfg["n"], B)] ^ flips)
    allow = bm = None
    if cfg["filt"]:
        allow = rng.random(cfg["n"]) < cfg["filt"]
        bm = _native.mask_bitmap(allow)
    ivf = _native.GpuIvfBinary(data)
    flat = _native.GpuBinary(x)
    p = _native.make_params(k, cfg["nprobes"], max_nprobes=cfg["nprobes"] if cfg["filt"] else 0)
    dq = torch.from_numpy(q).cuda()
    di = torch.empty((B, k), dtype=torch.int64, device="cuda")
    dd = torch.empty((B, k), dtype=torch.float32, device="cuda")
    dc = torch.empty(B, dtype=torch.int32, device="cuda")
    if cfg["filt"]:
        ivf_fn = lambda: ivf.search(q, k=k, nprobes=cfg["nprobes"], allow=bm, allow_bits=cfg["n"])  # noqa: E731
        flat_fn = lambda: flat.search(q, k=k, allow=bm, allow_bits=cfg["n"])                        # noqa: E731
    else:
        ivf_fn = lambda: ivf.search_device(dq.data_ptr(), B, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(),  # noqa: E731
                                           torch.cuda.current_stream().cuda_stream)
        flat_fn = lambda: flat.search_device(dq.data_ptr(), B, p, di.data_ptr(), dd.data_ptr(), dc.data_ptr(),  # noqa: E731
                                             torch.cuda.current_stream().cuda_stream)
    ms = time_steps(ivf_fn, steps, warmup)
    flat_ms = time_steps(flat_fn, steps, warmup)
    _native.set_profiling(True)
    got = ivf.search(q, k=k, nprobes=cfg["nprobes"], allow=bm, allow_bits=cfg["n"] if cfg["filt"] else 0)
    stages = {s: round(v, 4) for s, v in _native.last_stage_ms().items()}
    scanned = _native.last_scanned_code_bytes()
    _native.set_profiling(False)
    want = flat.search(q, k=k, allow=bm, allow_bits=cfg["n"] if cfg["filt"] else 0)
    recall = recall_at_k(got, want, k)
    swept = {}
    if not cfg["filt"] and B > 1:
        for npb in sweep:
            ps = _native.make_params(k, npb)
            fn = lambda: ivf.search_device(dq.data_ptr(), B, ps, di.data_ptr(), dd.data_ptr(), dc.data_ptr(),  # noqa: E731
                                           torch.cuda.current_stream().cuda_stream)
            swept[npb] = {"ms": round(time_steps(fn, steps, warmup), 4),
                          "recall": round(recall_at_k(ivf.search(q, k=k, nprobes=npb), want, k), 4)}
    nq = min(B, 16)
    o = ivf_binary_oracle.search(data, q[:nq], k=k, nprobes=cfg["nprobes"], allow=allow,
                                 max_nprobes=cfg["nprobes"] if cfg["filt"] else 0)
    ok = (np.array_equal(got[0][:nq], o[0]) and np.array_equal(got[2][:nq], o[2]) and
          np.array_equal(got[1][:nq].view(np.uint32), o[1].view(np.uint32)))
    rows_probed = scanned // data_nbytes_pad(nb)
    compulsory = rows_probed * nb
    out = {"workload": name, "device": gpu_name, "power_limit": power, "n": cfg["n"], "bits": cfg["bits"],
           "nlist": cfg["nlist"], "nprobes": cfg["nprobes"], "batch": B, "k": k, "prefilter": cfg["filt"],
           "ms": round(ms, 4), "qps": round(B / ms * 1e3, 1), "stages_ms": stages,
           "probed_rows": int(rows_probed), "compulsory_bytes": int(compulsory),
           "compulsory_ms_at_3.35TBps": round(compulsory / HBM_BYTES_PER_S * 1e3, 4),
           "recall_at_k_vs_flat": round(recall, 4), "flat_ms": round(flat_ms, 4),
           "flat_qps": round(B / flat_ms * 1e3, 1), "speedup_vs_flat": round(flat_ms / ms, 2),
           "nprobes_sweep": swept, "train_s": round(train_s, 1), "kmodes_iters": iters, "oracle_ok": bool(ok)}
    print(json.dumps(out), flush=True)
    ivf.close()
    flat.close()


def data_nbytes_pad(nb):
    return (nb + 31) // 32 * 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="IB2,IB1,IB3,IB4")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10, help="k-modes rounds of the trainer")
    ap.add_argument("--sweep", default="10,20,50,100,200", help="nprobes values of the sweep ('' = none)")
    a = ap.parse_args()
    sweep = [int(v) for v in a.sweep.split(",") if v]
    gpu_name, power = device_info()
    for w in a.workloads.split(","):
        run(w, WORKLOADS[w], a.steps, a.warmup, a.iters, sweep, gpu_name, power)


if __name__ == "__main__":
    main()

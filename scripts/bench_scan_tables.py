#!/usr/bin/env python
"""Does the IVF_PQ filter scan wait on its per-query tables?  The scan stage against the batch size on bench.py's C2
index (1M x 768, nlist 1024, m 96, nprobes 20, k 10, latent data, l2).

Each tile of scan3_kernel stages the 16-bit tables of its <= 8 queries (nch x 4 KB per query), so one query's table
is read once per probe slot, and at B 1024 the 50 MB of tables plus the code stream do not fit in the 50 MB L2.  If
re-reading the tables from HBM bounded the scan, the time per probe slot would be clearly lower at B 256 (12.6 MB of
tables, L2-resident) than at B 1024.  One JSON line per batch size: card and power limit, step ms (mean, L2 flushed
between steps as in bench.py), the library's "scan" stage (median of profiled steps), us per probe slot, the modelled
table bytes (footprint, and stagings: one per probe slot -- a lower bound, partitions above 1536 rows stage once per
row block), the L2 size, filter_stats and a hash of the outputs (to compare builds on the same inputs).

    python scripts/bench_scan_tables.py [--batches 256,512,1024,2048] [--steps 20] [--lib path/to/liblancedb_b200.so]

The index is built or loaded as bench.py does (cached under the system's temporary directory).
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:                             # the timings are still worth printing
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,512,1024,2048")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--lib", help="liblancedb_b200.so to load instead of the tree's build")
    args = ap.parse_args()
    if args.lib:
        os.environ["LGPU_LIB_PATH"] = os.path.abspath(args.lib)

    import torch
    import bench
    from lancedb_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_scan_tables.py needs a CUDA device")
    device = "cuda:0"
    cfg = bench.WORKLOADS["c2"]
    ix, _, _, _ = bench.get_index(cfg, "c2", device)
    gpu = _native.GpuIvfPq(ix, device=0, with_vectors=False)
    k, nprobes, dim = cfg["k"], cfg["nprobes"], cfg["dim"]
    nch = (cfg["m"] + 7) // 8
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    dev = card()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    p = _native.make_params(k=k, nprobes=nprobes)
    st = torch.cuda.current_stream().cuda_stream
    for B in [int(b) for b in args.batches.split(",")]:
        nb = 8
        dq = bench.synth_vectors(cfg, nb * B, 43, device).reshape(nb, B, dim)
        d_ids = torch.empty(B, k, dtype=torch.int64, device=device)
        d_dist = torch.empty(B, k, dtype=torch.float32, device=device)
        d_cnt = torch.empty(B, dtype=torch.int32, device=device)

        def step(i):
            gpu.search_device(dq[i % nb].data_ptr(), B, p, d_ids.data_ptr(), d_dist.data_ptr(), d_cnt.data_ptr(), st)

        for i in range(5):
            step(i)
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        for i in range(args.steps):
            flush.zero_()
            ev[i][0].record()
            step(i)
            ev[i][1].record()
        torch.cuda.synchronize()
        step_ms = [a.elapsed_time(b) for a, b in ev]
        stages = []
        _native.set_profiling(True)
        for i in range(args.steps):             # profiled separately: the stage events are not in the timed steps
            flush.zero_()
            step(i)
            torch.cuda.synchronize()
            stages.append(_native.last_stage_ms())
        fstats = _native.last_filter_stats()
        _native.set_profiling(False)
        step(0)
        torch.cuda.synchronize()
        h = hashlib.sha1(d_ids.cpu().numpy().tobytes() + d_dist.cpu().numpy().tobytes() +
                         d_cnt.cpu().numpy().tobytes()).hexdigest()[:16]
        stage = {s: float(np.median([x[s] for x in stages])) for s in stages[0]}
        slots = B * nprobes
        print(json.dumps({
            "device": dev, "batch": B, "step_ms": float(np.mean(step_ms)), "step_ms_min": float(np.min(step_ms)),
            "scan_ms": stage["scan"], "scan_us_per_probe_slot": stage["scan"] * 1e3 / slots, "stage_ms": stage,
            "table_bytes": B * nch * 4096, "table_staging_bytes_min": slots * nch * 4096, "l2_bytes": l2,
            "filter_stats": fstats, "outputs_sha1": h}), flush=True)


if __name__ == "__main__":
    main()

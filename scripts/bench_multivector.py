#!/usr/bin/env python
"""Multivector columns (late interaction, MaxSim over cosine): flat search throughput on the GPU, one JSON line per
workload.

Workloads (seeded latent data: every vector is z A + 0.05 eps with z a rank-32 Gaussian, as in bench.py's notes):
  colbert       100 000 rows x 128 vectors x d 128, nq 32, B 64
  colbert_b1    the same at B 1
  colbert_pf    the same with a 10 % prefilter at B 8
  variable      200 000 rows x 1..256 vectors (mean ~64) x d 128, nq 32, B 64
  colpali       20 000 rows x 1030 vectors x d 128, nq 24, B 16
  below_tc / above_tc  500 / 520 rows x 128 vectors (64 000 / 66 560 stored vectors, either side of the tensor-core
                       path's 65 536-vector threshold), nq 32, B 64
Unfiltered workloads of at least 65 536 stored vectors take the tensor-core path (fp16 MaxSim GEMM -> shortlist ->
exact re-score), the prefiltered one the exact SIMT path; the `path` column is read from the run's filter counters.
--scale shrinks the row counts of the first five (the numbers are then for the smaller column; the line says so).

Per line: device name and power limit (read in the same run), ms per step (median of --steps timed host-buffer calls
after --warmup), QPS, the path, pairwise dot products per second (B * nq * T / time), the share of the H100 SXM's
dense FP16 tensor-core data-sheet rate (989.4 TFLOP/s; 2 d flops per pair) that the whole step reaches, the CPU
oracle's QPS on all threads, and a bit-exact check of --check queries against it."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from lancedb_b200 import _native  # noqa: E402
from tests.multivec_oracle import flat_search_mv, offsets_of  # noqa: E402

WORKLOADS = {
    "colbert": dict(n=100_000, lens=("fixed", 128), dim=128, nq=32, batch=64, filt=0.0),
    "colbert_b1": dict(n=100_000, lens=("fixed", 128), dim=128, nq=32, batch=1, filt=0.0),
    "colbert_pf": dict(n=100_000, lens=("fixed", 128), dim=128, nq=32, batch=8, filt=0.1),
    "variable": dict(n=200_000, lens=("uniform", 256), dim=128, nq=32, batch=64, filt=0.0),
    "colpali": dict(n=20_000, lens=("fixed", 1030), dim=128, nq=24, batch=16, filt=0.0),
    # either side of MV_TC_MIN_T = 65536 stored vectors (the tensor-core path's threshold)
    "below_tc": dict(n=500, lens=("fixed", 128), dim=128, nq=32, batch=64, filt=0.0),
    "above_tc": dict(n=520, lens=("fixed", 128), dim=128, nq=32, batch=64, filt=0.0),
}
FP16_DENSE_FLOPS = 989.4e12
LATENT_RANK = 32


def latent(n, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(LATENT_RANK, dim, generator=torch.Generator(device="cuda").manual_seed(44), device="cuda")
    out = np.empty((n, dim), np.float32)
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        z = torch.randn(e - s, LATENT_RANK, generator=g, device="cuda")
        x = z @ A / LATENT_RANK ** 0.5 + 0.05 * torch.randn(e - s, dim, generator=g, device="cuda")
        out[s:e] = x.cpu().numpy()
    return out


def device_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, power


def run(name, w, args, card, power):
    rng = np.random.default_rng(7)
    n = w["n"] if name.endswith("_tc") else max(1, int(w["n"] * args.scale))
    kind, m = w["lens"]
    lens = np.full(n, m) if kind == "fixed" else rng.integers(1, m + 1, n)
    off = offsets_of(lens)
    x = latent(int(off[-1]), w["dim"], 1)
    B, nq = w["batch"], w["nq"]
    qoff = offsets_of(np.full(B, nq))
    q = latent(B * nq, w["dim"], 2)
    allow = None
    if w["filt"]:
        mask = rng.random(n) < w["filt"]
        allow = (_native.mask_bitmap(mask), n)
    mv = _native.GpuMultivec(x, off)

    def step():
        if allow is None:
            return mv.search(q, k=args.k, q_offsets=qoff)
        return mv.search(q, k=args.k, q_offsets=qoff, allow=allow[0], allow_bits=allow[1])

    for _ in range(args.warmup):
        step()
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        ids, dist, cnt = step()
        times.append(time.perf_counter() - t0)
    ms = float(np.median(times)) * 1e3
    _native.set_profiling(True)
    step()
    st = _native.last_filter_stats()
    _native.set_profiling(False)
    path = "exact-simt" if st["rescored"] == B * n and st["candidates"] == 0 else "tensor-core"
    T = int(off[-1])
    pairs = B * nq * T
    c = min(args.check, B)
    co = offsets_of(np.full(c, nq))
    t0 = time.perf_counter()
    oi, od, oc = flat_search_mv(x, off, q[:c * nq], co, args.k,
                                allow=None if allow is None else mask, nthreads=0)
    cpu_s = time.perf_counter() - t0
    exact = bool(np.array_equal(ids[:c], oi) and np.array_equal(cnt[:c], oc) and
                 np.array_equal(dist[:c].view(np.uint32), od.view(np.uint32)))
    mv.close()
    return dict(workload=name, card=card, power_limit=power, rows=n, vectors=T, dim=w["dim"], nq=nq, batch=B,
                prefilter=w["filt"], scale=args.scale, path=path, rows_rescored=st["rescored"], queries_redone=st["flagged_queries"], ms_per_step=round(ms, 3),
                qps=round(B / (ms / 1e3), 2), pair_dots_per_s=float(f"{pairs / (ms / 1e3):.4g}"),
                fp16_dense_share=float(f"{2 * w['dim'] * pairs / (ms / 1e3) / FP16_DENSE_FLOPS:.4g}"),
                cpu_oracle_qps=round(c / cpu_s, 4), checked_queries=c, bit_exact=exact)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of each workload's rows")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--check", type=int, default=2, help="queries checked bit for bit against the C oracle")
    args = ap.parse_args()
    card, power = device_info()
    for name in args.workloads.split(","):
        print(json.dumps(run(name, WORKLOADS[name], args, card, power)), flush=True)


if __name__ == "__main__":
    main()

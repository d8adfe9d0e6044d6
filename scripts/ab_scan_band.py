#!/usr/bin/env python
"""The filter scan's band on small-norm data: dense-mode flagged queries and step time, one JSON line per scale.

C2-shaped synthetic index (1M x 768, nlist 1024, m 96, random codes and codebooks, component scale s for centroids,
codebooks and queries), batch 1024, nprobes 20, k 10, LGPU_DENSE_FILTER=1 (the band check decides every query).
s = 1/sqrt(768) (unit-norm vectors) and s = 0.02 by default.  Per line: device and power limit, queries the band check
flagged (they go through the exact fix-up), and the median wall time of 10 host-buffer searches after 3 warm-ups.  To
compare two versions, run the script from each version's tree.

    python scripts/ab_scan_band.py [--scale S ...]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_one(scale, steps=10, warmup=3):
    sys.path.insert(0, ROOT)
    os.environ["LGPU_DENSE_FILTER"] = "1"
    from lancedb_b200 import _native
    from tests.util import queries, random_index
    rng = np.random.default_rng(42)
    ix = random_index(rng, dim=768, nlist=1024, m=96, n=1_000_000, scale=scale, shuffle_ids=False)
    Q = queries(np.random.default_rng(43), 1024, 768, scale=scale)
    gpu = _native.GpuIvfPq(ix, with_vectors=False)
    _native.set_profiling(True)
    gpu.search(Q, k=10, nprobes=20)
    st = _native.last_filter_stats()
    _native.set_profiling(False)
    for _ in range(warmup):
        gpu.search(Q, k=10, nprobes=20)
    ts = []
    for _ in range(steps):
        t = time.perf_counter()
        gpu.search(Q, k=10, nprobes=20)
        ts.append(time.perf_counter() - t)
    gpu.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return dict(scale=scale, flagged_queries=st["flagged_queries"], queries=st["queries"],
                ms_per_step=1e3 * float(np.median(ts)), device=smi[0] if smi else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, action="append", default=[])
    a = ap.parse_args()
    for s in a.scale or [1 / np.sqrt(768), 0.02]:
        print(json.dumps(run_one(s)), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Binary vectors (packed uint8, Hamming distance): flat search throughput on the GPU, one JSON line per workload.

Workloads (W1-W4) straddle the path selection of lgpu_binary_search (api.cu, DESIGN.md section 6): W1/W2 batched and
W3 one query take the tensor-core list path, W4 under a 10 % prefilter the SIMT kernel + select; D64 / D256 (60000
rows, inside the dense range 4096..65536) lie either side of the dense tensor-core path's 128-query threshold.
LGPU_NO_TENSOR_CORE=1 in the environment sends every workload through the SIMT kernel, for comparison.  Each runs on two
kinds of data: `latent` = sign bits of rank-32 latent Gaussian vectors (x = z A + 0.05 eps, the construction of
bench.py's data notes; what binary-quantised embeddings look like, many ties) and `uniform` random bits.

Per line: device name and power limit (read in the same run), ms per step and QPS (CUDA events around the device
entry point, after warm-up; W4 times the host-buffer filtered call, which includes its copies), the kernels that ran
(one profiled call), the list-path and tensor-core counters, the HBM lower bound (N * padded row bytes per pass / 3.35 TB/s, the H100
SXM data-sheet bandwidth), the achieved bit-AND-popcount rate B * N * 8 * nbytes / time (NVIDIA publishes no b1
tensor-core peak for the H100, so no share of peak is given), the CPU oracle's QPS on all threads, and a bit-exact
check of 16 queries against it."""
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
from tests.hamming_oracle import flat_search_u8  # noqa: E402

WORKLOADS = {
    "W1": dict(n=10_000_000, bits=1024, batch=1024, k=10, filt=0.0),
    "W2": dict(n=1_000_000, bits=256, batch=1024, k=10, filt=0.0),
    "W3": dict(n=10_000_000, bits=1024, batch=1, k=10, filt=0.0),
    "W4": dict(n=1_000_000, bits=1024, batch=64, k=10, filt=0.1),
    "D64": dict(n=60_000, bits=1024, batch=64, k=10, filt=0.0),
    "D256": dict(n=60_000, bits=1024, batch=256, k=10, filt=0.0),
}
HBM_BYTES_PER_S = 3.35e12
LATENT_RANK = 32


def packed(n, bits, kind, seed):
    """[n, bits / 8] uint8 rows generated on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty(n, bits // 8, dtype=torch.uint8, device="cuda")
    if kind == "uniform":
        return out.random_(0, 256, generator=g).cpu().numpy()
    A = torch.randn(LATENT_RANK, bits, generator=torch.Generator(device="cuda").manual_seed(44), device="cuda")
    w = (2 ** torch.arange(7, -1, -1, device="cuda")).to(torch.int32)
    for s in range(0, n, 1 << 17):
        e = min(n, s + (1 << 17))
        z = torch.randn(e - s, LATENT_RANK, generator=g, device="cuda")
        x = z @ A / LATENT_RANK ** 0.5 + 0.05 * torch.randn(e - s, bits, generator=g, device="cuda")
        out[s:e] = ((x > 0).to(torch.int32).view(e - s, bits // 8, 8) * w).sum(-1).to(torch.uint8)   # np.packbits order
    return out.cpu().numpy()


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
        name = "gemm_dist_kernel<B1Hamming>" if "B1Hamming" in e.key else (m.group(1) if m else e.key)
        out[name] = round(out.get(name, 0.0) + us / 1e3, 4)
    return out


def run(name, cfg, kind, steps, warmup, check, gpu_name, power):
    n, nb, B, k = cfg["n"], cfg["bits"] // 8, cfg["batch"], cfg["k"]
    x = packed(n, cfg["bits"], kind, 1)
    q = packed(4 * B, cfg["bits"], kind, 2).reshape(4, B, nb)
    bx = _native.GpuBinary(x)
    allow = allow_bits = mask = None
    if cfg["filt"]:
        mask = np.random.default_rng(3).random(n) < cfg["filt"]
        allow, allow_bits = _native.mask_bitmap(mask), n
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty(B, k, dtype=torch.int64, device="cuda"); dist = torch.empty(B, k, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    p = _native.make_params(k=k)
    st = torch.cuda.current_stream().cuda_stream
    host_out = {}

    def step(i):
        if allow is None:
            bx.search_device(dq[i % 4].data_ptr(), B, p, ids.data_ptr(), dist.data_ptr(), cnt.data_ptr(), st)
        else:
            host_out["r"] = bx.search(q[i % 4], k=k, allow=allow, allow_bits=allow_bits)

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
    if allow is None:
        gi, gd, gc = ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
    else:
        gi, gd, gc = host_out["r"]
    _native.set_profiling(True)
    step(last)
    torch.cuda.synchronize()
    stats = _native.last_filter_stats()
    _native.set_profiling(False)
    path = kernels_of(lambda: step(last))
    out = {"workload": name, "data": kind, "device": gpu_name, "power_limit": power,
           "config": f"{n} x {cfg['bits']} bits, batch {B}, k {k}" + (f", {cfg['filt']:.0%} prefilter" if mask is not None else ""),
           "ms_per_step": ms, "qps": B / (ms / 1e3), "timed": "device entry point" if allow is None else "host call",
           "kernel_ms": path, "list_candidates": stats["candidates"], "fixup_queries": stats["flagged_queries"],
           "tensor_core_distances": stats["rescored"],
           "hbm_lower_bound_ms": n * ((nb + 31) // 32 * 32) / HBM_BYTES_PER_S * 1e3,
           "bit_and_popc_per_s": B * n * 8.0 * nb / (ms / 1e3)}
    c = min(check, B)
    t0 = time.perf_counter()
    oi, od, oc = flat_search_u8(x, q[last, :c], k, allow=mask, nthreads=os.cpu_count())
    out["oracle_qps_cpu_all_threads"] = c / (time.perf_counter() - t0)
    out["oracle_check"] = bool(np.array_equal(gi[:c], oi) and np.array_equal(gc[:c], oc) and
                               np.array_equal(np.ascontiguousarray(gd[:c]).view(np.uint32), od.view(np.uint32)))
    bx.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="W1,W2,W3,W4,D64,D256")
    ap.add_argument("--data", default="latent,uniform")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="queries verified against the CPU oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_binary.py measures the GPU path and needs a CUDA device")
    gpu_name, power = device_info()
    for w in a.workloads.split(","):
        for kind in a.data.split(","):
            run(w, WORKLOADS[w], kind, a.steps, a.warmup, a.check, gpu_name, power)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""k above 2048 (the global-memory radix select, csrc/select_large.cu): search time, the large select's own time and
its rate, one JSON line per workload.

Workloads:
  pq_k10       C2-shaped IVF_PQ (1M x 768, nlist 1024, m 96, nprobes 20, B 1024, l2), k 10: the reference line
  pq_k4096     the same index at k 4096
  pq_refine    the same index at limit 100 x refine_factor 50 (5000 candidates re-ranked on the raw vectors)
  flat_k10000  flat float 1M x 768, B 64, k 10000
  binary_b1    flat binary 10M x 1024 bits, B 1, k 5000 (one query: the select's slicing spreads it over every SM)
  ivfbin_k4096 binary IVF_FLAT IB2 (1M x 256 bits, nlist 1024, nprobes 20, B 1024), k 4096
The IVF_PQ index is synthetic (random centroids, codebook and codes, uniform partition sizes, as scripts/bench_config.py
builds them): time and exactness do not depend on index quality.  Binary rows are bench_binary.py's latent sign bits.

Per line: device name and power limit (read in the same run), step ms (CUDA events around the device entry point,
median of --steps steps after --warmup), the large select's ms (the summed device time of its kernels, lk_*, in one
profiled call of its own), the candidates it ranked and their rate, the pass-count bound (the bytes its passes must
read at least -- three key-histogram passes over 4-byte distances and a compaction pass over distance and 8-byte id --
at 3.35 TB/s, the H100 SXM data sheet's HBM bandwidth), and a bit-exact check of min(16, B) queries against the C
oracle."""
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
from lancedb_b200.index import IvfPqIndexData, train_ivf_binary  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
NTH = min(32, os.cpu_count() or 1)


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


def select_ms(fn):
    """device ms of the large select's kernels (lk_*) in one profiled call"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if "lk_" in e.key:
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
    return tot


def outputs(B, k):
    return (torch.empty(B, k, dtype=torch.int64, device="cuda"), torch.empty(B, k, device="cuda"),
            torch.empty(B, dtype=torch.int32, device="cuda"))


def host(o, n):
    return o[0][:n].cpu().numpy().view(np.uint64), o[1][:n].cpu().numpy(), o[2][:n].cpu().numpy().view(np.uint32)


def exact(got, want):
    return bool(np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2]) and
                np.array_equal(got[1].view(np.uint32), np.asarray(want[1], np.float32).view(np.uint32)))


def pq_index(with_vectors):
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
    vec = None
    if with_vectors:
        vec = torch.randn(n, dim, generator=torch.Generator(device="cuda").manual_seed(9), device="cuda").cpu().numpy()
    return IvfPqIndexData(dim, nlist, m, "l2", cent, cb, off, codes, np.arange(n, dtype=np.uint64), vec)


def line(name, cfg, step, sel, cand, ok):
    dev, power = device_info()
    bound = cand * (3 * 4 + 12) / HBM_BYTES_PER_S * 1e3
    print(json.dumps(dict(workload=name, device=dev, power_limit=power, **cfg, step_ms=round(step, 4),
                          select_ms=round(sel, 4), candidates=int(cand),
                          candidates_per_s=float(f"{cand / (sel / 1e3):.4g}") if sel > 0 else None,
                          pass_bound_ms=round(bound, 4), oracle_ok=ok)), flush=True)


def run_pq(a, names):
    import oracle
    ix = pq_index("pq_refine" in names)
    gpu = _native.GpuIvfPq(ix, with_vectors=ix.vectors is not None)
    orc = oracle.OracleIndex.from_data(ix)
    B, NP = 1024, 20
    q = torch.randn(B, ix.dim, generator=torch.Generator().manual_seed(3))
    dq = q.cuda()
    st = torch.cuda.current_stream().cuda_stream
    sizes = np.diff(np.asarray(ix.part_offsets, np.int64))
    for name, k, rf in (("pq_k10", 10, 0), ("pq_k4096", 4096, 0), ("pq_refine", 100, 50)):
        if name not in names:
            continue
        o = outputs(B, k)
        p = _native.make_params(k=k, nprobes=NP, refine_factor=rf)

        def fn():
            gpu.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
        step = time_steps(fn, a.steps, a.warmup)
        sel = select_ms(fn)
        parts, _ = gpu.debug_coarse(q.numpy(), NP)
        # the large select's inputs: the PQ top-kk over the probed rows (kk = k x refine_factor), and the re-rank's
        # B x kk exact distances when k itself is above 2048 (k <= 2048 re-ranks on the small selects)
        kk = k * rf if rf else k
        cand = (int(sizes[parts].sum()) if kk > 2048 else 0) + (B * kk if rf and k > 2048 else 0)
        fn()
        torch.cuda.synchronize()
        ok = exact(host(o, 16), orc.search(q[:16].numpy(), k=k, nprobes=NP, refine_factor=rf, nthreads=NTH))
        line(name, dict(B=B, k=k, refine_factor=rf, nprobes=NP), step, sel, cand, ok)
    gpu.close()


def run_flat(a):
    import oracle
    n, dim, B, k = 1_000_000, 768, 64, 10000
    x = torch.randn(n, dim, generator=torch.Generator(device="cuda").manual_seed(11), device="cuda").cpu().numpy()
    fl = _native.GpuFlat(x)
    q = torch.randn(B, dim, generator=torch.Generator().manual_seed(12))
    dq = q.cuda()
    o = outputs(B, k)
    p = _native.make_params(k=k)
    st = torch.cuda.current_stream().cuda_stream

    def fn():
        fl.search_device("l2", dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    step = time_steps(fn, a.steps, a.warmup)
    sel = select_ms(fn)
    fn()
    torch.cuda.synchronize()
    ok = exact(host(o, 16), oracle.flat_search(x, q[:16].numpy(), k=k, nthreads=NTH))
    line("flat_k10000", dict(B=B, k=k, n=n, dim=dim), step, sel, B * n, ok)
    fl.close()


def run_binary(a):
    from tests.hamming_oracle import flat_search_u8
    n, bits, B, k = 10_000_000, 1024, 1, 5000
    x = packed(n, bits, "latent", 7)
    bx = _native.GpuBinary(x)
    rng = np.random.default_rng(5)
    q = x[rng.integers(0, n, B)].copy()
    q ^= (rng.random(q.shape) < 0.05).astype(np.uint8) << rng.integers(0, 8, q.shape).astype(np.uint8)
    dq = torch.from_numpy(q).cuda()
    o = outputs(B, k)
    p = _native.make_params(k=k)
    st = torch.cuda.current_stream().cuda_stream

    def fn():
        bx.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    step = time_steps(fn, a.steps, a.warmup)
    sel = select_ms(fn)
    fn()
    torch.cuda.synchronize()
    ok = exact(host(o, B), flat_search_u8(x, q, k=k, nthreads=NTH))
    line("binary_b1", dict(B=B, k=k, n=n, bits=bits), step, sel, B * n, ok)
    bx.close()


def run_ivf_binary(a):
    from tests import ivf_binary_oracle
    n, bits, nlist, NP, B, k = 1_000_000, 256, 1024, 20, 1024, 4096
    x = packed(n, bits, "latent", 7)
    data = train_ivf_binary(x, num_partitions=nlist, max_iterations=10, device="cuda")
    ib = _native.GpuIvfBinary(data)
    rng = np.random.default_rng(6)
    q = x[rng.integers(0, n, B)].copy()
    q ^= (rng.random(q.shape) < 0.05).astype(np.uint8) << rng.integers(0, 8, q.shape).astype(np.uint8)
    dq = torch.from_numpy(q).cuda()
    o = outputs(B, k)
    p = _native.make_params(k=k, nprobes=NP)
    st = torch.cuda.current_stream().cuda_stream

    def fn():
        ib.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    step = time_steps(fn, a.steps, a.warmup)
    _native.set_profiling(True)
    fn()
    torch.cuda.synchronize()
    cand = _native.last_scanned_code_bytes() // (bits // 8)
    _native.set_profiling(False)
    sel = select_ms(fn)
    fn()
    torch.cuda.synchronize()
    ok = exact(host(o, 16), ivf_binary_oracle.search(data, q[:16], k=k, nprobes=NP, nthreads=NTH))
    line("ivfbin_k4096", dict(B=B, k=k, n=n, bits=bits, nprobes=NP), step, sel, cand, ok)
    ib.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="pq_k10,pq_k4096,pq_refine,flat_k10000,binary_b1,ivfbin_k4096")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_large_k.py measures on the GPU: no CUDA device")
    names = set(a.only.split(","))
    t0 = time.time()
    if names & {"pq_k10", "pq_k4096", "pq_refine"}:
        run_pq(a, names)
    if "flat_k10000" in names:
        run_flat(a)
    if "binary_b1" in names:
        run_binary(a)
    if "ivfbin_k4096" in names:
        run_ivf_binary(a)
    print(json.dumps(dict(total_s=round(time.time() - t0, 1))), flush=True)


if __name__ == "__main__":
    main()

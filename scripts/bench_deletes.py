#!/usr/bin/env python
"""Deleted rows (lgpu_*_delete): what searching a handle with deletions costs, one JSON line per workload.

Workloads:
  flat_l2       flat 1M x 768 f32 L2, B 1024, k 10: unfiltered, 1 % of the rows deleted, and 1 % deleted with
                LGPU_NO_TENSOR_CORE=1 (the exact SIMT route every search with deletions took before the tensor-core
                paths honoured a row filter; run in a child process, the switch is read once)
  W4            flat binary 1M x 1024 bits, B 64, k 10 (bench_binary.py's W4 shape), 1 % deleted and a 10 % prefilter:
                tensor cores against SIMT
  IB4           flat binary 10M x 1024 bits, B 1024, k 10 (the shape of bench_ivf_binary.py's IB4 flat comparison),
                1 % deleted and a 10 % prefilter: tensor cores against SIMT
  C2            C2-shaped IVF_PQ (bench_large_k.py's synthetic 1M x 768, nlist 1024, m 96, nprobes 20, k 10, B 1024)
                unfiltered and with 1 % deleted (a handle with deletions runs every search as a prefiltered one: the
                dense filter mode of the scan, and maximum_nprobes widening)
  delete_10M    lgpu_binary_delete of 1 % of 10M row ids: the first call (builds the live bitmap) and a second one
Data: uniform random rows (time and exactness do not depend on the data here).  Per line: device name and power limit
(read in the same run), step ms (CUDA events around the device entry point, median of --steps after --warmup; the
prefiltered lines time the host-buffer filtered call, which includes the bitmap upload and the result copies) and a
16-query bit-exact check against the oracle under allow' = allow AND NOT deleted."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

import oracle  # noqa: E402
from bench_binary import device_info  # noqa: E402
from bench_large_k import exact, host, outputs, pq_index, time_steps  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from tests import unindexed_oracle as U  # noqa: E402
from tests.hamming_oracle import flat_search_u8  # noqa: E402

K = 10


def _rows(n, width, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == np.uint8:
        return torch.empty(n, width, dtype=torch.uint8, device="cuda").random_(0, 256, generator=g).cpu().numpy()
    return torch.randn(n, width, generator=g, device="cuda").cpu().numpy()


def _live(n, gone, call=None):
    m = np.ones(n, bool) if call is None else call.copy()
    m[gone] = False
    return m


def _emit(**kw):
    dev, power = device_info()
    print(json.dumps(dict(device=dev, power_limit=power, **kw)), flush=True)


def flat_l2(a, route):
    n, dim, B = 1_000_000, 768, 1024
    x = _rows(n, dim, np.float32, 1)
    q = _rows(B, dim, np.float32, 2)
    fl = _native.GpuFlat(x)
    dq = torch.from_numpy(q).cuda()
    o = outputs(B, K)
    p = _native.make_params(K, 0)
    st = torch.cuda.current_stream().cuda_stream

    def run():
        fl.search_device("l2", dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    lines = []
    if route == "tc":
        t = time_steps(run, a.steps, a.warmup)
        run(); torch.cuda.synchronize()
        lines.append(dict(workload="flat_l2", case="unfiltered", step_ms=round(t, 4),
                          oracle_ok=exact(host(o, 16), oracle.flat_search(x, q[:16], K, nthreads=0))))
    gone = np.random.default_rng(3).permutation(n)[:n // 100]
    fl.delete(gone)
    t = time_steps(run, a.steps, a.warmup)
    run(); torch.cuda.synchronize()
    ok = exact(host(o, 16), oracle.flat_search(x, q[:16], K, nthreads=0, allow=_live(n, gone)))
    lines.append(dict(workload="flat_l2", case="1% deleted" + ("" if route == "tc" else ", LGPU_NO_TENSOR_CORE=1"),
                      step_ms=round(t, 4), oracle_ok=ok))
    fl.close()
    for ln in lines:
        _emit(rows=n, dim=dim, B=B, k=K, **ln)


def binary(a, route, name, n, B):
    x = _rows(n, 128, np.uint8, 4)
    q = _rows(B, 128, np.uint8, 5)
    bx = _native.GpuBinary(x)
    dq = torch.from_numpy(q).cuda()
    o = outputs(B, K)
    p = _native.make_params(K, 0)
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(6)
    gone = rng.permutation(n)[:n // 100]
    call = rng.random(n) < 0.1
    bm = _native.mask_bitmap(call)

    def run():
        bx.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    res = {}

    def filtered():
        res["r"] = bx.search(q, k=K, allow=bm, allow_bits=n)
    if route == "tc":
        t = time_steps(run, a.steps, a.warmup)
        _emit(workload=name, case="unfiltered", rows=n, bits=1024, B=B, k=K, step_ms=round(t, 4), oracle_ok=None)
    bx.delete(gone)
    t = time_steps(run, a.steps, a.warmup)
    run(); torch.cuda.synchronize()
    ok = exact(host(o, 16), flat_search_u8(x, q[:16], K, allow=_live(n, gone)))
    tag = "" if route == "tc" else ", LGPU_NO_TENSOR_CORE=1"
    _emit(workload=name, case="1% deleted" + tag, rows=n, bits=1024, B=B, k=K, step_ms=round(t, 4), oracle_ok=ok)
    t = time_steps(filtered, a.steps, a.warmup)
    ok = exact(tuple(r[:16] for r in res["r"]), flat_search_u8(x, q[:16], K, allow=_live(n, gone, call)))
    _emit(workload=name, case="1% deleted + 10% prefilter (host call)" + tag, rows=n, bits=1024, B=B, k=K,
          step_ms=round(t, 4), oracle_ok=ok)
    bx.close()


def c2(a):
    ix = pq_index(False)
    n, B, NP = ix.nrows, 1024, 20
    gpu = _native.GpuIvfPq(ix, with_vectors=False)
    q = torch.randn(B, ix.dim, generator=torch.Generator().manual_seed(3))
    dq = q.cuda()
    o = outputs(B, K)
    p = _native.make_params(k=K, nprobes=NP, max_nprobes=NP)
    st = torch.cuda.current_stream().cuda_stream

    def run():
        gpu.search_device(dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)
    t0 = time_steps(run, a.steps, a.warmup)
    run(); torch.cuda.synchronize()
    ok0 = exact(host(o, 16), U.index_search(ix, q[:16].numpy(), K, NP))
    gone = np.random.default_rng(8).permutation(n)[:n // 100]
    gpu.delete(gone)
    t1 = time_steps(run, a.steps, a.warmup)
    run(); torch.cuda.synchronize()
    ok1 = exact(host(o, 16), U.index_search(ix, q[:16].numpy(), K, NP, allow=_live(n, gone), max_nprobes=NP))
    gpu.close()
    _emit(workload="C2", case="unfiltered", rows=n, B=B, k=K, nprobes=NP, step_ms=round(t0, 4), oracle_ok=ok0)
    _emit(workload="C2", case="1% deleted", rows=n, B=B, k=K, nprobes=NP, step_ms=round(t1, 4), oracle_ok=ok1)


def delete_latency():
    n = 10_000_000
    bx = _native.GpuBinary(_rows(n, 128, np.uint8, 9))
    rng = np.random.default_rng(10)
    ms = []
    for _ in range(2):
        gone = rng.permutation(n)[:n // 100].astype(np.uint64)
        torch.cuda.synchronize()
        t = time.perf_counter()
        got = bx.delete(gone)
        ms.append((time.perf_counter() - t) * 1e3)
    bx.close()
    _emit(workload="delete_10M", ids=n // 100, handle_rows=n, first_delete_ms=round(ms[0], 3),
          second_delete_ms=round(ms[1], 3), last_n_deleted=got)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workloads", default="flat_l2,W4,IB4,C2,delete_10M")
    ap.add_argument("--route", default="tc", choices=["tc", "simt"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    wl = a.workloads.split(",")
    if a.route == "tc":             # the SIMT lines come from a child with LGPU_NO_TENSOR_CORE=1
        simt = [w for w in wl if w in ("flat_l2", "W4", "IB4")]
        if simt:
            env = dict(os.environ, LGPU_NO_TENSOR_CORE="1")
            subprocess.run([sys.executable, __file__, "--route", "simt", "--workloads", ",".join(simt),
                            "--steps", str(a.steps), "--warmup", str(a.warmup)], env=env, check=True)
    for w in wl:
        if w == "flat_l2":
            flat_l2(a, a.route)
        elif w == "W4":
            binary(a, a.route, "W4", 1_000_000, 64)
        elif w == "IB4":
            binary(a, a.route, "IB4", 10_000_000, 1024)
        elif w == "C2" and a.route == "tc":
            c2(a)
        elif w == "delete_10M" and a.route == "tc":
            delete_latency()


if __name__ == "__main__":
    main()

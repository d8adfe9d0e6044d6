#!/usr/bin/env python
"""Multivector (MaxSim) search from vectors kept in pinned host memory (LGPU_MULTIVEC_HBM_BYTES=0) against vectors in
HBM, in one run.

Workloads (fixed row lengths, latent-factor vectors as in bench_multivector.py, k 10):
  colbert_b1   50 000 rows x 128 vectors x d 128, nq 32, B 1        (tensor-core route)
  colbert      the same at B 64                                     (tensor-core route)
  colpali      10 000 rows x 1030 vectors x d 128, nq 24, B 16      (tensor-core route)
  colbert_pf   the colbert column with a 10 % prefilter at B 8      (tensor-core route under the prefilter)
Each column is opened with both placements at a size that fits HBM.

Prints one JSON line each for
  device     the card's name and power limit, read in this run
  memcpy     pinned host -> device cudaMemcpy bandwidth (1 GiB, CUDA events), the PCIe yardstick
  workload   ms per call of each placement (CUDA events around lgpu_multivec_search_device, median of --steps, the two
             handles alternated call by call); open time of each placement (host clock); the PCIe bytes of one host call
             split into the streamed operand (fp16 on the tensor-core route, f32 on the exact one), the re-score's reads
             of the admitted rows (rows re-scored x row bytes x ceil(nq / 64), from lgpu_last_filter_stats) and the
             fix-up's copies (the f32 rows per pass when a query was flagged, else 0); their rate over the host call's
             time and its share of the memcpy rate; the device time of the re-score kernel and of the fix-up's
             launches (torch.profiler, one call; run with LGPU_NO_PDL=1 for these, since a kernel launched with
             programmatic dependent launch is timed from when it starts waiting on its predecessor); whether both placements returned the same bits on every timed call,
             and whether the first query equals the C oracle bit for bit
  oversized  a column larger than free HBM: not measured by this script
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from bench_binary import device_info, kernels_of  # noqa: E402
from bench_host_vectors import emit, memcpy_gbs  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from tests.multivec_oracle import flat_search_mv, offsets_of  # noqa: E402

K, DIM = 10, 128
WORKLOADS = [("colbert_b1", "colbert", 32, 1, 0.0), ("colbert", "colbert", 32, 64, 0.0),
             ("colpali", "colpali", 24, 16, 0.0), ("colbert_pf", "colbert", 32, 8, 0.1)]
COLUMNS = {"colbert": (50_000, 128), "colpali": (10_000, 1030)}
FIXUP = ("mv_copy_gated", "mv_rowmin", "mv_rowsum", "dist_matrix")


def latent(gen, n, rank=16):
    A = torch.randn(rank, DIM, generator=gen, device="cuda")
    return torch.randn(n, rank, generator=gen, device="cuda") @ A + 0.3 * torch.randn(n, DIM, generator=gen,
                                                                                      device="cuda")


def open_both(x, off):
    os.environ.pop("LGPU_MULTIVEC_HBM_BYTES", None)
    t0 = time.time()
    hbm = _native.GpuMultivec(x, off)
    t_hbm = time.time() - t0
    os.environ["LGPU_MULTIVEC_HBM_BYTES"] = "0"
    t0 = time.time()
    host = _native.GpuMultivec(x, off)
    t_host = time.time() - t0
    del os.environ["LGPU_MULTIVEC_HBM_BYTES"]
    assert host.rows_on_host and not hbm.rows_on_host
    return hbm, host, t_hbm, t_host


def workload(name, hbm, host, x, off, nq, B, filt, opened, bw, a):
    n, L = COLUMNS[name.split("_")[0]]
    T = n * L
    gen = torch.Generator(device="cuda").manual_seed(B + nq)
    q = latent(gen, B * nq).contiguous()
    qoff = offsets_of(np.full(B, nq))
    allow, bits = None, 0
    if filt:
        mask = np.random.default_rng(1).random(n) < filt
        allow, bits = _native.mask_bitmap(mask), n
    st = torch.cuda.current_stream().cuda_stream
    p = _native.make_params(k=K)
    outs = {nm: (h, torch.empty(B, K, dtype=torch.int64, device="cuda"), torch.empty(B, K, device="cuda"),
                 torch.empty(B, dtype=torch.int32, device="cuda")) for nm, h in (("hbm", hbm), ("host", host))}

    def call(nm):
        h, oi, od, oc = outs[nm]
        if allow is None:
            h.search_device(q.data_ptr(), qoff, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
        else:                                    # the prefilter takes the host-buffer filtered entry point
            r = h.search(q.cpu().numpy(), k=K, q_offsets=qoff, allow=allow, allow_bits=bits)
            oi.copy_(torch.from_numpy(r[0].view(np.int64))); od.copy_(torch.from_numpy(r[1]))
            oc.copy_(torch.from_numpy(r[2].view(np.int32)))

    ms = {"hbm": [], "host": []}
    same = True
    for i in range(a.warmup + a.steps):
        for nm in ("hbm", "host"):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            call(nm)
            e.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                ms[nm].append(s.elapsed_time(e))
        if i >= a.warmup:
            same &= all(torch.equal(outs["hbm"][j], outs["host"][j]) for j in (1, 3)) and \
                torch.equal(outs["hbm"][2].view(torch.int32), outs["host"][2].view(torch.int32))
    _native.set_profiling(True)
    call("host")
    torch.cuda.synchronize()
    stats = _native.last_filter_stats()
    _native.set_profiling(False)
    ker = kernels_of(lambda: call("host"))
    rescore_ms = sum(v for kk, v in ker.items() if "mv_rescore_host" in kk)
    fixup_ms = sum(v for kk, v in ker.items() if any(f in kk for f in FIXUP))
    tc = stats["rescored"] < B * n
    stream_b = T * DIM * (2 if tc else 4)
    rescore_b = stats["rescored"] * L * DIM * 4 * -(-nq // 64) if tc else 0
    fixup_b = T * DIM * 4 if tc and stats["flagged_queries"] else 0
    t_hbm, t_host = float(np.median(ms["hbm"])), float(np.median(ms["host"]))
    rate = (stream_b + rescore_b + fixup_b) / (t_host / 1e3) / 1e9
    qq = q[:nq].cpu().numpy()
    want = flat_search_mv(x, off, qq, qoff[:2], K, allow=None if allow is None else mask, nthreads=os.cpu_count())
    got = [outs["host"][j][:1].cpu().numpy() for j in (1, 2, 3)]
    oracle_same = np.array_equal(got[0].view(np.uint64), want[0]) and \
        np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)) and np.array_equal(got[2].view(np.uint32), want[2])
    emit(line="workload", name=name, rows=n, vectors_per_row=L, dim=DIM, nq=nq, B=B, k=K, prefilter=filt,
         route="tensor-core" if tc else "exact", ms_hbm=round(t_hbm, 3), ms_host=round(t_host, 3),
         open_s_hbm=opened[0], open_s_host=opened[1], pcie_operand_bytes=stream_b, pcie_rescore_bytes=rescore_b,
         pcie_fixup_bytes=fixup_b, pcie_GBps=round(rate, 2), share_of_memcpy=round(rate / bw, 3),
         rescore_kernel_ms=round(rescore_ms, 3), fixup_launches_ms=round(fixup_ms, 3), flagged=stats["flagged_queries"],
         rows_rescored=stats["rescored"], same_results=bool(same), oracle_bit_exact_first_query=bool(oracle_same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    bw = memcpy_gbs()
    emit(line="memcpy", h2d_pinned_GBps=round(bw, 2))
    for col, (n, L) in COLUMNS.items():
        gen = torch.Generator(device="cuda").manual_seed(n)
        x = latent(gen, n * L).cpu().numpy()
        off = offsets_of(np.full(n, L))
        hbm, host, t_hbm, t_host = open_both(x, off)
        for name, c, nq, B, filt in WORKLOADS:
            if c == col:
                workload(name, hbm, host, x, off, nq, B, filt, (round(t_hbm, 3), round(t_host, 3)), bw, a)
        hbm.close(); host.close()
        del x
    emit(line="oversized", status="not measured")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Float16 multivector handles (lgpu_multivec_open_f16) against f32 handles opened on the same rows upcast to f32,
alternated call by call in one run.

Columns (fixed row lengths, latent-factor vectors as in bench_multivector.py, stored as float16, k 10):
  colbert   20 000 rows x 128 vectors x d 128, nq 32
  colpali    2 000 rows x 1030 vectors x d 128, nq 24
Each column is opened four times: fp16 and f32, in HBM and in pinned host memory (LGPU_MULTIVEC_HBM_BYTES=0).
Workloads per placement: colbert at B 1 and B 64 and colpali at B 16, with no filter and with a 10 % prefilter (the
route each call took is reported; run with LGPU_NO_TENSOR_CORE=1 for the exact route).

Prints one JSON line each for
  device     the card's name and power limit, read in this run
  workload   ms per call of the fp16 and the f32 handle (CUDA events, median of --steps; the device entry point, or the
             host-buffer filtered entry point for the prefilter), device_bytes and host_bytes of both handles, the PCIe
             bytes of one call on a host handle (the streamed rows -- the fp16 operand on the tensor-core route for both
             row types, the stored vectors in the row type on the exact route -- plus the re-score's reads of the
             admitted rows and, when a query was flagged, the fix-up's copies), rows re-scored (lgpu_last_filter_stats)
             by both, and whether both handles returned the same bits on every timed call
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from bench_binary import device_info  # noqa: E402
from bench_host_vectors import emit  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from tests.multivec_oracle import offsets_of  # noqa: E402

K, DIM = 10, 128
COLUMNS = {"colbert": (20_000, 128, 32, (1, 64)), "colpali": (2_000, 1030, 24, (16,))}


def latent(gen, n, rank=16):
    A = torch.randn(rank, DIM, generator=gen, device="cuda")
    return torch.randn(n, rank, generator=gen, device="cuda") @ A + 0.3 * torch.randn(n, DIM, generator=gen,
                                                                                      device="cuda")


def open_pair(x16, off, host):
    if host:
        os.environ["LGPU_MULTIVEC_HBM_BYTES"] = "0"
    try:
        f16 = _native.GpuMultivec(x16, off)
        f32 = _native.GpuMultivec(x16.astype(np.float32), off)
    finally:
        os.environ.pop("LGPU_MULTIVEC_HBM_BYTES", None)
    assert f16.rows_on_host == host and f32.rows_on_host == host and f16.dtype == np.float16
    return {"f16": f16, "f32": f32}


def workload(col, handles, placement, nq, B, filt, a):
    n, L = COLUMNS[col][:2]
    T = n * L
    gen = torch.Generator(device="cuda").manual_seed(B + nq)
    q = latent(gen, B * nq).contiguous()
    qn = q.cpu().numpy()
    qoff = offsets_of(np.full(B, nq))
    mask = np.random.default_rng(1).random(n) < filt if filt else None
    st = torch.cuda.current_stream().cuda_stream
    p = _native.make_params(k=K)
    outs = {nm: (h, torch.empty(B, K, dtype=torch.int64, device="cuda"), torch.empty(B, K, device="cuda"),
                 torch.empty(B, dtype=torch.int32, device="cuda")) for nm, h in handles.items()}

    def call(nm):
        h, oi, od, oc = outs[nm]
        if mask is None:
            h.search_device(q.data_ptr(), qoff, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
        else:                                    # the prefilter takes the host-buffer filtered entry point
            r = h.search(qn, k=K, q_offsets=qoff, allow=_native.mask_bitmap(mask), allow_bits=n)
            oi.copy_(torch.from_numpy(r[0].view(np.int64))); od.copy_(torch.from_numpy(r[1]))
            oc.copy_(torch.from_numpy(r[2].view(np.int32)))

    ms = {"f16": [], "f32": []}
    same = True
    for i in range(a.warmup + a.steps):
        for nm in ("f16", "f32"):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            call(nm)
            e.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                ms[nm].append(s.elapsed_time(e))
        if i >= a.warmup:
            same &= all(torch.equal(outs["f16"][j], outs["f32"][j]) for j in (1, 3)) and \
                torch.equal(outs["f16"][2].view(torch.int32), outs["f32"][2].view(torch.int32))
    stats = {}
    for nm in ("f16", "f32"):
        _native.set_profiling(True)
        call(nm)
        torch.cuda.synchronize()
        stats[nm] = _native.last_filter_stats()
        _native.set_profiling(False)
    tc = stats["f16"]["rescored"] < B * n
    pcie = {}
    for nm, es in (("f16", 2), ("f32", 4)):
        if placement != "host":
            pcie[nm] = 0
            continue
        s = stats[nm]
        stream_b = T * DIM * (2 if tc else es)
        rescore_b = s["rescored"] * L * DIM * es * -(-nq // 64) if tc else 0
        fixup_b = T * DIM * es if tc and s["flagged_queries"] else 0
        pcie[nm] = stream_b + rescore_b + fixup_b
    emit(line="workload", column=col, placement=placement, rows=n, vectors_per_row=L, dim=DIM, nq=nq, B=B, k=K,
         prefilter=filt, route="tensor-core" if tc else "exact",
         ms_f16=round(float(np.median(ms["f16"])), 3), ms_f32=round(float(np.median(ms["f32"])), 3),
         device_bytes_f16=handles["f16"].device_bytes, device_bytes_f32=handles["f32"].device_bytes,
         host_bytes_f16=handles["f16"].host_bytes(), host_bytes_f32=handles["f32"].host_bytes(),
         pcie_bytes_f16=pcie["f16"], pcie_bytes_f32=pcie["f32"],
         rows_rescored_f16=stats["f16"]["rescored"], rows_rescored_f32=stats["f32"]["rescored"],
         flagged_f16=stats["f16"]["flagged_queries"], flagged_f32=stats["f32"]["flagged_queries"],
         same_results=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scale", type=float, default=1.0, help="multiply the row counts (a quick run: 0.05)")
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    for col, (n, L, nq, Bs) in list(COLUMNS.items()):
        n = max(1, int(n * a.scale))
        COLUMNS[col] = (n, L, nq, Bs)
        gen = torch.Generator(device="cuda").manual_seed(n)
        x16 = latent(gen, n * L).half().cpu().numpy()
        off = offsets_of(np.full(n, L))
        for placement in ("hbm", "host"):
            handles = open_pair(x16, off, placement == "host")
            for filt in (0.0, 0.1):
                for B in Bs:
                    workload(col, handles, placement, nq, B, filt, a)
            for h in handles.values():
                h.close()
        del x16


if __name__ == "__main__":
    main()

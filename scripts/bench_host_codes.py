#!/usr/bin/env python
"""IVF search from codes kept in pinned host memory (LGPU_CODES_HBM_BYTES=0) against codes in HBM, in one run.

Shapes: IVF_SQ at 10M x 768 (7.68 GB of codes), nlist 4096, nprobes 20 and 50, opened through lgpu_ivf_sq_open from
random codes and centroids (parity between the placements needs no training); binary IVF_FLAT at 10M x 1024 bits
(IB1 of bench_ivf_binary.py: 1.28 GB of packed rows), nlist 4096, nprobes 20.  B 1, 64 and 1024, k 10.
--huge N also opens one IVF_SQ index of N x 768 under no cap (it goes to the host when it does not fit in HBM) and
searches it once.

Prints one JSON line each for
  device        the card's name and power limit, read in this run
  memcpy        pinned host -> device cudaMemcpy bandwidth (1 GiB, CUDA events), the PCIe yardstick
  open          per shape: open time of the two placements (host clock), the HBM each handle holds (cudaMemGetInfo
                before and after its open) and the pinned code bytes of the host handle
  case          per shape, nprobes and B: ms per call of each placement (CUDA events around the _device call, median of
                --steps, the two handles alternated call by call), the bytes the host call's gated copies moved
                (lgpu_last_streamed_code_bytes of a profiled call on the same queries), their rate over the host call's
                time and its share of the memcpy rate, and whether both placements returned the same ids, counts and
                distance bits on every timed call
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

from bench_binary import device_info  # noqa: E402
from bench_host_vectors import emit, memcpy_gbs  # noqa: E402
from lancedb_b200 import _native  # noqa: E402
from lancedb_b200.index import IvfBinaryIndexData, IvfSqIndexData  # noqa: E402

K, NLIST = 10, 4096


def layout(n, seed):
    """part_offsets of NLIST partitions of about n / NLIST rows each (multinomial sizes), row ids 0..n-1"""
    sizes = np.random.default_rng(seed).multinomial(n, np.full(NLIST, 1.0 / NLIST))
    off = np.zeros(NLIST + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    return off, np.arange(n, dtype=np.uint64)


def rand_u8(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=g).cpu().numpy()


def sq_data(n, dim=768):
    off, rid = layout(n, 1)
    c = np.random.default_rng(2).standard_normal((NLIST, dim)).astype(np.float32)
    return IvfSqIndexData(dim=dim, nlist=NLIST, metric="l2", centroids=c, part_offsets=off, codes=rand_u8((n, dim), 3),
                          row_ids=rid, lo=-3.0, hi=3.0)


def binary_data(n, nbytes=128):
    off, rid = layout(n, 4)
    return IvfBinaryIndexData(nbytes=nbytes, nlist=NLIST, centroids=rand_u8((NLIST, nbytes), 5), part_offsets=off,
                              vectors=rand_u8((n, nbytes), 6), row_ids=rid)


def open_one(cls, data, cap):
    if cap is None:
        os.environ.pop("LGPU_CODES_HBM_BYTES", None)
    else:
        os.environ["LGPU_CODES_HBM_BYTES"] = cap
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.time()
    h = cls(data, device=0, **({} if cls is _native.GpuIvfBinary else dict(with_vectors=False)))
    t = time.time() - t0
    held = free0 - torch.cuda.mem_get_info()[0]
    os.environ.pop("LGPU_CODES_HBM_BYTES", None)
    return h, t, held


def open_both(name, cls, data):
    hbm, t_hbm, held_hbm = open_one(cls, data, None)
    host, t_host, held_host = open_one(cls, data, "0")
    assert host.codes_on_host and not hbm.codes_on_host
    emit(line="open", shape=name, hbm_s=round(t_hbm, 3), host_s=round(t_host, 3), hbm_held_hbm=held_hbm,
         hbm_held_host=held_host, code_host_bytes=host.code_host_bytes())
    return hbm, host


def streamed(h, q, nprobes):
    _native.set_profiling(True)
    try:
        h.search(q, k=K, nprobes=nprobes)
        return _native.last_streamed_code_bytes()
    finally:
        _native.set_profiling(False)


def run(name, hbm, host, make_q, nprobes_list, bs, bw, a):
    st = torch.cuda.current_stream().cuda_stream
    for nprobes in nprobes_list:
        for B in bs:
            dq = make_q(B)
            p = _native.make_params(k=K, nprobes=nprobes)
            outs = {nm: (h, torch.empty(B, K, dtype=torch.int64, device="cuda"), torch.empty(B, K, device="cuda"),
                         torch.empty(B, dtype=torch.int32, device="cuda")) for nm, h in (("hbm", hbm), ("host", host))}
            ms = {"hbm": [], "host": []}
            same = True
            for i in range(a.warmup + a.steps):
                for nm, (h, oi, od, oc) in outs.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    h.search_device(dq.data_ptr(), B, p, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), st)
                    e.record()
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        ms[nm].append(s.elapsed_time(e))
                if i >= a.warmup:
                    same &= all(torch.equal(outs["hbm"][j], outs["host"][j]) for j in (1, 3)) and \
                        torch.equal(outs["hbm"][2].view(torch.int32), outs["host"][2].view(torch.int32))
            t_hbm, t_host = float(np.median(ms["hbm"])), float(np.median(ms["host"]))
            moved = streamed(host, dq.cpu().numpy(), nprobes)
            rate = moved / (t_host / 1e3) / 1e9
            emit(line="case", shape=name, nprobes=nprobes, B=B, k=K, ms_hbm=round(t_hbm, 3), ms_host=round(t_host, 3),
                 ms_hbm_spread=[round(min(ms["hbm"]), 3), round(max(ms["hbm"]), 3)],
                 ms_host_spread=[round(min(ms["host"]), 3), round(max(ms["host"]), 3)],
                 pcie_bytes_per_call=moved, streamed_GBps=round(rate, 2), share_of_memcpy=round(rate / bw, 3),
                 same_results=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--huge", type=int, default=0, help="rows of an IVF_SQ index at dim 768 opened under no cap")
    a = ap.parse_args()
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    bw = memcpy_gbs()
    emit(line="memcpy", h2d_pinned_GBps=round(bw, 2))
    bs = (1, 64, 1024)

    data = sq_data(a.rows)
    hbm, host = open_both("sq-768", _native.GpuIvfSq, data)
    del data
    gen = torch.Generator(device="cuda").manual_seed(7)
    run("sq-768", hbm, host, lambda B: torch.randn(B, 768, device="cuda", generator=gen), (20, 50), bs, bw, a)
    hbm.close(); host.close()

    data = binary_data(a.rows)
    hbm, host = open_both("binary-1024", _native.GpuIvfBinary, data)
    del data
    run("binary-1024", hbm, host,
        lambda B: torch.randint(0, 256, (B, 128), dtype=torch.uint8, device="cuda", generator=gen), (20,), bs, bw, a)
    hbm.close(); host.close()

    if a.huge:
        data = sq_data(a.huge)
        h, t, held = open_one(_native.GpuIvfSq, data, None)
        del data
        q = torch.randn(64, 768, device="cuda", generator=gen).cpu().numpy()
        t0 = time.time()
        ids, dist, cnt = h.search(q, k=K, nprobes=20)
        emit(line="huge", rows=a.huge, codes_on_host=h.codes_on_host, open_s=round(t, 1), hbm_held=held,
             code_host_bytes=h.code_host_bytes(), search_B64_s=round(time.time() - t0, 3), full=bool((cnt == K).all()))
        h.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Float16 flat handles (lgpu_flat_open_f16) against f32 handles on the same rows' exact f32 upcast, one JSON line per
workload.

Workloads (seeded float16 rows and f32 queries, standard normal, k 10):
  C4        1M x 1536, B 1024, l2 (the tensor-core path: sampled threshold, fp16 wgmma against bf16 wgmma)
  C4cos     the same shape under cosine (the exact kernels on both row types)
  F768b1    1M x 768, B 1, l2 (the exact kernels: B < 8)
  F768b64   1M x 768, B 64, l2 (the tensor-core path)
The two handles are timed alternately in one run (--rounds rounds of --steps device-route calls after --warmup; the
median of all steps), and their full outputs at the timed batch are compared bit for bit.  Per line: device name and
power limit (read in the same run), ms per batch of each handle, their lgpu_flat_device_bytes, bytes per row, and the
largest row count each row type admits at dim 1536 on this card: its total memory over the bytes per row measured on
the C4 handles after a cosine search (row norms allocated; search workspaces not counted).  Nothing is allocated to
find that count."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from bench_binary import device_info  # noqa: E402
from bench_large_k import host, outputs  # noqa: E402
from lancedb_b200 import _native  # noqa: E402

K = 10


def _rows(n, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, dim, generator=g, device="cuda").half().cpu().numpy()


def _queries(B, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, dim, generator=g, device="cuda")


def _timed(fls, metric, dq, steps, warmup, rounds):
    """median ms per call of each handle, alternating handles every `steps` calls; the outputs of each"""
    B = dq.shape[0]
    p = _native.make_params(K, 0)
    st = torch.cuda.current_stream().cuda_stream
    outs = [outputs(B, K) for _ in fls]

    def call(i):
        o = outs[i]
        fls[i].search_device(metric, dq.data_ptr(), B, p, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), st)

    for i in range(len(fls)):
        for _ in range(warmup):
            call(i)
    torch.cuda.synchronize()
    ts = [[] for _ in fls]
    for _ in range(rounds):
        for i in range(len(fls)):
            for _ in range(steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call(i)
                b.record()
                b.synchronize()
                ts[i].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in ts], [host(o, B) for o in outs]


def run(name, n, dim, B, metric, steps, warmup, rounds, cache):
    key = (n, dim)
    if key not in cache:
        for fl in cache.pop("handles", []):
            fl.close()
        cache.clear()
        x16 = _rows(n, dim, 1)
        cache[key] = True
        cache["handles"] = [_native.GpuFlat(x16), _native.GpuFlat(x16.astype(np.float32))]
        del x16
    f16, f32 = cache["handles"]
    dq = _queries(B, dim, 2)
    (ms16, ms32), (o16, o32) = _timed([f16, f32], metric, dq, steps, warmup, rounds)
    same = bool(np.array_equal(o16[0], o32[0]) and np.array_equal(o16[2], o32[2]) and
                np.array_equal(o16[1].view(np.uint32), o32[1].view(np.uint32)))
    b16, b32 = f16.device_bytes, f32.device_bytes
    line = dict(workload=name, n=n, dim=dim, B=B, k=K, metric=metric, ms_f16=round(ms16, 3), ms_f32=round(ms32, 3),
                device_bytes_f16=b16, device_bytes_f32=b32, identical_outputs=same)
    return line, b16 / n, b32 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload names")
    a = ap.parse_args()
    dev, power = device_info()
    total = torch.cuda.get_device_properties(0).total_memory
    work = [("C4", 1_000_000, 1536, 1024, "l2"), ("C4cos", 1_000_000, 1536, 1024, "cosine"),
            ("F768b1", 1_000_000, 768, 1, "l2"), ("F768b64", 1_000_000, 768, 64, "l2")]
    if a.only:
        work = [w for w in work if w[0] in a.only.split(",")]
    cache = {}
    for name, n, dim, B, metric in work:
        steps = max(1, a.steps // 3) if metric == "cosine" else a.steps
        line, r16, r32 = run(name, n, dim, B, metric, steps, a.warmup, a.rounds, cache)
        if name == "C4cos":
            line.update(bytes_per_row_f16=round(r16, 2), bytes_per_row_f32=round(r32, 2), card_bytes=total,
                        max_rows_dim1536_f16=int(total // r16), max_rows_dim1536_f32=int(total // r32))
        print(json.dumps(dict(device=dev, power_limit=power, **line)), flush=True)
    for fl in cache.get("handles", []):
        fl.close()


if __name__ == "__main__":
    main()

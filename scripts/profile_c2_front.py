#!/usr/bin/env python
"""Timeline of the front of one bench.py C2 step (1M x 768, IVF_PQ nlist 1024, m 96, nprobes 20, k 10, B 1024).

Builds or loads the C2 index exactly as bench.py does, runs warm steps (L2 flushed between them, as in bench.py)
under torch.profiler with CUDA activity, and prints, per kernel and per stream, the median start and end relative
to the step start (the end of the flush), then the critical path of the step's front:
  - when gemm_dist_kernel starts compared with the first query-table CTA;
  - when the tables end compared with the end of the regroup (the scan waits for both);
  - how long scan3_kernel runs compared with the library's own "scan" stage (stage events on the search stream).
The card's name and power limit are read in the same run.  Writes trace.json and timeline.json under --out.

    python scripts/profile_c2_front.py [--out DIR] [--lib path/to/liblancedb_b200.so]

--out defaults to a directory under the system's temporary directory, so the tree is left untouched.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TABLE_KERNELS = ("qtable_minmax_kernel", "qtable_quant_kernel", "qtable_kernel")
GROUP_KERNELS = ("group_count_kernel", "group_scan_kernel", "group_fill_kernel", "tile_desc_kernel", "group_kernel")


def short_name(n):
    n = n.replace("(anonymous namespace)", "anon")
    n = re.sub(r"^void\s+", "", n)
    n = re.split(r"[<(]", n, 1)[0]
    return n.split("::")[-1]


def card():
    out = {}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        out = {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:                             # the timeline is still worth printing
        out = {"error": repr(e)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "profile_c2_front"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", help="liblancedb_b200.so to load instead of the tree's build")
    args = ap.parse_args()
    if args.lib:
        os.environ["LGPU_LIB_PATH"] = os.path.abspath(args.lib)
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from lancedb_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("profile_c2_front.py needs a CUDA device")
    device = "cuda:0"
    cfg = bench.WORKLOADS["c2"]
    ix, _, _, _ = bench.get_index(cfg, "c2", device)
    gpu = _native.GpuIvfPq(ix, device=0, with_vectors=False)
    B, k, dim, nb = cfg["batch"], cfg["k"], cfg["dim"], 8
    dq = bench.synth_vectors(cfg, nb * B, 43, device).reshape(nb, B, dim)
    d_ids = torch.empty(B, k, dtype=torch.int64, device=device)
    d_dist = torch.empty(B, k, dtype=torch.float32, device=device)
    d_cnt = torch.empty(B, dtype=torch.int32, device=device)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    p = _native.make_params(k=k, nprobes=cfg["nprobes"])
    st = torch.cuda.current_stream().cuda_stream

    def step(i):
        gpu.search_device(dq[i % nb].data_ptr(), B, p, d_ids.data_ptr(), d_dist.data_ptr(), d_cnt.data_ptr(), st)

    for i in range(args.warmup):
        flush.zero_()
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            flush.zero_()
            step(i)
        torch.cuda.synchronize()
    trace = os.path.join(args.out, "trace.json")
    prof.export_chrome_trace(trace)

    # the library's stage split (CUDA events on the search stream), in a run of its own
    _native.set_profiling(True)
    stages = collections.defaultdict(list)
    for i in range(args.steps):
        flush.zero_()
        step(i)
        for kk, v in _native.last_stage_ms().items():
            stages[kk].append(v)
    _native.set_profiling(False)
    torch.cuda.synchronize()
    gpu.close()

    with open(trace) as f:
        ev = json.load(f)["traceEvents"]
    kern = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    steps = []                                          # per step: [(name, stream, start, end)] relative to the flush end
    cur, t0 = None, None
    for e in kern:
        name = short_name(e["name"])
        if "lgpu" not in e["name"]:                     # the flush (torch) opens a step
            cur, t0 = [], e["ts"] + e["dur"]
            steps.append(cur)
            continue
        if cur is not None:
            cur.append((name, e["args"].get("stream"), e["ts"] - t0, e["ts"] + e["dur"] - t0))
    steps = [s for s in steps if s]
    if not steps:
        raise SystemExit("no library kernels in the trace")
    # the search stream is the one the scan runs on
    main_stream = next((x[1] for s in steps for x in s if x[0] == "scan3_kernel"), steps[0][0][1])
    rows = collections.OrderedDict()                    # (name, occurrence, stream) -> [(start, end)]
    for s in steps:
        seen = collections.Counter()
        for name, strm, a, b in s:
            key = (name, seen[(name, strm)], "search" if strm == main_stream else f"side({strm})")
            seen[(name, strm)] += 1
            rows.setdefault(key, []).append((a, b))
    med = lambda v: float(np.median(v))
    timeline = [{"kernel": n, "occurrence": o, "stream": s, "start_us": med([a for a, _ in v]),
                 "end_us": med([b for _, b in v]), "dur_us": med([b - a for a, b in v]), "steps": len(v)}
                for (n, o, s), v in rows.items()]
    timeline.sort(key=lambda r: r["start_us"])

    def per_step(fn):
        vals = [fn(s) for s in steps]
        vals = [v for v in vals if v is not None]
        return med(vals) if vals else None

    first = lambda s, names, f: min((f(x) for x in s if x[0] in names), default=None)
    last = lambda s, names, f: max((f(x) for x in s if x[0] in names), default=None)
    crit = {
        "gemm_start_us": per_step(lambda s: first(s, ("gemm_dist_kernel",), lambda x: x[2])),
        "gemm_end_us": per_step(lambda s: last(s, ("gemm_dist_kernel",), lambda x: x[3])),
        "first_table_start_us": per_step(lambda s: first(s, TABLE_KERNELS, lambda x: x[2])),
        "tables_end_us": per_step(lambda s: last(s, TABLE_KERNELS, lambda x: x[3])),
        "coarse_finish_end_us": per_step(lambda s: last(s, ("coarse_finish_kernel",), lambda x: x[3])),
        # the regroup before the scan (the exact fix-up pass after it regroups again)
        "group_end_us": per_step(lambda s: max((x[3] for x in s if x[0] in GROUP_KERNELS and
                                                x[2] < first(s, ("scan3_kernel",), lambda y: y[2])), default=None)),
        "scan3_start_us": per_step(lambda s: first(s, ("scan3_kernel",), lambda x: x[2])),
        "scan3_kernel_us": per_step(lambda s: sum(x[3] - x[2] for x in s if x[0] == "scan3_kernel") or None),
        "step_end_us": per_step(lambda s: max(x[3] for x in s)),
    }
    if crit["tables_end_us"] is not None and crit["group_end_us"] is not None:
        crit["join_wait_us"] = max(0.0, crit["tables_end_us"] - crit["group_end_us"])
    stage_ms = {kk: med(v) for kk, v in stages.items()}
    crit["scan_stage_us"] = stage_ms.get("scan", 0.0) * 1e3
    info = {"card": card(), "lib": os.environ.get("LGPU_LIB_PATH") or _native.LIB_PATH, "steps": len(steps),
            "stage_ms": stage_ms, "critical_path": crit, "timeline": timeline}
    with open(os.path.join(args.out, "timeline.json"), "w") as f:
        json.dump(info, f, indent=1)

    print(f"card: {info['card']}")
    print(f"{'kernel':32s} {'#':>2s} {'stream':12s} {'start_us':>9s} {'end_us':>9s} {'dur_us':>8s}")
    for r in timeline:
        print(f"{r['kernel'][:32]:32s} {r['occurrence']:2d} {r['stream']:12s} {r['start_us']:9.1f} {r['end_us']:9.1f} "
              f"{r['dur_us']:8.1f}")
    print("critical path (us from the step start, median over steps):")
    for kk, v in crit.items():
        print(f"  {kk:22s} {'-' if v is None else f'{v:9.1f}'}")
    print("stage_ms (library events): " + ", ".join(f"{kk} {v:.3f}" for kk, v in stage_ms.items()))


if __name__ == "__main__":
    main()

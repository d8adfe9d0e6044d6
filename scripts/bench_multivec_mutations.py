#!/usr/bin/env python
"""Multivector columns that change: appends in place against close + reopen, and filtered searches on the
tensor-core route against the exact route, in one run.

Column: DESIGN.md section 7's multivector shape, 20 000 rows x 128 vectors at d 128 (latent-factor vectors as in
bench_multivector.py), queries of nq 32, B 64, k 10; f32 and fp16 handles, rows in HBM and in pinned host memory
(LGPU_MULTIVEC_HBM_BYTES=0).

Prints one JSON line each for
  device    the card's name and power limit, read in this run
  append    per row type, placement and growth (1 %, 10 %, 100 % more rows), median of --steps repeats: host-clock
            seconds of lgpu_multivec_append and of close + reopen over the grown column, and ms of the first search
            after each (CUDA events); whether the two handles then return the same bits
  filtered  per row type, placement and filter (0 %, 1 %, 10 % deleted; a prefilter allowing 30 %, 1 %, and fewer
            than k rows): ms per call (median of --steps, host-buffer filtered entry point) on the tensor-core route and
            on the exact route (LGPU_NO_TENSOR_CORE=1, which the library reads once per process: two server processes
            hold the same handles and are called alternately); the route each took, rows admitted and rows re-scored
            (lgpu_last_filter_stats); whether the routes agree bit for bit and the first query equals the C oracle's
"""
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

N, L, DIM, NQ, B, K = 20_000, 128, 128, 32, 64, 10
DTYPES = ("f32", "f16")
PLACES = ("hbm", "host")
# (name, share of rows deleted, share of rows a prefilter allows; None: no prefilter), in the order they run: a
# server's deletes stay, so the prefilters run before them, and the 10 % deleted are a superset of the 1 %
FILTERS = [("deleted_0", 0.0, None), ("prefilter_30pct", 0.0, 0.30), ("prefilter_1pct", 0.0, 0.01),
           ("prefilter_below_k", 0.0, (K // 2) / N), ("deleted_1pct", 0.01, None), ("deleted_10pct", 0.10, None)]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def column(seed=0):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((16, DIM)).astype(np.float32)
    x = (rng.standard_normal((N * L, 16)).astype(np.float32) @ A).astype(np.float32)
    x += 0.3 * rng.standard_normal(x.shape, dtype=np.float32)
    q = (rng.standard_normal((B * NQ, 16)).astype(np.float32) @ A + 0.3 * rng.standard_normal((B * NQ, DIM))).astype(
        np.float32)
    return x, q


def open_handle(x, off, place, row_ids=None):
    from lancedb_b200 import _native
    if place == "host":
        os.environ["LGPU_MULTIVEC_HBM_BYTES"] = "0"
    h = _native.GpuMultivec(x, off, row_ids=row_ids)
    os.environ.pop("LGPU_MULTIVEC_HBM_BYTES", None)
    assert h.rows_on_host == (place == "host")
    return h


def timed_search(h, q, qoff, **kw):
    import torch
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    r = h.search(q, k=K, q_offsets=qoff, **kw)
    e.record()
    torch.cuda.synchronize()
    return r, s.elapsed_time(e)


def serve():
    """One route's server: opens every (row type, placement) handle once, then answers 'name dtype place steps'
    lines with one JSON line of median ms, the counters and the result bits."""
    from lancedb_b200 import _native
    from tests.multivec_oracle import offsets_of
    x, q = column()
    off = offsets_of(np.full(N, L))
    qoff = offsets_of(np.full(B, NQ))
    handles = {}
    for dt in DTYPES:
        xv = x.astype(np.float16) if dt == "f16" else x
        for place in PLACES:
            handles[dt, place] = open_handle(xv, off, place)
    del x
    print("ready", flush=True)
    deleted = set()
    for line in sys.stdin:
        name, dt, place, steps = line.split()
        _, gone, allow = next(f for f in FILTERS if f[0] == name)
        h = handles[dt, place]
        want_gone = int(gone * N)
        if want_gone and (dt, place, want_gone) not in deleted:     # deletes grow: 1 % then 10 % (a superset)
            h.delete(np.arange(0, N, N // want_gone, dtype=np.uint64)[:want_gone])
            deleted.add((dt, place, want_gone))
        kw = {}
        if allow is not None:
            mask = np.zeros(N, bool)
            mask[np.random.default_rng(2).choice(N, max(1, int(round(allow * N))), replace=False)] = True
            kw = dict(allow=_native.mask_bitmap(mask), allow_bits=N)
        ms = []
        for _ in range(int(steps)):
            r, t = timed_search(h, q, qoff, **kw)
            ms.append(t)
        _native.set_profiling(True)
        h.search(q, k=K, q_offsets=qoff, **kw)
        st = _native.last_filter_stats()
        _native.set_profiling(False)
        print(json.dumps(dict(ms=float(np.median(ms)), stats=st, ids=r[0].tolist(), dist=r[1].view(np.uint32).tolist(),
                              cnt=r[2].tolist())), flush=True)


def filtered(a):
    from tests.multivec_oracle import flat_search_mv, offsets_of
    procs = {}
    for route, extra in (("tensor-core", {}), ("exact", {"LGPU_NO_TENSOR_CORE": "1"})):
        env = dict(os.environ, PYTHONPATH=ROOT, **extra)
        procs[route] = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--serve"], stdin=subprocess.PIPE,
                                        stdout=subprocess.PIPE, text=True, env=env, cwd=ROOT)
        assert procs[route].stdout.readline().strip() == "ready"
    x, q = column()
    off = offsets_of(np.full(N, L))
    try:
        for dt in DTYPES:
            for place in PLACES:
                for name, gone, allow in FILTERS:
                    res = {}
                    for rep in range(2):                            # warm-up round, then the timed round
                        for route in ("tensor-core", "exact"):      # alternated
                            p = procs[route]
                            p.stdin.write(f"{name} {dt} {place} {a.steps if rep else a.warmup}\n")
                            p.stdin.flush()
                            res[route] = json.loads(p.stdout.readline())
                    tc, ex = res["tensor-core"], res["exact"]
                    same = all(tc[f] == ex[f] for f in ("ids", "dist", "cnt"))
                    live = np.ones(N, bool)
                    if gone:
                        live[np.arange(0, N, N // int(gone * N))[:int(gone * N)]] = False
                    if allow is not None:
                        mask = np.zeros(N, bool)
                        mask[np.random.default_rng(2).choice(N, max(1, int(round(allow * N))), replace=False)] = True
                        live &= mask
                    xv = x.astype(np.float16).astype(np.float32) if dt == "f16" else x
                    want = flat_search_mv(xv, off, q[:NQ], [0, NQ], K, allow=live, nthreads=os.cpu_count())
                    oracle_same = (tc["ids"][0] == want[0][0].tolist() and tc["cnt"][0] == int(want[2][0]) and
                                   tc["dist"][0] == want[1][0].view(np.uint32).tolist())
                    emit(line="filtered", workload=name, dtype=dt, placement=place, allowed_rows=int(live.sum()),
                         ms_tensor_core=round(tc["ms"], 3), ms_exact=round(ex["ms"], 3),
                         speedup=round(ex["ms"] / tc["ms"], 2),
                         route_taken="tensor-core" if tc["stats"]["rescored"] < B * N else "exact",
                         rows_admitted=tc["stats"]["candidates"], rows_rescored=tc["stats"]["rescored"],
                         flagged=tc["stats"]["flagged_queries"], exact_route_rescored=ex["stats"]["rescored"],
                         routes_same_bits=bool(same), oracle_bit_exact_first_query=bool(oracle_same))
    finally:
        for p in procs.values():
            p.stdin.close()
            p.wait()


def appends(a):
    """Each (row type, placement, growth) is measured --steps times, append and close + reopen alternated; medians."""
    from tests.multivec_oracle import offsets_of
    x, q = column()
    qoff = offsets_of(np.full(B, NQ))
    for dt in DTYPES:
        xv = x.astype(np.float16) if dt == "f16" else x
        for place in PLACES:
            for share in (0.01, 0.10, 1.0):
                m = int(share * N)
                grown = np.concatenate([xv, xv[:m * L]])
                t = {"append": [], "reopen": [], "search_append": [], "search_reopen": []}
                same = True
                for _ in range(a.steps):
                    h = open_handle(xv, offsets_of(np.full(N, L)), place)
                    t0 = time.time()
                    h.append(xv[:m * L], offsets_of(np.full(m, L)))
                    t["append"].append(time.time() - t0)
                    r1, ms = timed_search(h, q, qoff)
                    t["search_append"].append(ms)
                    h.close()
                    h = open_handle(xv, offsets_of(np.full(N, L)), place)
                    t0 = time.time()
                    h.close()
                    h = open_handle(grown, offsets_of(np.full(N + m, L)), place)
                    t["reopen"].append(time.time() - t0)
                    r2, ms = timed_search(h, q, qoff)
                    t["search_reopen"].append(ms)
                    h.close()
                    same &= all(np.array_equal(u.view(np.uint32), v.view(np.uint32)) for u, v in zip(r1, r2))
                med = {kk: float(np.median(v)) for kk, v in t.items()}
                emit(line="append", dtype=dt, placement=place, rows=N, appended_rows=m, repeats=a.steps,
                     append_s=round(med["append"], 3), close_reopen_s=round(med["reopen"], 3),
                     first_search_ms_after_append=round(med["search_append"], 3),
                     first_search_ms_after_reopen=round(med["search_reopen"], 3),
                     first_search_ms_after_append_all=[round(v, 1) for v in t["search_append"]], same_bits=bool(same))
                del grown


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--serve", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.serve:
        return serve()
    from bench_binary import device_info
    dev, power = device_info()
    emit(line="device", device=dev, power_limit=power)
    filtered(a)
    appends(a)


if __name__ == "__main__":
    main()

"""The cases of tests/test_gpu_sub_batches.py: searches whose workspace does not fit LGPU_WS_BYTES, so the library cuts the
batch into sub-batches of queries.  LGPU_WS_BYTES is read once per process, so the test runs this module as a child,

    python -m tests.sub_batch_cases <group> <out.npz> [--rehearse]

once with the default budget and once with the group's small one, and compares what the two children wrote.  A child
runs every case of one group on seeded data and stores, per case, the GPU's ids / distances / counts, the
kernel_launch_count() delta of the call, the oracle's answer (when SUB_BATCH_ORACLE=1) and whatever else the case
reports (sub-batch size from lgpu_debug_sub_batch_size, profiling counters).

--rehearse needs no device: it builds the data, runs the oracle, and checks the batch shapes against an estimate of the
sub-batch size (`_ivf_bs`), so that seeds, shapes and paths are debugged before a GPU is involved.  The estimate only
picks batch sizes; with a device the child asserts it against the library's own answer, and the test proves the split
from the launch counts."""
import contextlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MiB = 1 << 20
# group -> (small LGPU_WS_BYTES, CUDA graphs on)
GROUPS = {
    "pq8_l2": (MiB, False), "pq8_cosine": (MiB, False), "pq8_dot": (MiB, False),
    "pq8_small_tail": (16 * MiB, False), "pq8_tc_coarse": (MiB, False),
    "pq4": (MiB, False), "sq": (MiB, False), "rq": (MiB, False), "ivf_binary": (MiB, False),
    "flat": (MiB, False), "flat_big": (10 * MiB, False), "binary_flat": (MiB, False),
    "routes": (MiB, False), "graphs": (MiB, True), "timeout": (MiB, False), "profiling": (MiB, False),
}
NTH = min(16, os.cpu_count() or 1)
U64_MAX = np.iinfo(np.uint64).max


class Ctx:
    def __init__(self, gpu: bool, want_oracle: bool):
        self.gpu, self.want_oracle = gpu, want_oracle
        self.split = "LGPU_WS_BYTES" in os.environ          # this child runs under the small budget
        self.budget = int(os.environ.get("LGPU_WS_BYTES", 8 << 30))
        self.out = {}

    def put(self, case, **arrays):
        for k, v in arrays.items():
            self.out[f"{case}/{k}"] = np.asarray(v)

    def result(self, case, got, prefix=""):
        self.put(case, **{prefix + "ids": got[0], prefix + "dist": got[1], prefix + "cnt": got[2]})

    def run(self, case, call, oracle_call, env=None):
        """One case: `call()` on the GPU under `env` (the library re-reads its mode switches on every call), with the
        launch-count delta; `oracle_call()` on the CPU."""
        from lancedb_b200 import _native
        if self.gpu:
            with _env(env or {}):
                n0 = _native.kernel_launch_count()
                got = call()
                self.put(case, launches=_native.kernel_launch_count() - n0)
            self.result(case, got)
        if self.want_oracle or not self.gpu:
            self.result(case, oracle_call(), "o_")

    def sub_batch(self, case, gpu, B, nprobes, est=None):
        """Record the library's sub-batch size for the case; under the small budget `est` (the estimate the batch
        shape was chosen from) must be what the library picks."""
        if not self.gpu:
            return
        bs = gpu.debug_sub_batch_size(B, nprobes)
        self.put(case, bs=bs, B=B)
        if self.split and est is not None:
            assert bs == min(est, B), f"{case}: the library picks sub-batches of {bs}, the case was shaped for {est}"


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    for k, v in env.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _ivf_bs(sizes, nlist, nprobes, budget, fixed=0, per_probe=0):
    """Estimate of the IVF sub-batch size, for shaping batches: the budget over one query's distance segments (its
    nprobes largest partitions, each padded to 4 rows, 4 bytes a row), coarse scores (4 bytes a partition), `fixed`
    bytes (8-bit PQ: 8192 per 8 sub-vectors of exact tables) and `per_probe` bytes per probe slot."""
    pads = np.sort((np.asarray(sizes, np.int64) + 3) // 4 * 4)[::-1]
    per_q = int(pads[:min(nprobes, nlist)].sum()) * 4 + nlist * 4 + fixed + nprobes * per_probe
    return max(1, min(budget // max(per_q, 4), 65535))


def _sizes(ix):
    return np.diff(np.asarray(ix.part_offsets, np.int64))


def _mask(rng, row_ids, frac):
    """A random allow mask over row ids (bool [max id + 1]) and its bitmap"""
    from lancedb_b200 import _native
    m = rng.random(int(np.max(row_ids)) + 1) < frac
    return m, _native.mask_bitmap(m)


def _oracle_bitmap(mask):
    import oracle
    return oracle.allow_bitmap(np.nonzero(mask)[0], mask.size)


def _open(ctx, cls, *a, **kw):
    return cls(*a, **kw) if ctx.gpu else None


# ---- IVF_PQ, 8-bit ----
def _pq8_index(metric, seed=1):
    from tests.util import random_index
    rng = np.random.default_rng(seed)
    return rng, random_index(rng, dim=64, nlist=16, m=16, metric=metric, n=40000, with_vectors=True)


def _pq8(ctx, metric):
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries
    rng, ix = _pq8_index(metric)
    orc = oracle.OracleIndex.from_data(ix)
    gpu = _open(ctx, _native.GpuIvfPq, ix)
    NP, B = 8, 37
    bs = _ivf_bs(_sizes(ix), 16, NP, MiB, fixed=2 * 8192)
    assert 4 <= bs <= 12 and B % bs, bs              # 1 MiB: four or more sub-batches, a ragged tail
    q = queries(rng, B, 64)

    def case(name, env=None, qq=q, **kw):
        okw = dict(kw)
        if "allow" in okw:
            mask = okw.pop("allow")
            kw = dict(kw, allow=_native.mask_bitmap(mask), allow_bits=mask.size)
            okw.update(allow=_oracle_bitmap(mask), allow_bits=mask.size)
        ctx.sub_batch(name, gpu, len(qq), max(kw.get("nprobes", NP), kw.get("max_nprobes", 0) if "allow" in kw else 0))
        ctx.run(name, lambda: gpu.search(qq, **kw), lambda: orc.search(qq, nthreads=NTH, **okw), env)

    ctx.sub_batch("shape", gpu, B, NP, est=bs)
    case("k10", k=10, nprobes=NP)                                    # warp selector, 512-entry candidate lists
    case("k100", k=100, nprobes=NP)                                  # block selector, 2048-entry candidate lists
    case("dense_filter", {"LGPU_DENSE_FILTER": 1}, k=10, nprobes=NP)
    case("exact_scan", {"LGPU_EXACT_SCAN": 1}, k=10, nprobes=NP)
    case("cand_cap32", {"LGPU_CAND_CAP": 32}, k=10, nprobes=NP)      # every list overflows: the fix-up has work
    d = orc.search(q[:1], k=200, nprobes=NP)[1][0]
    case("range", k=20, nprobes=NP, lower=float(d[15]), upper=float(d[150]))
    case("refine", k=10, nprobes=NP, refine_factor=3)                # re-ranks on the raw queries, not the normalised
    case("refine_k100", k=100, nprobes=NP, refine_factor=2)          # 200 candidates: the dense filter mode
    half, _ = _mask(rng, ix.row_ids, 0.5)
    thin, _ = _mask(rng, ix.row_ids, 0.02)
    case("prefilter_half", k=10, nprobes=NP, allow=half)
    case("prefilter_thin", k=10, nprobes=NP, allow=thin)
    # widening: the allowed rows are those of partitions 0..7.  A query nearest to one of them finds k rows in its one
    # probe; a query nearest to partitions 8..15 finds none and is searched again over maximum_nprobes = 8.  The
    # second sub-batch holds only queries of the first sort (nothing to widen), the others a mix.
    ids = np.asarray(ix.row_ids, np.int64)
    off = np.asarray(ix.part_offsets, np.int64)
    lo8 = np.zeros(int(ids.max()) + 1, bool)
    lo8[ids[:off[8]]] = True
    pool = queries(rng, 400, 64)
    near = np.array([int(orc.find_partitions(oracle.normalize(v) if metric == "cosine" else v, 1)[0][0]) for v in pool])
    sat, starved = pool[near < 8], pool[near >= 8]
    assert len(sat) >= B and len(starved) >= B, (len(sat), len(starved))
    qw = sat[:B].copy()
    mix = [i for i in range(B) if not bs <= i < 2 * bs and i % 3 != 1]
    qw[mix] = starved[:len(mix)]
    case("widen", qq=qw, k=10, nprobes=1, max_nprobes=NP, allow=lo8)
    if ctx.want_oracle or not ctx.gpu:
        oc = ctx.out["widen/o_cnt"]
        assert (oc == 10).all()                                      # every starved query found its rows by widening
    # a NaN query first in the second sub-batch, an all-zero query inside the first
    qn = q.copy()
    qn[bs, 5] = np.nan
    qn[2] = 0
    case("nan_zero", qq=qn, k=10, nprobes=NP)
    case("nan_zero_dense", {"LGPU_DENSE_FILTER": 1}, qq=qn, k=10, nprobes=NP)
    if gpu:
        gpu.close()


def _pq8_small_tail(ctx):
    """Full sub-batches above 1024 probe slots (filter scan, candidate mode), a tail below (small.cu), in one call"""
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries
    rng, ix = _pq8_index("l2")
    orc = oracle.OracleIndex.from_data(ix)
    gpu = _open(ctx, _native.GpuIvfPq, ix)
    NP = 8
    bs = _ivf_bs(_sizes(ix), 16, NP, 16 * MiB, fixed=2 * 8192)
    B = 2 * bs + 11
    assert bs * NP > 1024 >= 11 * NP
    q = queries(rng, B, 64)
    ctx.sub_batch("shape", gpu, B, NP, est=bs)
    for name, slots in (("batched_tail", "0"), ("small_tail", None)):      # None: the library's default (1024)
        ctx.run(name, lambda: gpu.search(q, k=10, nprobes=NP), lambda: orc.search(q, k=10, nprobes=NP, nthreads=NTH),
                {"LGPU_SMALL_SLOTS": slots})
    if gpu:
        gpu.close()


def _pq8_tc_coarse(ctx):
    """nlist 1024 with the tensor-core coarse step forced: sub-batches of 8 or more take it, a tail below 8 the exact
    coarse kernels; then the list variant (LGPU_COARSE_LIST_MIN = 1024; it needs the centroid sample, kept from 1024
    lists)"""
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries, random_index
    for metric in ("l2", "cosine"):
        rng = np.random.default_rng(5)
        ix = random_index(rng, dim=64, nlist=1024, m=16, metric=metric, n=60000)
        orc = oracle.OracleIndex.from_data(ix)
        gpu = _open(ctx, _native.GpuIvfPq, ix, with_vectors=False)
        NP = 8
        bs = _ivf_bs(_sizes(ix), 1024, NP, MiB, fixed=2 * 8192)
        B = 2 * bs + 5
        assert bs >= 8
        q = queries(rng, B, 64)
        ctx.sub_batch(f"{metric}_shape", gpu, B, NP, est=bs)
        for name, env in (("dense", {"LGPU_FORCE_TC_COARSE": 1}),
                          ("list", {"LGPU_FORCE_TC_COARSE": 1, "LGPU_COARSE_LIST_MIN": 1024}),
                          ("exact", {})):
            ctx.run(f"{metric}_{name}", lambda: gpu.search(q, k=10, nprobes=NP),
                    lambda: orc.search(q, k=10, nprobes=NP, nthreads=NTH), env)
        if gpu:
            gpu.close()


# ---- the other IVF kinds ----
def _kind_cases(ctx, tag, gpu, data, search, q, NP, refine, bs_probe=None):
    """plain search at k 10 and k 100, distance_range, refine_factor, prefilter, prefilter + widening.
    search(queries, **kw): the kind's oracle (allow = bool mask over row ids)."""
    from lancedb_b200 import _native
    rng = np.random.default_rng(17)
    B = len(q)

    def case(name, **kw):
        okw = dict(kw)
        if "allow" in kw:
            mask = kw["allow"]
            kw = dict(kw, allow=_native.mask_bitmap(mask), allow_bits=mask.size)
        if bs_probe:
            ctx.sub_batch(f"{tag}{name}", gpu, B, max(kw["nprobes"], kw.get("max_nprobes", 0)))
        ctx.run(f"{tag}{name}", lambda: gpu.search(q, **kw), lambda: search(q, nthreads=NTH, **okw))

    case("k10", k=10, nprobes=NP)
    case("k100", k=100, nprobes=NP)
    d = search(q[:1], k=200, nprobes=NP, nthreads=NTH)[1][0]
    d = d[np.isfinite(d)]
    case("range", k=20, nprobes=NP, lower=float(d[len(d) // 10]), upper=float(d[len(d) * 3 // 4]))
    if refine:
        case("refine", k=10, nprobes=NP, refine_factor=3)
    half, _ = _mask(rng, data.row_ids, 0.5)
    case("prefilter_half", k=10, nprobes=NP, allow=half)
    # thin enough that some queries find fewer than 10 rows in NP probes and are searched again; where the partitions
    # allow it, others find 10 and are not
    if NP == 1:                      # one probe: 2 allowed rows in the largest partition, 15 in the next, 2, 15, ...
        ids, off = np.asarray(data.row_ids, np.int64), np.asarray(data.part_offsets, np.int64)
        thin = np.zeros(int(ids.max()) + 1, bool)
        for rank, p in enumerate(np.argsort(-_sizes(data), kind="stable")):
            thin[rng.choice(ids[off[p]:off[p + 1]], min(15 if rank % 2 else 2, off[p + 1] - off[p]), replace=False)] = True
    else:
        rows = float(np.sort(_sizes(data))[::-1][:NP].sum())
        thin, _ = _mask(rng, data.row_ids, min(0.5, 12.0 / rows))
    case("widen", k=10, nprobes=NP, max_nprobes=data.nlist, allow=thin)
    if ctx.want_oracle or not ctx.gpu:
        plain = search(q, k=10, nprobes=NP, allow=thin, nthreads=NTH)[2]
        assert (plain < 10).any(), "the widening case needs queries that find fewer than k rows"
        assert NP > 1 or (plain == 10).any(), "the one-probe widening case needs queries that are left alone too"


def _near_centroids(rng, data, B):
    """query i near centroid i mod nlist, so that a one-probe search visits every partition in turn"""
    c = np.asarray(data.centroids, np.float32)
    return (c[np.arange(B) % data.nlist] + 0.3 * rng.standard_normal((B, c.shape[1]))).astype(np.float32)


def _pq4(ctx):
    from lancedb_b200 import _native
    from tests import pq4_oracle
    from tests.util import queries
    rng = np.random.default_rng(2)
    for tag, kw, NP, B in (("seg_", dict(n=40000, dim=64, nlist=16, m=16), 8, 37),       # distance segments set the size
                           ("tab_", dict(n=3200, dim=256, nlist=64, m=128), 32, 45)):    # the per-slot u8 tables do
        for metric in ("l2", "cosine") if tag == "seg_" else ("l2",):
            ix = pq4_oracle.random_pq4_index(rng, metric=metric, empty=(), **kw)
            gpu = _open(ctx, _native.GpuIvfPq, ix)
            q = queries(rng, B, kw["dim"])
            _kind_cases(ctx, f"{tag}{metric}_", gpu, ix, lambda qq, **k: pq4_oracle.search(ix, qq, **k), q, NP, True, True)
            if gpu:
                gpu.close()


def _sq(ctx):
    from lancedb_b200 import _native
    from tests import sq_oracle
    from tests.util import queries
    rng = np.random.default_rng(3)
    for metric in ("l2", "cosine"):
        ix = sq_oracle.random_sq_index(rng, n=100000, dim=32, nlist=4, metric=metric, empty=(),
                                       unit_centroids=metric == "cosine")
        assert (_sizes(ix) > 2048).all()                     # every partition populated, cosine included
        gpu = _open(ctx, _native.GpuIvfSq, ix)
        q = _near_centroids(rng, ix, 37)
        _kind_cases(ctx, f"{metric}_", gpu, ix, lambda qq, **k: sq_oracle.search(ix, qq, **k), q, 1, True, True)
        if gpu:
            gpu.close()


def _rq(ctx):
    from lancedb_b200 import _native
    from tests import rq_oracle
    from tests.util import queries
    rng = np.random.default_rng(4)
    for tag, kw, NP, B in (("seg_", dict(n=100000, dim=32, nlist=4), 1, 37),             # distance segments set the size
                           ("planes_", dict(n=1280, dim=512, nlist=64), 32, 101)):       # the per-slot bit-planes do
        for metric in ("l2", "cosine") if tag == "seg_" else ("l2",):
            ix = rq_oracle.random_rq_index(rng, metric=metric, empty=(), unit_centroids=metric == "cosine", **kw)
            assert NP > 1 or (_sizes(ix) > 2048).all()       # one-probe shapes: every partition populated
            gpu = _open(ctx, _native.GpuIvfRq, ix)
            q = _near_centroids(rng, ix, B) if NP == 1 else queries(rng, B, kw["dim"])
            _kind_cases(ctx, f"{tag}{metric}_", gpu, ix, lambda qq, **k: rq_oracle.search(ix, qq, **k), q, NP, True, True)
            if gpu:
                gpu.close()


def _ivf_binary(ctx):
    from lancedb_b200 import _native
    from tests import ivf_binary_oracle as ibo
    rng = np.random.default_rng(6)
    ix = ibo.random_index(rng, 100000, 16, 4)
    gpu = _open(ctx, _native.GpuIvfBinary, ix)
    q = np.concatenate([ix.vectors[rng.integers(0, 100000, 20)], rng.integers(0, 256, (17, 16), dtype=np.uint8)])
    _kind_cases(ctx, "", gpu, ix, lambda qq, **k: ibo.search(ix, qq, **k), q, 1, False)
    if gpu:
        gpu.close()


# ---- flat ----
def _flat(ctx):
    """N = 8192: a row of scores is 32 KiB, so 1 MiB gives sub-batches of 32; 69 queries run as 32 + 32 + 5, the l2
    tail below the 8 queries the tensor-core shortlist needs"""
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries
    rng = np.random.default_rng(7)
    N, dim, B = 8192, 32, 69
    v = queries(rng, N, dim)
    q = queries(rng, B, dim)
    q[33] = 0                                                        # cosine: no direction, first rows of sub-batch 2
    rid = rng.permutation(N).astype(np.uint64) * 2 + 1
    mask = rng.random(2 * N + 1) < 0.3
    bm = _native.mask_bitmap(mask)
    for ids_tag, ids in (("", None), ("rid_", rid)):
        fl = _open(ctx, _native.GpuFlat, v, row_ids=ids)
        for metric in ("cosine", "l2", "dot"):                       # cosine first: the row norms are computed by a split call
            t = f"{ids_tag}{metric}_"
            ora = lambda **kw: oracle.flat_search(v, q, metric=metric, row_ids=ids, nthreads=NTH, **kw)
            ctx.run(t + "k10", lambda: fl.search(q, k=10, metric=metric), lambda: ora(k=10))
            ctx.run(t + "k100", lambda: fl.search(q, k=100, metric=metric), lambda: ora(k=100))
            d = ora(k=200)[1][0]
            lo, hi = float(d[20]), float(d[150])
            ctx.run(t + "range", lambda: fl.search(q, k=50, metric=metric, lower=lo, upper=hi),
                    lambda: ora(k=50, lower=lo, upper=hi))
            ctx.run(t + "prefilter", lambda: fl.search(q, k=10, metric=metric, allow=bm, allow_bits=mask.size),
                    lambda: ora(k=10, allow=_oracle_bitmap(mask), allow_bits=mask.size))
        if fl:
            fl.close()


def _flat_big(ctx):
    """N = 262144: a row of scores is 1 MiB, so 10 MiB gives sub-batches of 10; 25 queries run as 10 + 10 + 5 -- the
    filtered tensor-core variant, then the exact kernels for the tail"""
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries
    rng = np.random.default_rng(8)
    v = queries(rng, 262144, 16)
    q = queries(rng, 25, 16)
    fl = _open(ctx, _native.GpuFlat, v)
    for name, env in (("filtered", {"LGPU_FLAT_DENSE": None}), ("dense", {"LGPU_FLAT_DENSE": 1})):
        ctx.run(name, lambda: fl.search(q, k=10), lambda: oracle.flat_search(v, q, k=10, nthreads=NTH), env)
    if fl:
        fl.close()


def _binary_flat(ctx):
    """N = 60000 <= 65536 rows: the dense (non-list) branch.  A row of scores is 240 KB: sub-batches of 4.  The kernel
    is chosen from the size of the whole batch, not of the sub-batch: with 131 queries every 4-query sub-batch goes
    through the b1 tensor-core kernel (its M tail), with 21 queries through the SIMT kernel."""
    from lancedb_b200 import _native
    from tests.hamming_oracle import flat_search_u8
    rng = np.random.default_rng(9)
    N = 60000
    x = rng.integers(0, 256, (N, 16), dtype=np.uint8)
    rid = rng.permutation(N).astype(np.uint64) * 2 + 1
    mask = rng.random(2 * N + 1) < 0.3
    bm = _native.mask_bitmap(mask)
    bx = _open(ctx, _native.GpuBinary, x, row_ids=rid)
    for tag, B in (("wgmma_", 131), ("simt_", 21)):                  # the b1 tensor-core kernel from 128 queries
        q = np.concatenate([x[:3], rng.integers(0, 256, (B - 3, 16), dtype=np.uint8)])
        ctx.run(tag + "k10", lambda: bx.search(q, k=10), lambda: flat_search_u8(x, q, 10, row_ids=rid, nthreads=NTH))
        ctx.run(tag + "k100", lambda: bx.search(q, k=100), lambda: flat_search_u8(x, q, 100, row_ids=rid, nthreads=NTH))
        ctx.run(tag + "prefilter", lambda: bx.search(q, k=10, allow=bm, allow_bits=mask.size),
                lambda: flat_search_u8(x, q, 10, row_ids=rid, allow=mask, nthreads=NTH))
        ctx.run(tag + "range", lambda: bx.search(q, k=20, lower=50.0, upper=58.0),
                lambda: flat_search_u8(x, q, 20, row_ids=rid, lower=50.0, upper=58.0, nthreads=NTH))
    if bx:
        bx.close()


# ---- every route ----
GUARD = 64           # rows of guard band either side of the device outputs


def _device_call(B, k, call):
    """search_device on a caller stream into torch tensors pre-filled with a sentinel, a guard band either side.
    Returns the results and whether the guard bands are untouched."""
    import torch
    st = torch.cuda.Stream()
    ids = torch.full(((B + 2 * GUARD) * k,), 0x5a5a5a5a5a5a5a5a, dtype=torch.int64, device="cuda")
    dist = torch.full(((B + 2 * GUARD) * k,), -7.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((B + 2 * GUARD,), 0x5a5a5a5a, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    call(ids.data_ptr() + GUARD * k * 8, dist.data_ptr() + GUARD * k * 4, cnt.data_ptr() + GUARD * 4, st.cuda_stream)
    st.synchronize()
    i, d, c = ids.cpu().numpy().view(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
    inner = lambda a, w: a[GUARD * w:(GUARD + B) * w]
    edge = lambda a, w: np.concatenate([a[:GUARD * w], a[(GUARD + B) * w:]])
    clean = ((edge(i, k) == 0x5a5a5a5a5a5a5a5a).all() and (edge(d, k) == -7.0).all() and (edge(c, 1) == 0x5a5a5a5a).all())
    return (inner(i, k).reshape(B, k), inner(d, k).reshape(B, k), inner(c, 1)), bool(clean)


def _routes(ctx):
    import oracle
    from lancedb_b200 import _native
    from tests import sq_oracle
    from tests.util import queries
    rng, ix = _pq8_index("cosine")
    sx = sq_oracle.random_sq_index(rng, n=100000, dim=32, nlist=4, metric="l2", empty=())
    orc = oracle.OracleIndex.from_data(ix)
    for tag, data, cls, NP, dim, ora in (
            ("pq8_", ix, _native.GpuIvfPq, 8, 64, lambda qq, **kw: orc.search(qq, nthreads=NTH, **kw)),
            ("sq_", sx, _native.GpuIvfSq, 1, 32, lambda qq, **kw: sq_oracle.search(sx, qq, nthreads=NTH, **kw))):
        gpu = _open(ctx, cls, data)
        B, k = 37, 10
        q, q2 = queries(rng, B, dim), queries(rng, B, dim)
        ctx.sub_batch(tag + "shape", gpu, B, NP)
        # thin enough that rows past `count` exist: they must hold id UINT64_MAX and distance +inf
        mask, bm = _mask(rng, data.row_ids, 6.0 / float(np.sort(_sizes(data))[::-1][:NP].sum()))
        oallow = dict(allow=_oracle_bitmap(mask), allow_bits=mask.size) if tag == "pq8_" else dict(allow=mask)
        ctx.run(tag + "host", lambda: gpu.search(q, k=k, nprobes=NP), lambda: ora(q, k=k, nprobes=NP))
        ctx.run(tag + "filtered", lambda: gpu.search(q, k=k, nprobes=NP, allow=bm, allow_bits=mask.size),
                lambda: ora(q, k=k, nprobes=NP, **oallow))
        if ctx.want_oracle or not ctx.gpu:
            oi, od, oc = (ctx.out[f"{tag}filtered/o_{n}"] for n in ("ids", "dist", "cnt"))
            assert (oc < k).any()
            for b in range(B):
                assert (oi[b, oc[b]:] == U64_MAX).all() and np.isposinf(od[b, oc[b]:]).all()
        p = _native.make_params(k=k, nprobes=NP)
        d0 = ora(q[:1], k=50, nprobes=NP)[1][0]
        lo, hi = float(d0[2]), float(d0[8])
        rc = ora(q, k=k, nprobes=NP, lower=lo, upper=hi)[2]
        assert (rc < k).any() and (rc > 0).any(), rc
        if ctx.gpu:
            import torch
            dq = torch.from_numpy(q).cuda()
            clean = []

            def device():
                got, ok = _device_call(B, k, lambda i, d, c, s: gpu.search_device(dq.data_ptr(), B, p, i, d, c, s))
                clean.append(ok)
                return got
            ctx.run(tag + "device", device, lambda: ora(q, k=k, nprobes=NP))
            ctx.put(tag + "device", guard_clean=clean[0])
            # a narrow distance_range: most queries find fewer than k rows, so the rows past `count` of the caller's
            # sentinel-filled device buffers must come back as id UINT64_MAX / +inf
            pr = _native.make_params(k=k, nprobes=NP, lower=lo, upper=hi)

            def device_range():
                got, ok = _device_call(B, k, lambda i, d, c, s: gpu.search_device(dq.data_ptr(), B, pr, i, d, c, s))
                clean.append(ok)
                return got
            ctx.run(tag + "device_range", device_range, lambda: ora(q, k=k, nprobes=NP, lower=lo, upper=hi))
            ctx.put(tag + "device_range", guard_clean=clean[1])
            # two tickets in flight on one handle
            pin = lambda a: torch.from_numpy(a).pin_memory().numpy()
            bufs = [(pin(np.zeros((B, k), np.int64)).view(np.uint64), pin(np.zeros((B, k), np.float32)),
                     pin(np.zeros(B, np.int32)).view(np.uint32)) for _ in range(2)]
            qs = [pin(q), pin(q2)]
            n0 = _native.kernel_launch_count()
            tickets = [gpu.search_async(qs[i], p, *bufs[i]) for i in range(2)]
            for t in tickets:
                _native.ticket_wait(t)
            ctx.put(tag + "async0", launches=_native.kernel_launch_count() - n0)
            ctx.put(tag + "async1", launches=_native.kernel_launch_count() - n0)
            ctx.result(tag + "async0", [b.copy() for b in bufs[0]])
            ctx.result(tag + "async1", [b.copy() for b in bufs[1]])
            gpu.close()
        else:
            ctx.result(tag + "device", ora(q, k=k, nprobes=NP), "o_")
            ctx.result(tag + "device_range", ora(q, k=k, nprobes=NP, lower=lo, upper=hi), "o_")
        if ctx.want_oracle or not ctx.gpu:
            ctx.result(tag + "async0", ora(q, k=k, nprobes=NP), "o_")
            ctx.result(tag + "async1", ora(q2, k=k, nprobes=NP), "o_")


def _graphs(ctx):
    """The same split call three times (eager warm-up, capture, replay), then other queries of the same shape"""
    import oracle
    from lancedb_b200 import _native
    from tests import sq_oracle
    from tests.util import queries
    rng, ix = _pq8_index("l2")
    sx = sq_oracle.random_sq_index(rng, n=100000, dim=32, nlist=4, metric="l2", empty=())
    orc = oracle.OracleIndex.from_data(ix)
    for tag, data, cls, NP, dim, ora in (
            ("pq8_", ix, _native.GpuIvfPq, 8, 64, lambda qq, **kw: orc.search(qq, nthreads=NTH, **kw)),
            ("sq_", sx, _native.GpuIvfSq, 1, 32, lambda qq, **kw: sq_oracle.search(sx, qq, nthreads=NTH, **kw))):
        gpu = _open(ctx, cls, data)
        q, q2 = queries(rng, 37, dim), queries(rng, 37, dim)
        ctx.sub_batch(tag + "shape", gpu, 37, NP)
        for name, qq in (("warmup", q), ("capture", q), ("replay", q), ("replay_other", q2)):
            ctx.run(tag + name, lambda: gpu.search(qq, k=10, nprobes=NP), lambda: ora(qq, k=10, nprobes=NP))
        if gpu:
            gpu.close()


def _timeout(ctx):
    import oracle
    from lancedb_b200 import _native
    from tests.util import queries
    rng, ix = _pq8_index("l2")
    orc = oracle.OracleIndex.from_data(ix)
    gpu = _open(ctx, _native.GpuIvfPq, ix)
    q = queries(rng, 37, 64)
    ora = lambda: orc.search(q, k=10, nprobes=8, nthreads=NTH)
    ctx.sub_batch("shape", gpu, 37, 8)
    ctx.run("generous", lambda: gpu.search(q, k=10, nprobes=8, timeout_ms=600000), ora)
    if ctx.gpu:
        # 4001 queries: hundreds of sub-batches under the small budget, far more than a millisecond of work either way.
        # One attempt: the call must give up, leave the outputs alone, and leave the handle usable.
        big = queries(rng, 4001, 64)
        ids = np.full((4001, 10), 123, np.uint64); dist = np.full((4001, 10), -7.0, np.float32)
        cnt = np.full(4001, 99, np.uint32)
        raised = False
        try:
            gpu.search_into(big, _native.make_params(k=10, nprobes=8, timeout_ms=1), ids, dist, cnt)
        except TimeoutError:
            raised = True
        ctx.put("impossible", raised=raised,
                untouched=bool((ids == 123).all() and (dist == -7.0).all() and (cnt == 99).all()))
    ctx.run("after_timeout", lambda: gpu.search(q, k=10, nprobes=8), ora)
    ctx.run("after_timeout_dense", lambda: gpu.search(q, k=10, nprobes=8), ora, {"LGPU_DENSE_FILTER": 1})
    if gpu:
        gpu.close()


def _profiling(ctx):
    """set_profiling(True) on a split call: the counters, the scanned bytes and the stage times cover the whole call"""
    import oracle
    from lancedb_b200 import _native
    from tests import ivf_binary_oracle as ibo
    from tests.util import queries
    rng, ix = _pq8_index("l2")
    orc = oracle.OracleIndex.from_data(ix)
    gpu = _open(ctx, _native.GpuIvfPq, ix)
    B, NP = 37, 8
    q = queries(rng, B, 64)
    bix = ibo.random_index(rng, 100000, 16, 4)
    bq = rng.integers(0, 256, (B, 16), dtype=np.uint8)
    bgpu = _open(ctx, _native.GpuIvfBinary, bix)

    def profiled(case, call, ora, env=None):
        def run():
            _native.set_profiling(True)
            try:
                got = call()
                st = _native.last_filter_stats()
                ctx.put(case, stats=[st["candidates"], st["rescored"], st["flagged_queries"], st["queries"]],
                        scanned=_native.last_scanned_code_bytes(), total_ms=_native.last_stage_ms()["total"])
            finally:
                _native.set_profiling(False)
            return got
        ctx.run(case, run, ora, env)

    ora = lambda: orc.search(q, k=10, nprobes=NP, nthreads=NTH)
    ctx.sub_batch("shape", gpu, B, NP)
    profiled("candidates", lambda: gpu.search(q, k=10, nprobes=NP), ora)
    profiled("cand_cap32", lambda: gpu.search(q, k=10, nprobes=NP), ora, {"LGPU_CAND_CAP": 32})
    profiled("dense", lambda: gpu.search(q, k=10, nprobes=NP), ora, {"LGPU_DENSE_FILTER": 1})
    # a query holding a NaN has no provable shortlist: the dense mode flags it.  Three of them in three sub-batches
    # (first, second and the tail) add three to the count; a batch of nothing but such queries is flagged whole.
    q3 = q.copy()
    q3[[0, 9, 36], 7] = np.nan
    profiled("dense_3_nan", lambda: gpu.search(q3, k=10, nprobes=NP),
             lambda: orc.search(q3, k=10, nprobes=NP, nthreads=NTH), {"LGPU_DENSE_FILTER": 1})
    qa = q.copy()
    qa[:, 7] = np.nan
    profiled("dense_all_nan", lambda: gpu.search(qa, k=10, nprobes=NP),
             lambda: orc.search(qa, k=10, nprobes=NP, nthreads=NTH), {"LGPU_DENSE_FILTER": 1})
    profiled("exact", lambda: gpu.search(q, k=10, nprobes=NP), ora, {"LGPU_EXACT_SCAN": 1})
    profiled("ivf_binary", lambda: bgpu.search(bq, k=10, nprobes=1), lambda: ibo.search(bix, bq, k=10, nprobes=1, nthreads=NTH))
    # the rows a query's probes hold, summed over the batch: what the scanned-bytes counter must report (m = 16 code
    # bytes a row; 16 bytes a binary row)
    if ctx.want_oracle or not ctx.gpu:
        off = np.asarray(ix.part_offsets, np.int64)
        rows = sum(int((off[p + 1] - off[p]).sum()) for p in (orc.find_partitions(v, NP)[0].astype(np.int64) for v in q))
        ctx.put("candidates", o_scanned=rows * 16)
    for g in (gpu, bgpu):
        if g:
            g.close()


RUN = {"pq8_l2": lambda c: _pq8(c, "l2"), "pq8_cosine": lambda c: _pq8(c, "cosine"), "pq8_dot": lambda c: _pq8(c, "dot"),
       "pq8_small_tail": _pq8_small_tail, "pq8_tc_coarse": _pq8_tc_coarse, "pq4": _pq4, "sq": _sq, "rq": _rq,
       "ivf_binary": _ivf_binary, "flat": _flat, "flat_big": _flat_big, "binary_flat": _binary_flat, "routes": _routes,
       "graphs": _graphs, "timeout": _timeout, "profiling": _profiling}


def main(argv):
    group, path = argv[0], argv[1]
    rehearse = "--rehearse" in argv[2:]
    os.environ.setdefault("LGPU_SMALL_SLOTS", "0")       # the batched kernels, unless a case asks for the default
    ctx = Ctx(gpu=not rehearse, want_oracle=os.environ.get("SUB_BATCH_ORACLE") == "1")
    RUN[group](ctx)
    np.savez(path, **ctx.out)
    print(f"{group}: {len({k.split('/')[0] for k in ctx.out})} cases" + (" (rehearsal, no device)" if rehearse else ""))


if __name__ == "__main__":
    main(sys.argv[1:])

"""The top-k selection every search ends in (csrc/select.cu: the warp kernel for k <= 32, the shared-memory bitonic
kernel above), run alone through lgpu_debug_select, and the public merge lgpu_merge_topk_device, against the exact
restatement in tests/select_oracle.py.  Every case runs once and must match bit for bit: ids, distance bits, counts and
positions, in output buffers filled with a sentinel and framed by guard bands, so untouched queries and stray writes
show.  The inputs are shaped where selection goes wrong: ties at the k-th entry, -0 next to +0, NaNs, infinities and
denormals, both sides of the warp / block switch and of the block kernel's compaction trigger max(512, 2 k), staged
counts built to land on that trigger, unaligned dense rows, every mode-2 layout the library uses, and the filters."""
import numpy as np
import pytest

from lancedb_b200 import _native
from lancedb_b200.distributed import merge_records
from tests import select_oracle as so

pytestmark = pytest.mark.gpu

GUARD = 256             # sentinel bytes on each side of every output buffer
FILL = 0xA5
INPUTS = ("dist", "seg_off", "probes", "part_n", "part_off", "row_ids", "dense", "col_ids", "cand_ids", "cand_pos",
          "ncols_q", "cand_rec", "only", "gate", "allow")
SCALARS = ("mode", "nprobes", "nlist", "ncols", "row_stride", "inner", "outer_stride", "B", "k", "has_lower",
           "has_upper", "lower", "upper", "allow_bits", "dist_len")
KS = [1, 2, 31, 32, 33, 64, 127, 128, 129, 255, 256, 432, 511, 512, 513, 1024, 2047, 2048]


def _upload(arr, shift=0):
    """a device copy of arr's bytes, `shift` bytes into a fresh allocation: (tensor, address)"""
    import torch
    b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    t = torch.zeros(b.size + shift + 16, dtype=torch.uint8, device="cuda")
    t[shift:shift + b.size].copy_(torch.from_numpy(b.copy()))
    return t, t.data_ptr() + shift


def _guarded(nbytes):
    import torch
    return torch.full((nbytes + 2 * GUARD,), FILL, dtype=torch.uint8, device="cuda")


def _compare(what, name, got, exp):
    g = np.ascontiguousarray(got).view(np.uint8).reshape(exp.shape[0], -1)
    e = np.ascontiguousarray(exp).view(np.uint8).reshape(exp.shape[0], -1)
    bad = np.nonzero((g != e).any(axis=1))[0]
    if bad.size:
        q = int(bad[0])
        col = int(np.nonzero(g[q] != e[q])[0][0]) // max(1, exp.dtype.itemsize)
        raise AssertionError(f"{what}: {name} differs in {bad.size} queries, first q={q} at entry {col}: "
                             f"got {got[q][col:col + 4] if got.ndim > 1 else got[q]}, "
                             f"want {exp[q][col:col + 4] if exp.ndim > 1 else exp[q]}")


def run(a, what, pos=False, rec=False, dense_shift=0, refused=None):
    """lgpu_debug_select on device copies of case `a` (the dense block `dense_shift` floats past a 16-byte boundary),
    then every output byte, guard bands included, against the reference"""
    import torch
    keep, args = [], {n: (float if n in ("lower", "upper") else int)(a[n]) for n in SCALARS if a.get(n) is not None}
    for n in INPUTS:
        if a.get(n) is not None:
            t, args[n] = _upload(a[n], 4 * dense_shift if n == "dense" else 0)
            keep.append(t)
    B, k = a["B"], a["k"]
    exp = so.outputs(B, k, pos, rec, FILL)
    bufs = {}
    for n, arr in exp.items():
        bufs[n] = _guarded(arr.nbytes)
        args["out_" + n] = bufs[n].data_ptr() + GUARD
    launches = _native.kernel_launch_count()
    if refused:
        with pytest.raises(ValueError, match=refused):
            _native.debug_select(**args)
    else:
        _native.debug_select(**args)
        so.select(a, exp)
    torch.cuda.synchronize()
    assert _native.kernel_launch_count() - launches == (0 if refused or B == 0 else 1), what
    for n, t in bufs.items():
        got = t.cpu().numpy()
        assert np.all(got[:GUARD] == FILL) and np.all(got[-GUARD:] == FILL), f"{what}: write outside {n}"
        _compare(what, n, got[GUARD:-GUARD].view(exp[n].dtype).reshape(exp[n].shape), exp[n])


ORDERS = ["asc", "desc", "equal", "equal_permuted", "two", "mixed"]


def _rows(order, n, B, rng):
    base = "equal" if order == "equal_permuted" else order
    return [so.values(base, n, rng, shift=0.25 * q) for q in range(B)]


@pytest.mark.parametrize("layout", ["dense", "cands"])
@pytest.mark.parametrize("k", KS)
def test_every_k_regime_and_candidate_count(k, layout):
    """0, 1, 3, k - 1, k, k + 1, 1023, 1024, 1025 and 100003 candidates per query in every order: ascending,
    descending (every candidate passes, the block kernel compacts on every iteration), all equal (ids decide, also
    with non-monotone ids), two values, and a mix of signs, +-0, +-inf, denormals and NaNs; B = 1, 3 and 37"""
    rng = np.random.default_rng(k * 7 + (layout == "cands"))
    counts = sorted({0, 1, 3, k - 1, k, k + 1, 1023, 1024, 1025, 100003} - {-1})
    i = 0
    for n in counts:
        for order in ORDERS:
            B = 3 if n > 2000 else (1, 3, 37)[i % 3]
            rows = _rows(order, n, B, rng)
            if layout == "dense":
                ids = None if order in ("asc", "desc", "two", "equal") else \
                    (rng.permutation(n).astype(np.uint64) * 3 + 1 if order == "equal_permuted" else
                     so.unique_ids(rng, n))
                a = so.dense_case(np.stack(rows) if n else np.zeros((B, 0), np.float32), k, col_ids=ids)
            else:
                a = so.cands_case(rows, [so.unique_ids(rng, n) for _ in range(B)], k)
            run(a, f"{layout} k={k} n={n} {order} B={B}", pos=i % 2 == 0, rec=i % 3 == 1)
            i += 1


def trigger_rows(k, B, rng):
    """Per query, candidate values laid out 1024 per iteration of the block kernel (the candidates one iteration
    stages) so that its staged count at the end of consecutive iterations is exactly trigger - 1, trigger and
    trigger + 1, in a different order per query.  Each iteration's passing values lie below everything before them, so
    they all pass; the others are NaN, +inf, 1e30 or the next float above the current k-th best, which all fail.
    Returns the rows and, per query, the staged count at the end of every iteration."""
    T = max(512, 2 * k)
    pattern = [T - 1, T, T + 1, T, T - 1, T + 1, T + 1, T - 1, T, T + 1]
    rows, hits = [], []
    for q in range(B):
        chunks, staged, tau, low, hit = [], 0, None, 0, []

        def chunk(p):
            nonlocal low
            good = (low - 1 - np.arange(p)).astype(np.float32)          # strictly below every earlier value
            low -= p
            if tau is None:                                             # no threshold yet: only NaN fails
                fill = np.full(1024 - p, np.nan, np.float32)
            else:
                above = np.nextafter(np.float32(tau), np.float32(np.inf))
                fill = rng.choice(np.array([np.nan, np.inf, 1e30, above], np.float32), 1024 - p)
            c = np.concatenate([good, fill])
            rng.shuffle(c)
            chunks.append(c)

        for t in pattern[q:] + pattern[:q]:
            while t - staged > 1024:                                    # climb without reaching the trigger
                p = min(1024, T - 1 - staged)
                chunk(p)
                staged += p
                hit.append(staged)
            chunk(t - staged)
            staged = t
            hit.append(t)
            if staged >= T:                                             # compaction: keep the k smallest
                staged, tau = k, low + k - 1
        tail = (low - 1 - np.arange(37)).astype(np.float32)             # a last, partial iteration
        rows.append(np.concatenate(chunks + [tail]))
        hits.append(hit)
    n = max(len(r) for r in rows)
    return [np.concatenate([r, np.full(n - len(r), np.nan, np.float32)]) for r in rows], hits


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("k", [33, 64, 255, 256, 432, 511, 512, 513, 1024, 2047, 2048])
def test_block_kernel_staged_count_on_its_trigger(k, mode):
    rng = np.random.default_rng(k + 10 * mode)
    B = 3
    rows, hits = trigger_rows(k, B, rng)
    T = max(512, 2 * k)
    for h in hits:
        assert all(h.count(t) >= 3 for t in (T - 1, T, T + 1))
        if k < 1024:                # above, one iteration cannot refill from k to T + 1
            assert any(h[i:i + 3] == [T - 1, T, T + 1] for i in range(len(h) - 2))
    n = len(rows[0])
    if mode == 0:
        a = so.segments_case(rows, np.arange(B, dtype=np.uint64)[:, None], k,
                             row_ids=rng.permutation(B * n).astype(np.uint64))
    elif mode == 1:
        a = so.dense_case(np.stack(rows), k)
    else:
        a = so.cands_case(rows, [so.unique_ids(rng, n) for _ in range(B)], k)
    for pos in (False, True):
        run(a, f"trigger mode {mode} k={k} pos={pos}", pos=pos)


@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 128, 432, 1024, 2048])
def test_ivf_segments(k):
    """mode 0: partitions of 0 .. 3001 rows, empty ones probed, unused probe slots, shuffled row ids, positions; the
    padding of every segment holds -inf, which must not be read"""
    rng = np.random.default_rng(300 + k)
    sizes = [0, 1, 3, 4, 5, 255, 256, 257, 1023, 1024, 1025, 3001, 0]
    B, nprobes = 5, 6
    for order in ("mixed", "equal", "desc"):
        parts = [so.values(order, n, rng, shift=p) for p, n in enumerate(sizes)]
        row_ids = rng.permutation(sum(sizes)).astype(np.uint64) * 5 + 3
        probes = np.stack([rng.permutation(len(sizes))[:nprobes] for _ in range(B)]).astype(np.uint64)
        probes[rng.random(probes.shape) < 0.2] = so.U64_MAX
        probes[1, 2] = len(sizes)                                       # >= nlist: unused too
        probes[4] = [0, 12, 0, so.U64_MAX, 1, 12]                       # empty partitions, one row
        for pos in (False, True):
            a = so.segments_case(parts, probes, k, row_ids=None if order == "desc" else row_ids,
                                 gap=4 * int(rng.integers(0, 3)))
            run(a, f"segments k={k} {order} pos={pos}", pos=pos, rec=order == "equal")


@pytest.mark.parametrize("k", [5, 32, 33, 500])
def test_dense_rows_aligned_and_not(k):
    """mode 1 with the block 16-byte aligned or one float past it, and row strides that are or are not a multiple of
    4; the columns between ncols and the stride hold -inf, which must not be read"""
    rng = np.random.default_rng(400 + k)
    for n in (255, 256, 1000, 1025, 5000):
        for stride, shift in ((n + (-n) % 4, 0), (n + 1, 0), (n + (-n) % 4, 1), (n + 3, 1)):
            V = np.stack([so.values("mixed", n, rng) for _ in range(3)])
            ids = so.unique_ids(rng, n) if stride % 2 else None
            run(so.dense_case(V, k, col_ids=ids, stride=stride), f"dense k={k} n={n} stride={stride} shift={shift}",
                pos=shift == 1, dense_shift=shift)


@pytest.mark.parametrize("k", [1, 7, 32, 33, 100, 600])
def test_strided_lists(k):
    """mode 2 in the three layouts the library uses: select_cands (lists of different lengths, unused slots), the
    same cut by ncols_q with positions from cand_pos (the filter scan's re-score), and the merge layout (inner = k,
    outer stride B k) with ids + values and with packed records; each into ids + values and into records"""
    rng = np.random.default_rng(500 + k)
    B = 6
    lens = rng.integers(0, 3 * k + 40, B)
    lens[0], lens[1], lens[3] = 0, k, 3 * k + 39
    vals = [so.values("mixed", int(m), rng) for m in lens]
    ids = [so.unique_ids(rng, int(m)) for m in lens]
    pos = [rng.integers(0, 1 << 40, int(m)).astype(np.uint64) for m in lens]
    for cut in (False, True):
        for p in (None, pos):
            a = so.cands_case(vals, ids, k, pos=p, ncols_q=cut)
            if cut:
                a["ncols_q"][3] += 5                                    # above ncols: the kernels clamp it
            for rec in (False, True):
                run(a, f"cands k={k} ncols_q={cut} cand_pos={p is not None} rec={rec}", pos=True, rec=rec)
    L = 3
    counts = rng.integers(0, k + 1, (L, B))
    counts[:, 0], counts[:, 1] = k, 0
    lids, ldist = so.search_lists(rng, L, B, k, counts, so.values("two", 64, rng))
    for rec_in in (False, True):
        for rec in (False, True):
            run(so.merge_case(lids, ldist, k, rec=rec_in), f"merge layout k={k} rec_in={rec_in} rec={rec}",
                pos=rec_in, rec=rec)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("k", [7, 32, 33, 300])
def test_filters(k, mode):
    """distance range at its edges (lower == upper, bounds on present values, infinite bounds), allow bitmaps shorter
    than the largest id, `only` with flagged and unflagged queries, and the gate"""
    rng = np.random.default_rng(600 + 10 * k + mode)
    B, n = 6, 1500
    rows = [so.values("mixed", n, rng) for _ in range(B)]
    if mode == 0:
        a = so.segments_case(rows, np.arange(B, dtype=np.uint64)[:, None], k,
                             row_ids=rng.permutation(B * n).astype(np.uint64))
        top = B * n
    elif mode == 1:
        a = so.dense_case(np.stack(rows), k, col_ids=rng.permutation(n).astype(np.uint64))
        top = n
    else:
        a = so.cands_case(rows, [rng.permutation(B * n)[:n].astype(np.uint64) for _ in range(B)], k)
        top = B * n
    finite = np.sort(np.concatenate(rows)[np.isfinite(np.concatenate(rows))])
    v1, v2 = float(finite[len(finite) // 3]), float(finite[len(finite) // 2])
    bitmap = rng.integers(0, 1 << 32, (top + 31) // 32, dtype=np.uint64).astype(np.uint32)
    only = np.array([1, 0, 1, 1, 0, 0], np.uint32)
    variants = [
        dict(has_lower=1, lower=v1, has_upper=1, upper=v1),
        dict(has_lower=1, lower=v1, has_upper=1, upper=v2),
        dict(has_lower=1, lower=-np.inf, has_upper=1, upper=np.inf),
        dict(has_lower=1, lower=np.inf),
        dict(has_upper=1, upper=-np.inf),
        dict(has_upper=1, upper=0.0),
        dict(has_lower=1, lower=0.0),
        dict(allow=bitmap, allow_bits=int(top * 0.6)),
        dict(allow=bitmap, allow_bits=0),
        dict(only=only),
        dict(only=only, gate=np.array([1], np.uint32)),
        dict(gate=np.array([0], np.uint32)),
        dict(has_lower=1, lower=v1, has_upper=1, upper=np.inf, allow=bitmap, allow_bits=top - 7, only=only,
             gate=np.array([2], np.uint32)),
    ]
    for i, v in enumerate(variants):
        run({**a, **v}, f"filters mode {mode} k={k} variant {i}", pos=i % 2 == 1, rec=i % 3 == 2)


@pytest.mark.parametrize("k", [1, 10, 32, 33, 100, 2048])
@pytest.mark.parametrize("L", [1, 2, 3, 8])
def test_merge_topk_device(L, k):
    """lgpu_merge_topk_device on one GPU: L top-k lists per query as searches emit them (valid prefixes of different
    lengths, padded), ties across the lists, one NaN and one -0, merged on a non-default stream; the result equals the
    reference's and distributed.merge_records'"""
    import torch
    rng = np.random.default_rng(L * 10000 + k)
    B = 5
    counts = rng.integers(0, k + 1, (L, B))
    counts[:, 0], counts[:, 1], counts[0, 2] = k, 0, k
    ids, dist = so.search_lists(rng, L, B, k, counts, np.array([-1.0, -0.0, 0.0, 0.5, 0.5, 2.0, 7.0], np.float32))
    dist[0, 2, 0], dist[L - 1, 0, k - 1] = np.nan, -0.0
    exp = so.select(so.merge_case(ids, dist, k), so.outputs(B, k))
    m_ids, m_dist, m_cnt = merge_records(so.merge_case(ids, dist, k, rec=True)["cand_rec"].reshape(L, B, k), k)
    assert np.array_equal(m_ids, exp["ids"]) and np.array_equal(m_cnt, exp["count"])
    assert np.array_equal(m_dist.view(np.uint32), exp["dist"].view(np.uint32))

    d_ids = torch.zeros(L * B * k, dtype=torch.int64, device="cuda")
    d_dist = torch.zeros(L * B * k, dtype=torch.float32, device="cuda")
    h_ids = torch.from_numpy(ids.reshape(-1).view(np.int64).copy()).pin_memory()
    h_dist = torch.from_numpy(dist.reshape(-1).copy()).pin_memory()
    outs = {n: _guarded(arr.nbytes) for n, arr in so.outputs(B, k).items()}
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        # hold the stream back, then write the inputs on it: a merge launched on another stream would read zeros
        torch.cuda._sleep(20_000_000)
        d_ids.copy_(h_ids, non_blocking=True)
        d_dist.copy_(h_dist, non_blocking=True)
        _native.merge_topk_device(0, L, B, k, d_ids.data_ptr(), d_dist.data_ptr(), outs["ids"].data_ptr() + GUARD,
                                  outs["dist"].data_ptr() + GUARD, outs["count"].data_ptr() + GUARD, s.cuda_stream)
    s.synchronize()
    for n, t in outs.items():
        got = t.cpu().numpy()
        assert np.all(got[:GUARD] == FILL) and np.all(got[-GUARD:] == FILL), f"write outside {n}"
        _compare(f"merge L={L} k={k}", n, got[GUARD:-GUARD].view(exp[n].dtype).reshape(exp[n].shape), exp[n])


def test_debug_select_checks_the_probed_segments():
    """mode 0: a segment off a multiple of 4 floats, or one whose padding to 4 runs past dist_len, is refused and
    nothing is written; the same segment inside dist_len is served"""
    a = so.segments_case([np.arange(10, dtype=np.float32)[::-1].copy()], np.array([[0], [1]], np.uint64), 4)
    a["dist"] = np.concatenate([np.full(4, -np.inf, np.float32), a["dist"]])
    for seg, dist_len, refused in ((2, 64, "multiple of 4"), (4, 15, "runs past dist_len"),
                                   (8, 16, "runs past dist_len"), (4, 16, None)):
        b = dict(a, seg_off=np.array([seg, 0], np.uint64), dist_len=dist_len)
        run(b, f"seg_off={seg} dist_len={dist_len}", refused=refused)

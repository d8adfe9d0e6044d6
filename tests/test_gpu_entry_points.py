"""The search entry points of every column kind (IVF_PQ, IVF_SQ, flat under each metric, binary, binary IVF_FLAT,
multivector) on each route (host buffers, host buffers with a prefilter, device pointers) behave alike: B = 0 is a
no-op, a closed handle, a live handle of another kind, a null output buffer and a null bitmap are refused, the routes
return the same bits, and repeated host calls (eager, CUDA-graph capture, replay) return the same bits with the same
launch count."""
import ctypes as C

import numpy as np
import pytest

from lancedb_b200 import _native
from tests import ivf_binary_oracle
from tests.multivec_oracle import offsets_of
from tests.sq_oracle import random_sq_index
from tests.util import queries, random_index

pytestmark = pytest.mark.gpu

K = 5
KINDS = ["ivf_pq", "ivf_sq", "flat_l2", "flat_cosine", "flat_dot", "binary", "ivf_binary", "multivec"]
ROUTES = ["host", "filtered", "device"]
SYMBOL = {"ivf": "lgpu_search", "flat": "lgpu_flat_search", "binary": "lgpu_binary_search",
          "ivf_binary": "lgpu_ivf_binary_search", "multivec": "lgpu_multivec_search"}
# the handle kind of each family, as the library's messages name it, and its close function
NAME = {"ivf": "index", "flat": "flat", "binary": "binary", "ivf_binary": "binary IVF index", "multivec": "multivector"}
CLOSE = {"ivf": "lgpu_index_close", "flat": "lgpu_flat_close", "binary": "lgpu_binary_close",
         "ivf_binary": "lgpu_ivf_binary_close", "multivec": "lgpu_multivec_close", "comm": "lgpu_comm_destroy"}


class Case:
    """One column kind: its handle, a batch of queries and the raw C call of each route."""

    def __init__(self, kind, B=6):
        rng = np.random.default_rng(7)
        self.kind, self.family = kind, kind if kind == "ivf_binary" else kind.split("_")[0]
        self.metric = _native.METRICS[kind.split("_")[1]] if self.family == "flat" else None
        self.off = None
        if kind == "ivf_pq":
            self.obj, self.q = _native.GpuIvfPq(random_index(rng, dim=32, nlist=8, m=8, n=3000)), queries(rng, B, 32)
        elif kind == "ivf_sq":
            self.obj, self.q = _native.GpuIvfSq(random_sq_index(rng, n=3000, dim=24, nlist=8)), queries(rng, B, 24)
        elif self.family == "flat":
            self.obj, self.q = _native.GpuFlat(queries(rng, 5000, 32)), queries(rng, B, 32)
        elif kind == "binary":
            self.obj = _native.GpuBinary(rng.integers(0, 256, (5000, 16), dtype=np.uint8))
            self.q = rng.integers(0, 256, (B, 16), dtype=np.uint8)
        elif kind == "ivf_binary":
            self.obj = _native.GpuIvfBinary(ivf_binary_oracle.random_index(rng, 3000, 16, 8))
            self.q = rng.integers(0, 256, (B, 16), dtype=np.uint8)
        else:
            lens = rng.integers(0, 5, 2000)
            off = offsets_of(lens)
            self.obj = _native.GpuMultivec(rng.standard_normal((int(off[-1]), 16)).astype(np.float32), off)
            self.off = offsets_of(rng.integers(1, 4, B)).astype(np.uint32)
            self.q = rng.standard_normal((int(self.off[-1]), 16)).astype(np.float32)
        self.B = B
        self.nrows = 5000 if self.family in ("flat", "binary") else (2000 if self.family == "multivec" else 3000)
        self.params = _native.make_params(k=K, nprobes=4)

    def first(self, B):
        """the same handle with the first B queries"""
        c = object.__new__(Case)
        c.__dict__.update(self.__dict__)
        c.B = B
        if self.off is not None:
            c.off, c.q = self.off[: B + 1], self.q[: self.off[B]]
        else:
            c.q = self.q[:B]
        return c

    def call(self, route, h, q, B, outs, allow=None, allow_bits=0, stream=None):
        """the raw C call: q and outs are addresses (host or device), returns the status"""
        head = (h,) + ((self.metric,) if self.family == "flat" else ()) + (q,)
        head += ((self.off.ctypes.data if self.off is not None else None), B) if self.family == "multivec" else (B,)
        name = SYMBOL[self.family] + {"host": "", "filtered": "_filtered", "device": "_device"}[route]
        args = head + (C.byref(self.params),)
        args += (allow, allow_bits) if route == "filtered" else ()
        args += tuple(outs) + ((stream,) if route == "device" else ())
        return getattr(_native.load(), name)(*args)

    def bitmap(self):
        return np.full((self.nrows + 31) // 32, 0x5555_5555, np.uint32)

    def host(self, route="host"):
        """the route's results as host arrays (ids, dist bits, count)"""
        ids, dist, cnt = np.full((self.B, K), 7, np.uint64), np.full((self.B, K), 7, np.float32), np.full(self.B, 7, np.uint32)
        outs = (ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
        if route == "device":
            import torch
            dq = torch.from_numpy(self.q).cuda()
            di = torch.empty(self.B, K, dtype=torch.int64, device="cuda")
            dd = torch.empty(self.B, K, dtype=torch.float32, device="cuda")
            dc = torch.empty(self.B, dtype=torch.int32, device="cuda")
            _native.check(self.call("device", self.obj._h, dq.data_ptr(), self.B, (di.data_ptr(), dd.data_ptr(),
                                                                                   dc.data_ptr()),
                                    stream=torch.cuda.current_stream().cuda_stream))
            torch.cuda.synchronize()
            return di.cpu().numpy().view(np.uint64), dd.cpu().numpy().view(np.uint32), dc.cpu().numpy().view(np.uint32)
        bm = self.bitmap() if route == "filtered" else None
        _native.check(self.call(route, self.obj._h, self.q.ctypes.data, self.B, outs,
                                None if bm is None else bm.ctypes.data, self.nrows if bm is not None else 0))
        return ids, dist.view(np.uint32), cnt


@pytest.fixture(scope="module", params=KINDS)
def case(request):
    c = Case(request.param)
    yield c
    c.obj.close()


def _equal(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("route", ROUTES)
def test_empty_batch_is_ok_and_leaves_the_outputs(case, route):
    if route == "device":
        import torch
        outs = [torch.full((K,), 3, dtype=t, device="cuda") for t in (torch.int64, torch.float32, torch.int32)]
        rc = case.call(route, case.obj._h, outs[1].data_ptr(), 0, [o.data_ptr() for o in outs],
                       stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc == _native.LGPU_OK
        assert all(bool((o == 3).all()) for o in outs)
    else:
        outs = [np.full(K, 3, t) for t in (np.uint64, np.float32, np.uint32)]
        bm = case.bitmap()
        rc = case.call(route, case.obj._h, case.q.ctypes.data, 0, [o.ctypes.data for o in outs], bm.ctypes.data, 32)
        assert rc == _native.LGPU_OK
        assert all((o == 3).all() for o in outs)


@pytest.mark.parametrize("route", ROUTES)
def test_null_output_buffer_and_null_bitmap_are_refused(case, route):
    q = case.q.ctypes.data
    ids, dist = np.zeros((case.B, K), np.uint64), np.zeros((case.B, K), np.float32)
    rc = case.call(route, case.obj._h, q, case.B, (ids.ctypes.data, dist.ctypes.data, None), case.bitmap().ctypes.data,
                   32)
    assert rc == _native.LGPU_INVALID_INPUT and _native.load().lgpu_last_error() == b"null buffer"
    if route == "filtered":
        cnt = np.zeros(case.B, np.uint32)
        rc = case.call(route, case.obj._h, q, case.B, (ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data), None, 32)
        assert rc == _native.LGPU_INVALID_INPUT and _native.load().lgpu_last_error() == b"allow bitmap is null"


def test_routes_return_the_same_bits(case):
    host = case.host("host")
    assert _equal(host, case.host("device"))
    assert case.host("filtered")[2].sum() > 0
    if case.family == "ivf":
        import torch
        ids = torch.empty(case.B, K, dtype=torch.int64).pin_memory().numpy().view(np.uint64)
        dist = torch.empty(case.B, K, dtype=torch.float32).pin_memory().numpy()
        cnt = torch.empty(case.B, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        _native.ticket_wait(case.obj.search_async(case.q, case.params, ids, dist, cnt))
        assert _equal(host, (ids, dist.view(np.uint32), cnt))


def test_repeated_host_calls_return_the_same_bits_and_launches(case):
    """eager (new key), capture, replay: the same results and the same kernel launches per call"""
    case.first(case.B - 1).host("host")   # another shape first: one-time work (norms, allocations) happens here
    runs, launches = [], []
    for _ in range(3):
        n0 = _native.kernel_launch_count()
        runs.append(case.host("host"))
        launches.append(_native.kernel_launch_count() - n0)
    print(f"{case.kind}: kernel launches per host call {launches}")
    assert _equal(runs[0], runs[1]) and _equal(runs[0], runs[2])
    assert launches[0] > 0 and launches[0] == launches[2]


@pytest.mark.parametrize("route", ROUTES)
def test_closed_handle_is_refused(route):
    for k in (Case(kind, B=2) for kind in ("ivf_pq", "flat_l2", "binary", "ivf_binary", "multivec")):
        h = C.c_void_p(k.obj._h.value)
        k.obj.close()
        outs = [np.zeros(2 * K, np.uint64), np.zeros(2 * K, np.float32), np.zeros(2, np.uint32)]
        rc = k.call(route, h, k.q.ctypes.data, 2, [o.ctypes.data for o in outs], k.bitmap().ctypes.data, 32)
        assert rc == _native.LGPU_INVALID_INPUT
        assert b"closed" in _native.load().lgpu_last_error()


def test_a_live_handle_of_another_kind_is_refused():
    """Every live handle, passed to every other kind's search on every route, to the index-only entry points and as a
    communicator, is refused on the host before it is read; a close of another kind leaves it open and unchanged."""
    lib = _native.load()
    cases = [Case(kind) for kind in KINDS]
    before = [c.host("host") for c in cases]
    ids, dist, cnt = np.zeros(64, np.uint64), np.zeros(64, np.float32), np.zeros(8, np.uint32)
    outs = (ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data)

    def refused(rc, want, got):
        assert rc == _native.LGPU_INVALID_INPUT
        article = "an" if got == "index" else "a"
        assert lib.lgpu_last_error().decode() == f"{want} handle expected, got {article} {got} handle"

    for h in cases:
        got = NAME[h.family]
        for c in cases:
            if c.family == h.family:
                continue
            for route in ROUTES:
                bm = c.bitmap()
                refused(c.call(route, h.obj._h, c.q.ctypes.data, c.B, outs, bm.ctypes.data, 32), NAME[c.family], got)
        if h.family != "ivf":
            refused(lib.lgpu_index_device_bytes(h.obj._h, C.byref(C.c_uint64())), "index", got)
        t = (C.c_float * 3)()
        refused(lib.lgpu_comm_last_stage_ms(h.obj._h, t), "communicator", got)
    ix, q = cases[KINDS.index("ivf_pq")], cases[KINDS.index("ivf_pq")].q
    p = C.byref(ix.params)
    refused(lib.lgpu_search_sharded(ix.obj._h, ix.obj._h, q.ctypes.data, 1, p, *outs), "communicator", "index")
    refused(lib.lgpu_search_sharded_device(ix.obj._h, ix.obj._h, q.ctypes.data, 1, p, *outs, None), "communicator",
            "index")
    ivb = cases[KINDS.index("ivf_binary")].obj._h
    refused(lib.lgpu_search_sharded_device(ivb, ix.obj._h, q.ctypes.data, 1, p, *outs, None), "index",
            "binary IVF index")
    parts, L = np.zeros(64, np.uint32), np.zeros(64 * 64, np.float32)
    refused(lib.lgpu_debug_filter_bounds(ivb, q.ctypes.data, 1, 4, 64, parts.ctypes.data, L.ctypes.data,
                                         dist.ctypes.data, dist.ctypes.data, cnt.ctypes.data), "index", "binary IVF index")
    refused(lib.lgpu_debug_partition_distances(ivb, q.ctypes.data, 0, L.ctypes.data), "index", "binary IVF index")

    for h in cases:
        for family, close in CLOSE.items():
            if family != h.family:
                getattr(lib, close)(h.obj._h)
    try:
        for c, b in zip(cases, before):
            assert _equal(c.host("host"), b), c.kind
    finally:
        for c in cases:
            c.obj.close()

"""Every search, close and ticket entry point of the C ABI against a null or stale handle, without a GPU: the call
is refused with LGPU_INVALID_INPUT and a message naming the handle's kind, before anything touches a device.  Also
the documented order of the checks made before the handle is resolved."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lancedb_b200 import _native

STALE = C.c_void_p(0x1000)          # never returned by an open: not a live handle
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    return _native.load()


def _searches(h, comm):
    """(kind, symbol, arguments) of every search entry point, B = 1 with real buffers"""
    p = _native.make_params(k=4, nprobes=2)
    q = np.zeros(8, np.float32)
    off = np.array([0, 1], np.uint32)
    bm = np.zeros(1, np.uint32)
    ids, dist, cnt = np.zeros(4, np.uint64), np.zeros(4, np.float32), np.zeros(1, np.uint32)
    out = (ids.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
    pp, qp = C.byref(p), q.ctypes.data
    return [
        ("index", "lgpu_search", (h, qp, 1, pp) + out),
        ("index", "lgpu_search_filtered", (h, qp, 1, pp, bm.ctypes.data, 32) + out),
        ("index", "lgpu_search_device", (h, qp, 1, pp) + out + (None,)),
        ("index", "lgpu_search_sharded", (h, comm, qp, 1, pp) + out),
        ("index", "lgpu_search_sharded_device", (h, comm, qp, 1, pp) + out + (None,)),
        ("index", "lgpu_search_async", (h, qp, 1, pp) + out + (C.byref(C.c_void_p()),)),
        ("flat", "lgpu_flat_search", (h, 0, qp, 1, pp) + out),
        ("flat", "lgpu_flat_search_filtered", (h, 0, qp, 1, pp, bm.ctypes.data, 32) + out),
        ("flat", "lgpu_flat_search_device", (h, 0, qp, 1, pp) + out + (None,)),
        ("binary", "lgpu_binary_search", (h, qp, 1, pp) + out),
        ("binary", "lgpu_binary_search_filtered", (h, qp, 1, pp, bm.ctypes.data, 32) + out),
        ("binary", "lgpu_binary_search_device", (h, qp, 1, pp) + out + (None,)),
        ("binary IVF index", "lgpu_ivf_binary_search", (h, qp, 1, pp) + out),
        ("binary IVF index", "lgpu_ivf_binary_search_filtered", (h, qp, 1, pp, bm.ctypes.data, 32) + out),
        ("binary IVF index", "lgpu_ivf_binary_search_device", (h, qp, 1, pp) + out + (None,)),
        ("multivector", "lgpu_multivec_search", (h, qp, off.ctypes.data, 1, pp) + out),
        ("multivector", "lgpu_multivec_search_filtered", (h, qp, off.ctypes.data, 1, pp, bm.ctypes.data, 32) + out),
        ("multivector", "lgpu_multivec_search_device", (h, qp, off.ctypes.data, 1, pp) + out + (None,)),
    ], (ids, dist, cnt, q, off, bm, p)


def _refused(rc, kind):
    assert rc == _native.LGPU_INVALID_INPUT
    msg = _lib().lgpu_last_error().decode()
    assert msg.startswith(f"{kind} handle is null, closed"), msg


@pytest.mark.parametrize("handle", [None, STALE], ids=["null", "stale"])
def test_every_search_entry_point_refuses_a_dead_handle(handle):
    lib = _lib()
    calls, keep = _searches(handle, STALE)
    assert len(calls) == 18
    for kind, name, args in calls:
        _refused(getattr(lib, name)(*args), kind)


@pytest.mark.parametrize("handle", [None, STALE], ids=["null", "stale"])
def test_the_handle_is_checked_before_the_arguments(handle):
    """null params, B = 0 and null buffers: still the handle's error"""
    lib = _lib()
    _refused(lib.lgpu_search(handle, None, 0, None, None, None, None), "index")
    _refused(lib.lgpu_search_filtered(handle, None, 3, None, None, 64, None, None, None), "index")
    _refused(lib.lgpu_flat_search(handle, 99, None, 0, None, None, None, None), "flat")
    _refused(lib.lgpu_binary_search_device(handle, None, 0, None, None, None, None, None), "binary")
    _refused(lib.lgpu_multivec_search(handle, None, None, 2, None, None, None, None), "multivector")


def test_coalesced_search_refuses_a_dead_handle():
    """in a process of its own: the first lgpu_search_coalesced call fixes the batching window for the process"""
    code = ("import ctypes as C, numpy as np; from lancedb_b200 import _native as n; lib = n.load(); "
            "q, i, d, c = np.zeros(8, np.float32), np.zeros(4, np.uint64), np.zeros(4, np.float32), np.zeros(1, np.uint32); "
            "p = n.make_params(k=4); "
            "rc = [lib.lgpu_search_coalesced(h, q.ctypes.data, C.byref(p), i.ctypes.data, d.ctypes.data, c.ctypes.data) "
            "for h in (None, C.c_void_p(0x1000))]; "
            "print(rc, lib.lgpu_last_error().decode())")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == f"[{_native.LGPU_INVALID_INPUT}, {_native.LGPU_INVALID_INPUT}] index handle is null, " \
        "closed, or was opened in another process (fork)"


def test_other_handle_entry_points_name_their_kind():
    lib = _lib()
    b, t = C.c_uint64(), (C.c_float * 3)()
    _refused(lib.lgpu_index_device_bytes(STALE, C.byref(b)), "index")
    _refused(lib.lgpu_comm_last_stage_ms(STALE, t), "communicator")
    _refused(lib.lgpu_comm_last_stage_ms(None, t), "communicator")


def test_close_accepts_null_and_stale_handles():
    lib = _lib()
    for name in ("lgpu_index_close", "lgpu_flat_close", "lgpu_binary_close", "lgpu_multivec_close",
                 "lgpu_ivf_binary_close", "lgpu_comm_destroy"):
        getattr(lib, name)(None)
        getattr(lib, name)(STALE)


def test_ticket_entry_points_refuse_a_null_ticket():
    lib = _lib()
    assert lib.lgpu_ticket_wait(None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"ticket is null"
    d = C.c_int()
    assert lib.lgpu_ticket_poll(None, C.byref(d)) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"null argument"


def test_async_checks_the_ticket_then_the_params_then_the_handle():
    lib = _lib()
    p = _native.make_params(k=4)
    t = C.c_void_p()
    assert lib.lgpu_search_async(None, None, 1, None, None, None, None, None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"ticket is null"
    assert lib.lgpu_search_async(None, None, 1, None, None, None, None, C.byref(t)) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"search params are null"
    _refused(lib.lgpu_search_async(None, None, 1, C.byref(p), None, None, None, C.byref(t)), "index")
    assert not t.value


def test_merge_topk_checks_its_shape_before_its_buffers_and_device():
    lib = _lib()
    for nlists, k in ((0, 4), (2, 0), (2, 4097)):
        assert lib.lgpu_merge_topk_device(-1, nlists, 1, k, None, None, None, None, None, None) == \
            _native.LGPU_INVALID_INPUT
        assert lib.lgpu_last_error() == b"bad merge shape"
    assert lib.lgpu_merge_topk_device(-1, 2, 1, 4, None, None, None, None, None, None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_last_error() == b"null buffer"

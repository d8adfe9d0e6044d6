"""CPU-side checks of the host-vector plumbing: lgpu_debug_refine_host and its binding refuse malformed input before
any device work, so these pass without a GPU."""
import numpy as np
import pytest

from lancedb_b200 import _native

f32 = np.float32


def test_debug_refine_host_checks_shapes_before_the_call():
    with pytest.raises(ValueError, match="queries must be"):
        _native.debug_refine_host(np.ones((2, 8), f32), np.ones((4, 7), f32), np.zeros((2, 3), np.uint64))
    with pytest.raises(ValueError, match="queries must be"):
        _native.debug_refine_host(np.ones((1, 8), f32), np.ones((4, 8), f32), np.zeros((2, 3), np.uint64))


def test_debug_refine_host_refuses_bad_positions_and_metrics_before_the_device():
    q, x = np.ones((1, 8), f32), np.ones((4, 8), f32)
    with pytest.raises(ValueError, match="position"):
        _native.debug_refine_host(q, x, np.array([[1, 4]], np.uint64))
    lib = _native.load()
    pos = np.zeros((1, 1), np.uint64)
    out = np.empty((1, 1), f32)
    assert lib.lgpu_debug_refine_host(q.ctypes.data, 1, x.ctypes.data, 4, 8, pos.ctypes.data, 1, 7, 0,
                                      out.ctypes.data) == _native.LGPU_INVALID_INPUT
    assert b"distance type" in lib.lgpu_last_error()


def test_host_bytes_refuses_a_handle_it_does_not_know():
    lib = _native.load()
    import ctypes as C
    b, where = C.c_uint64(0), C.c_int(0)
    assert lib.lgpu_index_host_bytes(None, C.byref(b), C.byref(where)) != _native.LGPU_OK
    assert lib.lgpu_index_host_bytes(None, None, None) == _native.LGPU_INVALID_INPUT

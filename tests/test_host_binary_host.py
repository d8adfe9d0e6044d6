"""CPU-side checks of binary handles kept in host memory: lgpu_binary_host_bytes and lgpu_binary_device_bytes refuse a
null or unknown handle before any device work, and the Python accessors refuse a closed handle, so these pass without a
GPU."""
import ctypes as C

import pytest

from lancedb_b200 import _native


def test_binary_byte_accessors_refuse_a_handle_they_do_not_know():
    lib = _native.load()
    b, where = C.c_uint64(0), C.c_int(0)
    assert lib.lgpu_binary_host_bytes(None, None, None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_binary_host_bytes(None, C.byref(b), C.byref(where)) == _native.LGPU_INVALID_INPUT
    assert b"binary handle is null" in lib.lgpu_last_error()
    assert lib.lgpu_binary_host_bytes(C.c_void_p(0x1000), C.byref(b), None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_binary_device_bytes(None, C.byref(b)) == _native.LGPU_INVALID_INPUT
    assert b"binary handle is null" in lib.lgpu_last_error()
    assert lib.lgpu_binary_device_bytes(C.c_void_p(0x1000), C.byref(b)) == _native.LGPU_INVALID_INPUT
    assert b.value == 0 and where.value == 0


def test_python_accessors_refuse_a_closed_handle():
    bx = object.__new__(_native.GpuBinary)
    bx._h = None
    with pytest.raises(ValueError):
        bx.host_bytes()
    with pytest.raises(ValueError):
        bx.rows_on_host
    with pytest.raises(ValueError):
        bx.device_bytes

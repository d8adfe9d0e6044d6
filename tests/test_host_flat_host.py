"""CPU-side checks of flat handles kept in host memory: lgpu_flat_host_bytes and the Python accessors refuse a null or
unknown handle before any device work, so these pass without a GPU."""
import ctypes as C

import pytest

from lancedb_b200 import _native


def test_flat_host_bytes_refuses_a_handle_it_does_not_know():
    lib = _native.load()
    b, where = C.c_uint64(0), C.c_int(0)
    assert lib.lgpu_flat_host_bytes(None, None, None) == _native.LGPU_INVALID_INPUT
    assert lib.lgpu_flat_host_bytes(None, C.byref(b), C.byref(where)) == _native.LGPU_INVALID_INPUT
    assert b"flat handle is null" in lib.lgpu_last_error()
    assert lib.lgpu_flat_host_bytes(C.c_void_p(0x1000), C.byref(b), None) == _native.LGPU_INVALID_INPUT
    assert b.value == 0 and where.value == 0


def test_python_accessors_refuse_a_closed_handle():
    fl = object.__new__(_native.GpuFlat)
    fl._h = None
    with pytest.raises(ValueError):
        fl.host_bytes()
    with pytest.raises(ValueError):
        fl.rows_on_host

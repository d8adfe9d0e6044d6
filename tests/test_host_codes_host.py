"""CPU-side checks of IVF indexes whose codes may be kept in host memory: lgpu_index_code_bytes and
lgpu_ivf_binary_code_bytes refuse a null or unknown handle before any device work, and the Python accessors refuse a
closed handle, so these pass without a GPU."""
import ctypes as C

import pytest

from lancedb_b200 import _native


@pytest.mark.parametrize("fn,kind", [("lgpu_index_code_bytes", b"index"),
                                     ("lgpu_ivf_binary_code_bytes", b"binary IVF index")])
def test_code_bytes_refuses_a_handle_it_does_not_know(fn, kind):
    lib = _native.load()
    b, where = C.c_uint64(0), C.c_int(0)
    f = getattr(lib, fn)
    assert f(None, None, None) == _native.LGPU_INVALID_INPUT
    assert f(None, C.byref(b), C.byref(where)) == _native.LGPU_INVALID_INPUT
    assert kind + b" handle is null" in lib.lgpu_last_error()
    assert f(C.c_void_p(0x1000), C.byref(b), None) == _native.LGPU_INVALID_INPUT
    assert f(C.c_void_p(0x1000), None, C.byref(where)) == _native.LGPU_INVALID_INPUT
    assert b.value == 0 and where.value == 0


def test_last_streamed_code_bytes_refuses_a_null_output():
    lib = _native.load()
    assert lib.lgpu_last_streamed_code_bytes(None) == _native.LGPU_INVALID_INPUT


@pytest.mark.parametrize("cls", ["GpuIvfSq", "GpuIvfRq", "GpuIvfBinary"])
def test_python_accessors_refuse_a_closed_handle(cls):
    h = object.__new__(getattr(_native, cls))
    h._h = None
    with pytest.raises(ValueError):
        h.code_host_bytes()
    with pytest.raises(ValueError):
        h.codes_on_host

"""fdb_wrapper_compile's two-call protocol (size query, then copy) on the CPU: the copy is the image the
query sized, and a buffer smaller than the image is refused instead of being left unwritten."""
import ctypes as C

import pytest

from firedrake_b200 import _lib, op2
from firedrake_b200.codegen import CStringKernel, WrapperSpec


def _spec():
    s = op2.Set(10)
    d = op2.Dat(op2.DataSet(s, 2))
    return WrapperSpec(CStringKernel("static void k(double *x) { x[0] = 1.0; x[1] = x[0] * 2.0; }", "k"),
                       [d(op2.WRITE)])


def test_query_then_copy_gives_the_queried_image():
    spec = _spec()
    L = _lib.load()
    for _ in range(4):
        need = C.c_size_t()
        _lib.check(L.fdb_wrapper_compile(C.byref(spec.desc), None, 0, C.byref(need)))
        buf = (C.c_char * need.value)()
        got = C.c_size_t()
        _lib.check(L.fdb_wrapper_compile(C.byref(spec.desc), buf, need.value, C.byref(got)))
        assert got.value == need.value and bytes(buf)[:4] == b"\x7fELF"


def test_too_small_buffer_is_an_error():
    spec = _spec()
    need = len(spec.compile())
    L = _lib.load()
    buf = (C.c_char * 16)()
    got = C.c_size_t()
    assert L.fdb_wrapper_compile(C.byref(spec.desc), buf, 16, C.byref(got)) != 0
    assert got.value == need
    with pytest.raises(_lib.EngineError, match="needs"):
        _lib.check(L.fdb_wrapper_compile(C.byref(spec.desc), buf, 16, C.byref(got)))

"""The index-write session of the C ABI: a plain C99 program type-checks against it, and null arguments are refused
without a GPU."""
import ctypes
import os
import subprocess

from conftest import ROOT


def test_c_program_compiles_against_the_index_write_entries():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "index_write_abi_check.c")], check=True)


def test_index_write_entries_reject_null_arguments():
    from universal_recommender_b200 import _native as N
    L = N.lib()
    h = ctypes.c_void_p()
    prm = N.IndexWriteParamsT(1000, 1 << 20)
    n, p64, pc = ctypes.c_int64(), ctypes.POINTER(ctypes.c_int64)(), ctypes.c_void_p()
    assert L.cco_index_write_begin(None, b"", 0, ctypes.byref(prm), ctypes.byref(h)) == N.E_INVALID_ARG
    assert L.cco_index_write_fields(None, ctypes.byref(n), ctypes.byref(p64), ctypes.byref(pc)) == N.E_INVALID_ARG
    assert L.cco_index_write_requests(None, ctypes.byref(n), ctypes.byref(p64), ctypes.byref(p64)) == N.E_INVALID_ARG
    assert L.cco_index_write_response(None, 0, b"{}", 2) == N.E_INVALID_ARG
    assert L.cco_index_write_retry(None, ctypes.byref(N.IndexWriteRetryT())) == N.E_INVALID_ARG
    assert L.cco_index_write_finish(None, ctypes.byref(N.IndexWriteOutT())) == N.E_INVALID_ARG
    assert L.cco_index_write_free(None) == N.OK

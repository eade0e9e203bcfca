"""The clean write-back entries of the C ABI: a plain C99 program type-checks against them, and null arguments are refused
without a GPU."""
import ctypes
import os
import subprocess

from conftest import ROOT


def test_c_program_compiles_against_the_clean_entries():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_clean_abi_check.c")], check=True)


def test_clean_entries_reject_null_arguments():
    from universal_recommender_b200 import _native as N
    L = N.lib()
    x, out, n = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_int64()
    st = N.EventCleanStatsT()
    assert L.cco_event_log_clean_begin(None, 0, ctypes.byref(x)) == N.E_INVALID_ARG
    assert L.cco_event_log_clean_append(None, b"x", 1, ctypes.byref(out), ctypes.byref(n)) == N.E_INVALID_ARG
    assert L.cco_event_log_clean_finish(None, ctypes.byref(out), ctypes.byref(n), ctypes.byref(st)) == N.E_INVALID_ARG
    assert L.cco_event_log_clean_free(None) == N.OK

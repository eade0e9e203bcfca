"""The erase entries of the C ABI: a plain C99 program type-checks against them, and null arguments are refused without a
GPU."""
import ctypes
import os
import subprocess

from conftest import ROOT


def test_c_program_compiles_against_the_erase_entries():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_erase_abi_check.c")], check=True)


def test_erase_entries_reject_null_arguments():
    from universal_recommender_b200 import _native as N
    L = N.lib()
    off = (ctypes.c_int64 * 2)(0, 1)
    st, n = N.EventEraseStatsT(), ctypes.c_int64()
    assert L.cco_event_log_erase(None, 0, None, None, 0, None, None, None) == N.E_INVALID_ARG
    assert b"null argument" in L.cco_last_error()
    assert L.cco_event_log_erase(None, 1, off, b"u", 0, None, None, ctypes.byref(st)) == N.E_INVALID_ARG
    assert L.cco_event_log_erased(None, ctypes.byref(n)) == N.E_INVALID_ARG
    assert L.cco_event_log_erased(None, None) == N.E_INVALID_ARG

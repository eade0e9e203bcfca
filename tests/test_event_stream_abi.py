"""The streamed event-log entries of the C ABI: a plain C99 program type-checks against them, and null arguments are refused
without a GPU."""
import ctypes
import os
import subprocess

from conftest import ROOT


def test_c_program_compiles_against_the_streamed_event_log_entries():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_stream_abi_check.c")], check=True)


def test_streamed_event_log_entries_reject_null_arguments():
    from universal_recommender_b200 import _native as N
    L = N.lib()
    h = ctypes.c_void_p()
    assert L.cco_event_log_begin(None, 1 << 20, ctypes.byref(h)) == N.E_INVALID_ARG
    assert L.cco_event_log_append(None, b"x", 1) == N.E_INVALID_ARG
    assert L.cco_event_log_finish(None) == N.E_INVALID_ARG

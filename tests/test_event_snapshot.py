"""Event log snapshots without a GPU: the host reader of tests/snapshot_ref.py against the layout include/cco_b200.h
documents (constants, section kinds, the checksum), its refusals, and the C entries' null-argument checks."""
import os
import re
import struct
import subprocess

import pytest

import snapshot_ref as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cco_b200.h")


def layout_comment() -> str:
    text = open(HEADER).read()
    i = text.index(" * Snapshots:")
    return text[i:text.index("*/", i)]


def checksum_by_the_words(data: bytes) -> int:
    """the documented checksum in plain integer arithmetic"""
    m = (1 << 64) - 1

    def mix(x):
        x ^= x >> 30
        x = (x * 0xBF58476D1CE4E5B9) & m
        x ^= x >> 27
        x = (x * 0x94D049BB133111EB) & m
        return x ^ (x >> 31)

    padded = data + b"\0" * (-len(data) % 8)
    h = mix(len(data))
    for i in range(len(padded) // 8):
        w = int.from_bytes(padded[8 * i:8 * i + 8], "little")
        h = (h + mix(w ^ ((i * 0x9E3779B97F4A7C15) & m))) & m
    return h


def test_kinds_and_version_are_the_documented_ones():
    doc = layout_comment()
    assert S.header_version(HEADER) == 1
    assert '"CCOLOGSN"' in doc and S.MAGIC == b"CCOLOGSN"
    assert "bytes [0, 64)" in doc and "40 n_sections" in doc and "multiples of 256" in doc
    named = dict((int(k), v) for k, v in re.findall(r"\b(\d+) ([a-z_]+)\b(?=[:;( ])", doc) if 1 <= int(k) <= 30)
    for k in (1, 2, 3, 4, 5, 12, 13, 14, 15, 16, 17, 18, 19):
        assert S.KINDS[k - 1] == named[k], (k, named.get(k))
    assert len(S.KINDS) == 30


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 255, 256, 1000])
def test_checksum_is_the_documented_sum(n):
    data = bytes((i * 131 + 7) % 256 for i in range(n))
    assert S.checksum(data) == checksum_by_the_words(data)
    if n:
        flipped = bytearray(data)
        flipped[n // 2] ^= 0x10
        assert S.checksum(bytes(flipped)) != S.checksum(data)


def sample_image():
    state = struct.pack("<16q", 2, 1, -5, 1 << 16, 10, 0, 1, 0, 0, 3, 2, -1, 0, 0, 0, 0)
    names = struct.pack("<4q", 2, 0, 3, 7) + b"buyview"
    counts = struct.pack("<4q", 4, 2, 0, 1)
    return S.write_image([(S.KIND["state"], state, 0), (S.KIND["names"], names, 0), (S.KIND["counts"], counts, 0),
                          (S.KIND["rank_times"], struct.pack("<q", 99), 16)], 1, 2)


def test_a_written_image_reads_back():
    img = sample_image()
    h = S.read_header(img)
    assert (h.version, h.abi, h.total) == (1, 2, len(img))
    assert [s.name for s in h.sections] == ["state", "names", "counts", "rank_times"]
    assert all(s.offset % 256 == 0 for s in h.sections) and h.sections[0].offset == 256
    S.check_sections(img, h)
    assert S.strings(img[h.sections[1].offset:h.sections[1].offset + h.sections[1].length]) == [b"buy", b"view"]


def test_the_reader_refuses_what_the_layout_forbids():
    img = bytearray(sample_image())
    with pytest.raises(ValueError, match="magic"):
        S.read_header(b"X" + bytes(img[1:]))
    bad = bytearray(img)
    bad[64 + 8] ^= 1   # the first section's offset
    with pytest.raises(ValueError, match="header checksum"):
        S.read_header(bytes(bad))
    h = S.read_header(bytes(img))
    bad = bytearray(img)
    bad[h.sections[2].offset] ^= 1
    with pytest.raises(ValueError, match="counts: checksum"):
        S.check_sections(bytes(bad), S.read_header(bytes(bad)))
    # a table entry past the end, re-sealed with a valid header checksum: refused by the layout, not the checksum
    secs = [(s.kind, bytes(img[s.offset:s.offset + s.length]), s.device_bytes) for s in h.sections]
    img2 = bytearray(S.write_image(secs, 1, 2))
    struct.pack_into("<q", img2, 64 + 40 * 3 + 16, 1 << 20)
    tab = bytes(img2[:64 + 40 * 4])
    struct.pack_into("<Q", img2, 32, S.checksum(tab[:32] + b"\0" * 8 + tab[40:]))
    with pytest.raises(ValueError, match="rank_times"):
        S.read_header(bytes(img2))


def build_c_program(tmp_path) -> str:
    from universal_recommender_b200 import _native
    exe = str(tmp_path / "event_snapshot_abi_check")
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_snapshot_abi_check.c"), "-o", exe, "-L", libdir, "-lcco_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_c_program_refuses_null_arguments_without_a_gpu(tmp_path):
    p = subprocess.run([build_c_program(tmp_path)], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout == "ok\n", (p.returncode, p.stdout, p.stderr)


def test_python_entries_refuse_null_arguments():
    import ctypes
    from universal_recommender_b200 import _native as N
    L = N.lib()
    b = ctypes.c_int64()
    assert L.cco_event_log_save_size(None, ctypes.byref(b)) == N.E_INVALID_ARG
    assert L.cco_event_log_save(None, 0, None, 0) == N.E_INVALID_ARG
    assert L.cco_event_log_load_begin(None, None) == N.E_INVALID_ARG
    assert L.cco_event_log_load_append(None, None, 0) == N.E_INVALID_ARG
    assert L.cco_event_log_load_finish(None) == N.E_INVALID_ARG

"""A host reader of event log snapshots (cco_event_log_save), written from the layout in include/cco_b200.h alone: the
header, the section table and the checksums, and a writer of images in that layout for the CPU tests."""
from __future__ import annotations

import re
import struct
from dataclasses import dataclass

import numpy as np

MAGIC = b"CCOLOGSN"
HEAD, ENTRY, ALIGN = 64, 40, 256
KINDS = ["state", "names", "counts", "fields", "property_lines", "train_users.offsets", "train_users.bytes",
         "train_items.offsets", "train_items.bytes", "rank_items.offsets", "rank_items.bytes", "rank_times", "train_lines",
         "rank_lines", "train_times", "train_keys", "records", "duplicate_times", "property_bytes", "properties.fields",
         "properties.value_offsets", "properties.values", "properties.item_offsets", "properties.item_bytes",
         "property_items.offsets", "property_items.bytes", "user_keys.offsets", "user_keys.bytes", "item_keys.offsets",
         "item_keys.bytes"]
KIND = {name: k + 1 for k, name in enumerate(KINDS)}
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


def _mix(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def checksum(data) -> int:
    """mix(n) + sum over words i of mix(w_i ^ i * golden) mod 2^64, the last word zero-filled"""
    b = bytes(data)
    n = len(b)
    w = np.frombuffer(b + b"\0" * (-n % 8), dtype="<u8")
    with np.errstate(over="ignore"):
        terms = _mix(w ^ (np.arange(len(w), dtype=np.uint64) * np.uint64(GOLDEN)))
        total = int(terms.sum(dtype=np.uint64)) if len(w) else 0
    return (total + int(_mix(np.array([n], dtype=np.uint64))[0])) & M64


@dataclass
class Section:
    kind: int
    offset: int
    length: int
    device_bytes: int
    checksum: int

    @property
    def name(self) -> str:
        return KINDS[self.kind - 1] if 1 <= self.kind <= len(KINDS) else "?"


@dataclass
class Header:
    version: int
    abi: int
    total: int
    checksum: int
    sections: list


def read_header(img) -> Header:
    """the header and section table of an image, checked as the layout states (ValueError otherwise)"""
    b = bytes(img[:HEAD])
    if len(b) < HEAD or b[:8] != MAGIC:
        raise ValueError("bad magic")
    version, abi, n, zero, total, hsum = struct.unpack_from("<IIIIqQ", b, 8)
    if zero or any(b[40:64]):
        raise ValueError("reserved header bytes are not 0")
    tab = bytes(img[:HEAD + ENTRY * n])
    if len(tab) < HEAD + ENTRY * n:
        raise ValueError("truncated section table")
    if checksum(tab[:32] + b"\0" * 8 + tab[40:]) != hsum:
        raise ValueError("header checksum mismatch")
    secs, end, kind = [], HEAD + ENTRY * n, 0
    for i in range(n):
        k, z, off, ln, dev, cs = struct.unpack_from("<IIqqqQ", tab, HEAD + ENTRY * i)
        s = Section(k, off, ln, dev, cs)
        if z or k <= kind or off % ALIGN or off < end or ln < 0 or off + ln > total:
            raise ValueError(f"section {i} ({s.name}) breaks the layout")
        if (k <= KIND["property_lines"]) != (dev == 0):
            raise ValueError(f"section {s.name}: host sections have 0 device bytes, device sections more")
        secs.append(s)
        kind, end = k, off + ln
    if end != total:
        raise ValueError("the last section does not end at the total")
    return Header(version, abi, total, hsum, secs)


def check_sections(img, h: Header) -> None:
    for s in h.sections:
        if checksum(img[s.offset:s.offset + s.length]) != s.checksum:
            raise ValueError(f"section {s.name}: checksum mismatch")


def strings(b: bytes) -> list:
    """a string-list section: i64 n, i64 offsets [n + 1], bytes"""
    n = struct.unpack_from("<q", b, 0)[0]
    off = struct.unpack_from(f"<{n + 1}q", b, 8)
    base = 16 + 8 * n
    return [b[base + off[i]:base + off[i + 1]] for i in range(n)]


def header_version(path: str) -> int:
    """CCO_SNAPSHOT_VERSION as include/cco_b200.h defines it"""
    return int(re.search(r"#define CCO_SNAPSHOT_VERSION (\d+)", open(path).read()).group(1))


def write_image(sections: list, version: int, abi: int) -> bytes:
    """an image of [(kind, payload bytes, device bytes)] in the documented layout"""
    sections = sorted(sections)
    n = len(sections)
    at = -(-(HEAD + ENTRY * n) // ALIGN) * ALIGN
    place = []
    for k, data, dev in sections:
        place.append((k, at, data, dev))
        at = -(-(at + len(data)) // ALIGN) * ALIGN
    total = place[-1][1] + len(place[-1][2])
    tab = b"".join(struct.pack("<IIqqqQ", k, 0, off, len(d), dev, checksum(d)) for k, off, d, dev in place)
    head = MAGIC + struct.pack("<IIIIqQ", version, abi, n, 0, total, 0) + b"\0" * 24
    hs = checksum(head + tab)
    img = bytearray(head[:32] + struct.pack("<Q", hs) + head[40:] + tab)
    for k, off, d, dev in place:
        img += b"\0" * (off - len(img)) + d
    return bytes(img)

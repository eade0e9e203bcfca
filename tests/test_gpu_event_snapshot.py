"""Event log snapshots on the H100 (cco_event_log_save / cco_event_log_load_*): a saved and loaded log is the log that was
saved -- info, window_stats, resident_bytes, intern_stats, the ingest and every consumer's body -- for every flag
combination and window, the handmade fixtures and a C2-sized export; a loaded extendable log extends as the saved one
does; any chunking of save and load gives the same log; a damaged image is refused with a message naming its section,
and the context stays usable."""
import ctypes as C
import io
import os
import re
import struct
import subprocess
import sys

import numpy as np
import pytest

import snapshot_ref as S
import universal_recommender_b200 as ur
from conftest import load_golden
from test_event_extend import SEAM_CASES, W, dump
from test_event_snapshot import build_c_program
from test_event_window import DAY, NOW, random_export
from test_gpu_event_extend import outputs
from test_gpu_event_window import AP
from user_query_data import handmade_export, handmade_params
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FLAGS = {"none": {}, "history": dict(keep_history=True), "extendable": dict(extendable=True), "intern": dict(intern_ids=True),
         "all": dict(keep_history=True, extendable=True, intern_ids=True)}
WINDOWS = {"none": None, "both": W, "dedup": E.EventWindow(None, True)}


def image(log, chunk=None) -> bytes:
    f = io.BytesIO()
    n = log.save(f, chunk_bytes=chunk)
    assert n == len(f.getvalue()) == log.save_size()
    return f.getvalue()


def state(ctx, log, now, flags) -> dict:
    """every output of a log: outputs() of test_gpu_event_extend (without history, what needs none), resident bytes,
    intern stats and the refreshed properties"""
    if flags.get("keep_history"):
        out = outputs(ctx, log, now)
    else:
        out = {"info": log.info(), "stats": log.window_stats()}
        names = out["info"].names or ["none"]
        ds, users, items = ctx.ingest_event_log(log, names)
        try:
            out["ingest"] = (users, items, [[np.asarray(a).tolist() for a in ctx.dataset_to_host(ds, t)] for t in range(len(names))])
        finally:
            ctx.free_dataset(ds)
        try:
            out["calc_all"] = ur.calc_all_from_events(log, AP, 0, now_ms=now, ctx=ctx)
            out["calc_pop"] = ur.calc_pop_from_events(out["calc_all"], log, AP, now_ms=now, ctx=ctx)
        except ValueError as e:
            out["calc_all"] = str(e)
    if isinstance(out.get("calc_all"), bytes):
        r = ur.refresh_properties_from_events(out["calc_all"], log, AP, now_ms=now, ctx=ctx)
        out["refresh"] = (r.body, r.delta, r.deletes)
    out["resident"] = log.resident_bytes()
    if flags.get("intern_ids"):
        out["intern"] = log.intern_stats()
    return out


def reloaded(ctx, log, **kw):
    img = image(log)
    h = S.read_header(img)   # the host reader agrees with the library's layout and device checksums
    S.check_sections(img, h)
    back = ctx.load_events(img, **kw)
    assert image(back) == img
    return back, img


@pytest.mark.parametrize("window", sorted(WINDOWS))
@pytest.mark.parametrize("flags", sorted(FLAGS))
def test_round_trip(ctx, flags, window):
    fl = FLAGS[flags]
    for chunk in (None, 900):
        with ctx.read_events(random_export(5, 400), chunk_bytes=chunk, window=WINDOWS[window], now_ms=NOW, **fl) as log:
            want = state(ctx, log, NOW, fl)
            back, _ = reloaded(ctx, log)
            with back:
                assert state(ctx, back, NOW, fl) == want


def test_handmade_fixture_and_query_file(ctx):
    index = load_golden("item_queries_handmade.json")["index"].encode()
    qfile = load_golden("query_file_handmade.json")["file"].encode()
    for fl in (FLAGS["history"], FLAGS["all"]):
        with ctx.read_events(handmade_export(), **fl) as log:
            back, _ = reloaded(ctx, log)
            with back:
                assert state(ctx, back, NOW, fl) == state(ctx, log, NOW, fl)
                got, want = (ctx.query_file(x, index, handmade_params(), qfile, NOW) for x in (back, log))
                assert got[0] == want[0] and np.array_equal(got[1], want[1])


def test_c2_sized_export(ctx):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import synth
    from event_extend_bench import export_days
    from events_bench import END_MS
    whole, n_a, _ = export_days(synth.CONFIGS["C2"], 1.0, ctx.host_array)
    try:
        fl = FLAGS["all"]
        with ctx.read_events(whole, chunk_bytes=32 << 20, window=E.EventWindow("30 days", True), now_ms=END_MS, **fl) as log:
            want = state(ctx, log, END_MS, fl)
            back, img = reloaded(ctx, log)
            with back:
                assert state(ctx, back, END_MS, fl) == want
            assert len(img) < 2 * log.resident_bytes()
    finally:
        ctx.host_free(whole)


@pytest.mark.parametrize("case", sorted(SEAM_CASES))
def test_extend_after_load(ctx, case):
    a, b, now1, now2 = SEAM_CASES[case]
    a, b = dump(a), dump(b)
    fl = FLAGS["all"]
    for w in (W, E.EventWindow("5 days")):
        n2 = now2 if w.duration else now1
        with ctx.read_events(a, window=w, now_ms=now1, **fl) as log:
            back, _ = reloaded(ctx, log)
            with back:
                log.extend(b, window=w, now_ms=n2)
                back.extend(b, window=w, now_ms=n2)
                got = state(ctx, back, n2, fl)
                assert got == state(ctx, log, n2, fl)
                with ctx.read_events(a + b, window=w, now_ms=n2, keep_history=True) as fresh:
                    want = outputs(ctx, fresh, n2)
                assert {k: got[k] for k in want} == want


def test_extend_after_load_over_days(ctx):
    from test_gpu_event_extend import timed_export
    lines = timed_export(11, 900, 10).splitlines()
    parts = np.array_split(np.arange(len(lines)), 4)
    part = lambda k: b"".join(lines[i] + b"\n" for i in parts[k])
    w, now, fl = E.EventWindow("5 days", True), NOW - 3 * DAY, FLAGS["all"]
    with ctx.read_events(part(0), window=w, now_ms=now, **fl) as log:
        for k in range(1, 4):
            back, _ = reloaded(ctx, log)
            log.free()
            log = back
            now += DAY
            log.extend(part(k), window=w, now_ms=now)
        with ctx.read_events(b"".join(part(j) for j in range(4)), window=w, now_ms=now, keep_history=True) as fresh:
            want = outputs(ctx, fresh, now)
        got = state(ctx, log, now, fl)
        assert {k: got[k] for k in want} == want
        log.free()


@pytest.fixture(scope="module")
def snap(ctx):
    """an image with every section: a log with properties, history, records, duplicate times and interned ids"""
    a, b, now1, now2 = SEAM_CASES["properties_around_the_cutoff"]
    data = dump(a) + dump(b) + random_export(9, 300)
    with ctx.read_events(data, window=W, now_ms=now1, **FLAGS["all"]) as log:
        log.extend(random_export(9, 100), window=W, now_ms=now1)
        img = image(log)
        yield img, state(ctx, log, now1, FLAGS["all"]), now1


def test_every_chunking_gives_the_same_log(ctx, snap):
    img, want, now = snap
    h = S.read_header(img)
    with ctx.load_events(img) as log:
        assert image(log, chunk=1) == img
        for c in (255, 256, 257, 4099):
            assert image(log, chunk=c) == img
    cuts = sorted({x for s in h.sections for x in (s.offset - 1, s.offset, s.offset + 1, s.offset + s.length - 1,
                                                   s.offset + s.length + 1) if 0 < x < len(img)})
    for k in cuts:
        with ctx.load_events([img[:k], img[k:]]) as log:
            assert log.info() == want["info"] and log.resident_bytes() == want["resident"]
    with ctx.load_events(img, chunk_bytes=1) as log:
        assert state(ctx, log, now, FLAGS["all"]) == want


def test_load_from_a_file_and_save_to_a_path(ctx, snap, tmp_path):
    img, want, now = snap
    p = tmp_path / "log.snap"
    p.write_bytes(img)
    with ctx.load_events(str(p), chunk_bytes=1000) as log:
        assert state(ctx, log, now, FLAGS["all"]) == want
        q = tmp_path / "again.snap"
        assert log.save(str(q), chunk_bytes=777) == len(img)
        assert q.read_bytes() == img


def refused(ctx, data, message):
    with pytest.raises(N.CcoError, match=re.escape(message)) as e:
        ctx.load_events(data)
    assert e.value.status == N.E_INVALID_ARG


def reseal(img: bytes, name: str, mutate) -> bytes:
    """img with section `name` changed by mutate(bytearray) and its checksum and the header checksum made to match"""
    b = bytearray(img)
    h = S.read_header(img)
    i, s = next((i, s) for i, s in enumerate(h.sections) if s.name == name)
    sec = bytearray(b[s.offset:s.offset + s.length])
    mutate(sec)
    b[s.offset:s.offset + s.length] = sec
    struct.pack_into("<Q", b, 64 + 40 * i + 32, S.checksum(bytes(sec)))
    tab = bytes(b[:64 + 40 * len(h.sections)])
    struct.pack_into("<Q", b, 32, S.checksum(tab[:32] + b"\0" * 8 + tab[40:]))
    return bytes(b)


def test_damaged_images_are_refused_by_section(ctx, snap):
    img, want, now = snap
    h = S.read_header(img)
    names = [s.name for s in h.sections]
    assert {"records", "duplicate_times", "property_bytes", "train_keys", "user_keys.bytes", "properties.values"} <= set(names)
    for s in h.sections:   # truncation at every section boundary
        if s.length:
            refused(ctx, img[:s.offset], f"snapshot truncated at byte {s.offset} of {len(img)}: section {s.name} is incomplete")
    last = h.sections[-1]
    refused(ctx, img[:-1], f"snapshot truncated at byte {len(img) - 1} of {len(img)}: section {last.name} is incomplete")
    refused(ctx, img[:100], "snapshot truncated at byte 100: the header and section table are incomplete")
    refused(ctx, img + b"\0", f"snapshot: bytes past its end ({len(img)} bytes)")
    for s in h.sections:   # one flipped byte in every section
        if s.length:
            b = bytearray(img)
            b[s.offset + s.length // 2] ^= 0x04
            refused(ctx, bytes(b), f"snapshot section {s.name}: checksum mismatch")
    b = bytearray(img)
    b[64 + 8] ^= 1
    refused(ctx, bytes(b), "snapshot header: checksum mismatch")
    b = bytearray(img)
    struct.pack_into("<I", b, 8, 2)
    refused(ctx, bytes(b), "snapshot header: format version 2, this library reads 1")
    refused(ctx, b"XX" + img[2:], "snapshot header: not an event log snapshot (bad magic)")
    # a section table pointing past the end, sealed with a valid header checksum
    b = bytearray(img)
    n = len(h.sections)
    struct.pack_into("<q", b, 64 + 40 * (n - 1) + 16, last.length + 4096)
    tab = bytes(b[:64 + 40 * n])
    struct.pack_into("<Q", b, 32, S.checksum(tab[:32] + b"\0" * 8 + tab[40:]))
    refused(ctx, bytes(b), f"snapshot section {last.name}: [{last.offset}, +{last.length + 4096}) runs past the end ({len(img)} bytes)")
    # structural violations under valid checksums
    def dec(sec):
        struct.pack_into("<q", sec, 16, struct.unpack_from("<q", sec, 8)[0] + 10**6)
    refused(ctx, reseal(img, "train_users.offsets", dec), "snapshot section train_users.offsets: offset")
    refused(ctx, reseal(img, "train_keys", lambda sec: struct.pack_into("<Q", sec, 0, 1 << 62)),
            "snapshot section train_keys: entry 0 holds a key >= its table's key count")
    refused(ctx, reseal(img, "records", lambda sec: struct.pack_into("<q", sec, 40 + 24, -1)), "snapshot section records: record 1")
    refused(ctx, reseal(img, "train_lines", lambda sec: struct.pack_into("<q", sec, 0, 1 << 40)),
            "snapshot section train_lines: entry 0 is not a line of the log")
    refused(ctx, reseal(img, "properties.fields", lambda sec: struct.pack_into("<i", sec, 0, 999)),
            "snapshot section properties.fields: entry 0 is not a field")
    refused(ctx, reseal(img, "counts", lambda sec: struct.pack_into("<q", sec, 0, struct.unpack_from("<q", sec, 0)[0] + 1)),
            "snapshot section train_users.offsets:")
    # an id stored twice: the second user key's string made equal to the first's (when their lengths agree)
    u = next(s for s in h.sections if s.name == "user_keys.offsets")
    off = np.frombuffer(img[u.offset:u.offset + u.length], "<i8")
    ub = next(s for s in h.sections if s.name == "user_keys.bytes")
    first = img[ub.offset:ub.offset + off[1]]
    if off[2] - off[1] == len(first):
        def same(sec):
            sec[off[1]:off[2]] = first
        refused(ctx, reseal(img, "user_keys.bytes", same), "snapshot section user_keys.bytes: an id is stored twice")
    # the context and the image stay usable
    with ctx.load_events(img) as log:
        assert state(ctx, log, now, FLAGS["all"]) == want


def test_refusals_and_resources(ctx, snap):
    img, want, now = snap
    L = N.lib()
    with ctx.read_events(random_export(3, 50)) as fresh:
        before = fresh.resident_bytes()
    h = C.c_void_p()
    assert L.cco_event_log_load_begin(ctx._h, h) == N.OK
    assert L.cco_event_log_load_append(h, img, len(img) // 2) == N.OK
    assert L.cco_event_log_load_finish(h) == N.E_INVALID_ARG
    assert L.cco_event_log_load_append(h, img, 1) == N.E_INVALID_ARG   # a failed load answers with its failure
    L.cco_event_log_free(h)
    with ctx.read_events(random_export(3, 50)) as fresh:
        assert fresh.resident_bytes() == before
    # a log in progress or failed is not saved
    b = C.c_int64()
    assert L.cco_event_log_begin(ctx._h, 1 << 16, h) == N.OK
    assert L.cco_event_log_save_size(h, b) == N.E_INVALID_ARG
    assert L.cco_event_log_append(h, b"{}\n", 3) == N.OK
    assert L.cco_event_log_finish(h) == N.E_INVALID_ARG
    assert L.cco_event_log_save_size(h, b) == N.E_INVALID_ARG
    L.cco_event_log_free(h)
    # a log being loaded takes no other call
    assert L.cco_event_log_load_begin(ctx._h, h) == N.OK
    assert L.cco_event_log_append(h, b"{}\n", 3) == N.E_INVALID_ARG
    assert L.cco_event_log_save_size(h, b) == N.E_INVALID_ARG
    L.cco_event_log_free(h)
    g = ur.CcoContext(devices=[0])
    try:
        with pytest.raises(N.CcoError) as e:
            g.load_events(img)
        assert e.value.status == N.E_UNSUPPORTED
    finally:
        g.close()


def test_c_program_saves_and_loads(ctx, tmp_path):
    data = random_export(13, 400)
    (tmp_path / "a.json").write_bytes(data)
    exe = build_c_program(tmp_path)
    p = subprocess.run([exe, str(tmp_path / "a.json"), str(tmp_path / "a.snap"), "4093"], capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout, p.stderr)
    n_lines, rb, rb2, uk, size = (int(v) for v in p.stdout.split())
    with ctx.read_events(data, chunk_bytes=1 << 16, keep_history=True, extendable=True, intern_ids=True) as log:
        assert (n_lines, rb, rb2, uk) == (log.info().n_lines, log.resident_bytes(), log.resident_bytes(), log.intern_stats()[0])
    with ctx.load_events(str(tmp_path / "a.snap")) as back:
        assert back.save_size() == size == (tmp_path / "a.snap").stat().st_size

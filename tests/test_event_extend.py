"""Extendable event logs off the GPU: the host mirror's extend (events.extend_clean) restates the contract of
cco_event_log_extend over clean_events -- the state kept after A under an earlier window, extended with B under a later
one, is what one read of A followed by B under the later window keeps -- and the C entries type-check and refuse null
arguments without a GPU."""
import json
import os
import random
import subprocess

import pytest

from conftest import ROOT
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from universal_recommender_b200 import events as E

CUT = NOW - 5 * DAY
W = E.EventWindow("5 days", True)


def row(name, u, i=None, t=NOW - DAY, etype="user", **kw) -> dict:
    r = {"event": name, "entityType": etype, "entityId": u}
    if i is not None:
        r.update(targetEntityType="item", targetEntityId=i)
    r.update(kw)
    r["eventTime"] = iso_ms(t)
    return r


def dump(rows) -> bytes:
    return b"".join(json.dumps(r).encode() + b"\n" for r in rows)


def parsed(data: bytes) -> list:
    return [E.parse_line(i, raw) for i, raw in enumerate(E.export_lines(data))]


def contract(events, k, w1, now1, w2, now2):
    """extend_clean(clean_kept(A, w1), B, w2) against clean_events(A + B, w2): events, expired, duplicates"""
    kept = E.extend_clean(E.clean_kept(events[:k], w1, now1), events[k:], w2, now2)
    full, n_expired, n_dup = E.clean_events(events, w2, now2)
    assert [e.line for e in kept.events] == [e.line for e in full]
    assert (kept.n_expired, kept.n_duplicates) == (n_expired, n_dup)
    return kept


# the seam cases the device replays (tests/test_gpu_event_extend.py): (A rows, B rows, first now, second now); the window
# is W at both reads, so the cutoff moves by now2 - now1
SEAM_CASES = {
    # a line of B supersedes a retained line of A (B later), is dropped for it (B earlier), or wins the tie (equal time)
    "b_later": ([row("buy", "u1", "i1", NOW - 2 * DAY)], [row("buy", "u1", "i1", NOW - DAY)], NOW, NOW),
    "b_earlier": ([row("buy", "u1", "i1", NOW - DAY)], [row("buy", "u1", "i1", NOW - 2 * DAY)], NOW, NOW),
    "equal_time": ([row("view", "u1", "i1", NOW - DAY, prId="p")], [row("view", "u1", "i1", NOW - DAY, prId="p")], NOW, NOW),
    # an ignored line and a property line across the seam
    "ignored_and_property": ([row("like", "u1", t=NOW - 3 * DAY), row("$set", "i1", t=NOW - 3 * DAY, etype="item", properties={"a": 1})],
                             [row("like", "u1", t=NOW - DAY), row("$set", "i1", t=NOW - DAY, etype="item", properties={"a": 1})], NOW, NOW),
    # a duplicate of A dropped under c1 whose time falls at or before c2: expired, not a duplicate, after the extend
    "dup_expires": ([row("buy", "u1", "i1", NOW - 4 * DAY), row("buy", "u1", "i1", NOW - 2 * DAY), row("buy", "u2", "i2", NOW - 4 * DAY)],
                    [row("buy", "u3", "i1", NOW)], NOW, NOW + DAY + DAY // 2),
    # a retained line of A expires under c2, and its name keeps its place
    "a_expires": ([row("view", "u1", "i1", NOW - 4 * DAY), row("buy", "u2", "i2", NOW - DAY)], [row("buy", "u1", "i2", NOW + DAY)],
                  NOW, NOW + 2 * DAY),
    # $set / $unset never expire; an expired $delete lets the $set before it count again
    "properties_around_the_cutoff": (
        [row("$set", "i1", t=CUT - 9, etype="item", properties={"f": 1, "g": "x"}), row("$delete", "i1", t=CUT + 5, etype="item"),
         row("$unset", "i1", t=CUT - 1, etype="item", properties={"g": None}), row("$set", "i2", t=CUT + 1, etype="item", properties={"f": 2}),
         row("buy", "u1", "i1", NOW)],
        [row("$set", "i2", t=CUT + 1, etype="item", properties={"f": 2}), row("$delete", "i2", t=NOW, etype="item"),
         row("buy", "u2", "i2", NOW)], NOW, NOW + 10),
}


@pytest.mark.parametrize("case", sorted(SEAM_CASES))
def test_seam_cases(case):
    a, b, now1, now2 = SEAM_CASES[case]
    events = parsed(dump(a + b))
    for w in (W, E.EventWindow("5 days"), E.EventWindow(None, True)):
        contract(events, len(a), w, now1, w, now2 if w.duration else now1)


def test_seam_case_outcomes():
    """what the seam cases are about actually happens in them"""
    def run(case):
        a, b, now1, now2 = SEAM_CASES[case]
        ev = parsed(dump(a + b))
        return E.clean_kept(ev[:len(a)], W, now1), contract(ev, len(a), W, now1, W, now2)
    _, k = run("b_later")
    assert [e.line for e in k.events] == [1] and k.n_duplicates == 1
    _, k = run("b_earlier")
    assert [e.line for e in k.events] == [0] and k.n_duplicates == 1
    _, k = run("equal_time")
    assert [e.line for e in k.events] == [1]
    _, k = run("ignored_and_property")
    assert [e.line for e in k.events] == [2, 3] and k.n_duplicates == 2
    first, k = run("dup_expires")
    assert (first.n_expired, first.n_duplicates, first.dup_times) == (0, 1, [NOW - 4 * DAY])
    assert (k.n_expired, k.n_duplicates, k.dup_times) == (2, 0, [])
    first, k = run("a_expires")
    assert (first.n_expired, k.n_expired, [e.line for e in k.events]) == (0, 1, [1, 2])
    first, k = run("properties_around_the_cutoff")
    assert [e.event for e in first.events][:3] == ["$set", "$delete", "$unset"]
    assert [e.line for e in k.events] == [0, 2, 4, 5, 6, 7] and k.n_duplicates == 1 and k.n_expired == 1


@pytest.mark.parametrize("seed", range(5))
@pytest.mark.parametrize("window", [W, E.EventWindow("5 days"), E.EventWindow(None, True), None])
def test_random_exports_at_every_cutoff_step(seed, window):
    """split points 0, 1, middle, n - 1, n and random ones; c2 = c1, one ms later, a day later and past every line of A"""
    events = parsed(random_export(seed, 300))
    n = len(events)
    rng = random.Random(seed)
    for k in sorted({0, 1, n // 2, n - 1, n, rng.randrange(n), rng.randrange(n)}):
        last = max((e.time_ms for e in events[:k]), default=NOW)
        steps = [0, 1, DAY] + ([last - (NOW - 5 * DAY)] if window is not None and window.duration else [])
        for d in steps:
            contract(events, k, window, NOW, window, NOW + max(d, 0))


@pytest.mark.parametrize("seed", range(3))
def test_successive_extends_compose(seed):
    """ten one-day steps, each equal to one read of everything so far under that step's window"""
    events = parsed(random_export(seed, 400))
    bounds = sorted(random.Random(seed).sample(range(1, len(events)), 9))
    kept = E.clean_kept(events[:bounds[0]], W, NOW)
    for step, (b0, b1) in enumerate(zip(bounds, bounds[1:] + [len(events)]), 1):
        now = NOW + step * DAY // 3
        kept = E.extend_clean(kept, events[b0:b1], W, now)
        full, x, d = E.clean_events(events[:b1], W, now)
        assert ([e.line for e in kept.events], kept.n_expired, kept.n_duplicates) == ([e.line for e in full], x, d)
    assert kept.n_expired > 0 and kept.n_duplicates > 0


def test_an_earlier_cutoff_would_break_the_contract():
    """under c2 < c1 a whole read keeps lines of A that the state after A no longer has, so no extend could give it:
    the mirror refuses, as cco_event_log_extend does"""
    events = parsed(dump([row("buy", "u1", "i1", NOW - 4 * DAY), row("buy", "u2", "i2", NOW)]))
    kept = E.clean_kept(events[:1], W, NOW + 2 * DAY)
    assert kept.events == [] and kept.n_expired == 1
    full, _, _ = E.clean_events(events, W, NOW)
    assert [e.line for e in full] == [0, 1]          # line 0 is back under the earlier cutoff, and it is gone
    with pytest.raises(ValueError, match="cannot move back"):
        E.extend_clean(kept, events[1:], W, NOW)
    with pytest.raises(ValueError, match="cannot move back"):
        E.extend_clean(kept, events[1:], E.EventWindow(None, True), NOW)
    with pytest.raises(ValueError, match="removeDuplicates"):
        E.extend_clean(kept, events[1:], E.EventWindow("5 days"), NOW + 2 * DAY)


def test_c_program_compiles_against_the_extend_entries(tmp_path):
    src = os.path.join(ROOT, "tests", "abi", "event_extend_abi_check.c")
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), src],
                   check=True)


def test_c_program_refuses_null_arguments_without_a_gpu(tmp_path):
    from universal_recommender_b200 import _native
    exe = build_c_program(tmp_path)
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout == "ok\n", (p.returncode, p.stdout, p.stderr)
    assert _native.LOG_EXTENDABLE == 2


def build_c_program(tmp_path) -> str:
    from universal_recommender_b200 import _native
    exe = str(tmp_path / "event_extend_abi_check")
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_extend_abi_check.c"), "-o", exe, "-L", libdir, "-lcco_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_extend_entries_reject_null_arguments():
    import ctypes
    from universal_recommender_b200 import _native as N
    L = N.lib()
    b = ctypes.c_int64()
    w = N.EventWindowT(0, 0, 0)
    assert L.cco_event_log_extend(None, ctypes.byref(w)) == N.E_INVALID_ARG
    assert L.cco_event_log_extend(None, None) == N.E_INVALID_ARG
    assert L.cco_event_log_resident_bytes(None, ctypes.byref(b)) == N.E_INVALID_ARG
    h = ctypes.c_void_p()
    assert L.cco_event_log_begin_ex(None, 1, None, N.LOG_EXTENDABLE, ctypes.byref(h)) == N.E_INVALID_ARG

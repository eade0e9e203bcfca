"""Erasure off the GPU: the host mirror events.erase_kept against an independent restatement of the rule over the raw JSON
lines, and its three contracts -- erasing E from the state kept of X is the state kept of X - E (and stays so across
extends), lines read = retained + expired + duplicates + erased, and the kept lines after the erase are clean_export(X - E)
-- on random exports and the extend seam cases."""
import json
import random

import pytest

from test_event_extend import SEAM_CASES, W, dump, parsed
from test_event_window import NOW, DAY, random_export
from universal_recommender_b200 import events as E

WINDOWS = {"none": None, "duration": E.EventWindow("5 days"), "dedup": E.EventWindow(None, True), "both": W}


def ref_erased(raw: bytes, users: set, items: set) -> bool:
    """the rule restated over the JSON object: a user's event on an item target, any target in items, an item's property
    event"""
    o = json.loads(raw)
    target = o.get("targetEntityId")
    if target is None:
        return o["entityType"] == "item" and o["event"] in ("$set", "$unset", "$delete") and o["entityId"] in items
    if target in items:
        return True
    if o["entityType"] == "user" and o.get("targetEntityType") == "item" and o["entityId"] in users:
        return True
    return o["entityType"] == "item" and o["event"] in ("$set", "$unset", "$delete") and o["entityId"] in items


def without(data: bytes, users, items) -> bytes:
    """X - E: the export without the erased lines"""
    return b"".join(raw + b"\n" for raw in E.export_lines(data) if not ref_erased(raw, set(users), set(items)))


def id_sets(data: bytes, seed: int):
    """seeded user and item sets of an export: users only, items only, both, none, and ids it does not hold"""
    evs = parsed(data)
    us = sorted({e.entity_id for e in evs if e.entity_type == "user"})
    its = sorted({e.target_id for e in evs if e.target_id is not None} | {e.entity_id for e in evs if e.entity_type == "item"})
    rng = random.Random(seed)
    pick = lambda xs: rng.sample(xs, max(1, len(xs) // 3)) if xs else []
    return [(pick(us), []), ([], pick(its)), (pick(us), pick(its)), ([], []), (["nobody", "nobody"], ["nothing"])]


def original_lines(data: bytes, users, items) -> list:
    """the line of X of each line of X - E"""
    return [i for i, raw in enumerate(E.export_lines(data)) if not ref_erased(raw, set(users), set(items))]


def check(data: bytes, users, items, window, now):
    events = parsed(data)
    kept = E.clean_kept(events, window, now)
    got, n = E.erase_kept(kept, users, items)
    # the mirror against the restatement
    raws = E.export_lines(data)
    want = [e for e in kept.events if not ref_erased(raws[e.line], set(users), set(items))]
    assert [e.line for e in got.events] == [e.line for e in want] and n == len(kept.events) - len(want)
    assert (got.n_expired, got.n_duplicates, got.dup_times) == (kept.n_expired, kept.n_duplicates, kept.dup_times)
    # consumers: the state of X - E, by the lines of X
    rest = without(data, users, items)
    back = original_lines(data, users, items)
    fresh, _, _ = E.clean_events(parsed(rest), window, now)
    assert [back[e.line] for e in fresh] == [e.line for e in got.events]
    # the line balance
    assert len(events) == len(got.events) + got.n_expired + got.n_duplicates + n
    # write-back: the kept lines, verbatim, are clean_export(X - E); with compression too
    kept_bytes = b"".join(raws[e.line] + b"\n" for e in got.events)
    assert kept_bytes == E.clean_export(rest, window, now)
    assert E.clean_export(kept_bytes, window, now, True) == E.clean_export(rest, window, now, True)
    return got, n


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("window", sorted(WINDOWS))
def test_random_exports(seed, window):
    data = random_export(seed, 400)
    total = 0
    for users, items in id_sets(data, seed):
        _, n = check(data, users, items, WINDOWS[window], NOW)
        total += n
    assert total > 0


@pytest.mark.parametrize("case", sorted(SEAM_CASES))
def test_seam_cases_erase_then_extend(case):
    """erase after A, then extend with B: what (A - E) + B keeps; and extend, then erase: what (A + B) - E keeps"""
    a, b, now1, now2 = SEAM_CASES[case]
    da, db = dump(a), dump(b)
    evs = parsed(da + db)
    for users, items in id_sets(da + db, 1)[:3] + [(["u1"], []), ([], ["i1"]), ([], ["i2"])]:
        for w in (W, E.EventWindow("5 days"), E.EventWindow(None, True)):
            n2 = now2 if w.duration else now1
            kept, n = E.erase_kept(E.clean_kept(evs[:len(a)], w, now1), users, items)
            kept = E.extend_clean(kept, evs[len(a):], w, n2)
            rest_a = without(da, users, items)
            fresh = E.clean_events(parsed(rest_a + db), w, n2)[0]
            back = original_lines(da, users, items) + list(range(len(a), len(a) + len(b)))
            assert [back[e.line] for e in fresh] == [e.line for e in kept.events]
            assert len(evs) == len(kept.events) + kept.n_expired + kept.n_duplicates + n
            # extend, then erase
            both, m = E.erase_kept(E.extend_clean(E.clean_kept(evs[:len(a)], w, now1), evs[len(a):], w, n2), users, items)
            whole = da + db
            fresh = E.clean_events(parsed(without(whole, users, items)), w, n2)[0]
            back = original_lines(whole, users, items)
            assert [back[e.line] for e in fresh] == [e.line for e in both.events]
            assert len(evs) == len(both.events) + both.n_expired + both.n_duplicates + m


@pytest.mark.parametrize("seed", range(3))
def test_two_erases_are_one_erase_of_the_union(seed):
    data = random_export(seed, 400)
    kept = E.clean_kept(parsed(data), W, NOW)
    (u1, i1), (u2, i2) = id_sets(data, seed)[2], id_sets(data, seed + 7)[2]
    once, n = E.erase_kept(kept, u1 + u2, i1 + i2)
    a, n1 = E.erase_kept(kept, u1, i1)
    twice, n2 = E.erase_kept(a, u2, i2)
    assert [e.line for e in twice.events] == [e.line for e in once.events] and n1 + n2 == n


def test_extends_after_an_erase_stay_balanced_and_read_erased_ids_again():
    """ten one-day extends after an erase: each is what a read of X - E plus everything since keeps, and a new line of an
    erased user is read as any other (erasure is not a block list)"""
    events = parsed(random_export(4, 400))
    head = [e for e in events if e.line < 150]
    kept, n = E.erase_kept(E.clean_kept(head, W, NOW), ["u1", "u2"], ["i3"])
    assert n > 0
    data = random_export(4, 400)
    raws = E.export_lines(data)
    for step in range(1, 11):
        lo, hi = 150 + (step - 1) * 25, 150 + step * 25
        now = NOW + step * DAY // 3
        kept = E.extend_clean(kept, events[lo:hi], W, now)
        assert hi == len(kept.events) + kept.n_expired + kept.n_duplicates + n
        rest = without(b"".join(r + b"\n" for r in raws[:150]), ["u1", "u2"], ["i3"]) + b"".join(r + b"\n" for r in raws[150:hi])
        back = original_lines(b"".join(r + b"\n" for r in raws[:150]), ["u1", "u2"], ["i3"]) + list(range(150, hi))
        assert [back[e.line] for e in E.clean_events(parsed(rest), W, now)[0]] == [e.line for e in kept.events]
    assert any(e.entity_id in ("u1", "u2") and e.line >= 150 for e in kept.events)


def test_rule_edges():
    """a targeted $set on an erased target goes; a user $set and an item as a plain entityId stay; ids compare decoded"""
    rows = [
        {"event": "$set", "entityType": "item", "entityId": "i9", "targetEntityType": "item", "targetEntityId": "gone", "properties": {"a": 1}},
        {"event": "$set", "entityType": "user", "entityId": "bot", "properties": {"a": 1}},
        {"event": "view", "entityType": "user", "entityId": "bot", "targetEntityType": "category", "targetEntityId": "c"},
        {"event": "like", "entityType": "item", "entityId": "gone"},
        {"event": "view", "entityType": "user", "entityId": "bot", "targetEntityType": "item", "targetEntityId": "i1"},
        {"event": "$delete", "entityType": "item", "entityId": "gone"},
    ]
    for r in rows:
        r["eventTime"] = "2023-11-14T00:00:00.000Z"
    data = b"".join(json.dumps(r).encode() + b"\n" for r in rows)
    data += b'{"event":"buy","entityType":"user","entityId":"b\\u006ft","targetEntityType":"item","targetEntityId":"i2","eventTime":"2023-11-14T00:00:00.000Z"}\n'
    got, n = check(data, ["bot"], ["gone"], None, NOW)
    assert [e.line for e in got.events] == [1, 2, 3] and n == 4

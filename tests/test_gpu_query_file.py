"""CcoContext.query_file against the host mirror (ur_query.query_file over the same export, index and file): byte-identical
bodies and offsets on the golden file, on seeded files whose lines draw every member with whitespace and member-order
variants, unknown members, nulls, escapes and hostile ids, on a file where every line is its own template, on eventNames
subsets crossing blacklistEvents, on blacklistItems overlapping the user's blacklist, the item and the set around a
warp's width, on more lines than one launch has warps and on an empty file; a homogeneous file against cco_mixed_queries;
the error cases and the line each names."""
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from universal_recommender_b200 import CcoContext
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_query as Q
from conftest import load_golden
from user_query_data import ODD, handmade_export, handmade_params, random_export

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


@pytest.fixture(scope="module")
def hand(ctx):
    log = ctx.read_events(handmade_export(), keep_history=True)
    yield log, E.read_export(handmade_export()), load_golden("item_queries_handmade.json")["index"].encode()
    log.free()


def check(ctx, log, ev, index, text, ap=None, now_ms=NOW, header="{}"):
    data = text.encode("utf-8", "surrogatepass") if isinstance(text, str) else text
    dev = ctx.query_file(log, index, ap or handmade_params(), data, now_ms, header)
    host = Q.query_file(ev, index, ap or handmade_params(), data, now_ms, header)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    return dev


def dump(d, rng=None):
    """one line: the members in a random order with random JSON whitespace around the tokens"""
    if rng is None:
        return json.dumps(d)
    ws = lambda: rng.choice(["", " ", "\t", "  ", "\r"])
    items = list(d.items())
    rng.shuffle(items)
    return ws() + "{" + ",".join(ws() + json.dumps(k) + ws() + ":" + ws() + json.dumps(v, ensure_ascii=rng.random() < 0.5) + ws()
                                 for k, v in items) + "}" + ws()


def test_golden_file(ctx, hand):
    log, ev, index = hand
    fx = load_golden("query_file_handmade.json")
    body, off = check(ctx, log, ev, index, fx["file"], now_ms=fx["now_ms"])
    for r, text in fx["hand"].items():
        assert body[off[int(r)]:off[int(r) + 1]].decode().split("\n")[1] == text
    for ap in (handmade_params(userBias=-1, itemBias=-1), handmade_params(recsModel="collabFiltering", blacklistEvents=["view"])):
        check(ctx, log, ev, index, fx["file"], ap, header='{"index":"urindex"}')


def random_line(rng, users, items, templates):
    d = dict(rng.choice(templates))
    if rng.random() < 0.6:
        d["user"] = rng.choice(users)
    if rng.random() < 0.5:
        d["item"] = rng.choice(items)
    if rng.random() < 0.4:
        d["itemSet"] = [rng.choice(items) for _ in range(rng.randrange(5))]
    if rng.random() < 0.3:
        d["blacklistItems"] = [rng.choice(items) for _ in range(rng.randrange(4))]
    for k in ("item", "num", "dateRange", "eventNames", "fields"):
        if k not in d and rng.random() < 0.1:
            d[k] = None
    if rng.random() < 0.2:
        d["engineInstanceId"] = {"x": [1, "\\u0000", None]}
    if rng.random() < 0.2:
        d["withRanks"] = rng.random() < 0.5
    return d


TEMPLATES = [{}, {"eventNames": ["view"]}, {"eventNames": ["purchase", "view"], "userBias": 2}, {"returnSelf": True, "itemSetBias": 0},
             {"itemSetBias": -1, "itemBias": 3}, {"num": 3, "from": 2}, {"currentDate": "2020-01-01T00:00:00.000Z"},
             {"dateRange": {"name": "dé", "after": "2020"}}, {"fields": [{"name": "categories", "values": ["Tablets", "\"\\"], "bias": 20}]},
             {"fields": [{"name": "c", "values": ["x"], "bias": -1}, {"name": "c", "values": ["y"], "bias": 0}], "itemBias": 1.05}]


def test_seeded_files_handmade(ctx, hand):
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    users = fx["users"] + ["nobody", " "]
    items = fx["items"] + ["Soap", "Tablets", "\"q\\"]
    for seed in range(4):
        rng = random.Random(seed)
        text = "".join(dump(random_line(rng, users, items, TEMPLATES), rng) + "\n" for _ in range(300))
        check(ctx, log, ev, index, text if seed % 2 else text[:-1])


def test_seeded_files_hostile_ids(ctx):
    export = random_export(11, names=("purchase", "view", "category-pref", "other"))
    log = ctx.read_events(export, keep_history=True)
    try:
        ev = E.read_export(export)
        users = sorted({u for u, _, _, _ in ev.events})[:40] + ["u" + "".join(ODD)]
        items = sorted({i for _, _, i, _ in ev.events})[:40] + ["".join(ODD)]
        index = load_golden("item_queries_handmade.json")["index"].encode()
        rng = random.Random(5)
        text = "".join(dump(random_line(rng, users, items, TEMPLATES), rng) + "\n" for _ in range(400))
        check(ctx, log, ev, index, text)
    finally:
        log.free()


def test_every_line_its_own_template(ctx, hand):
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    rng = random.Random(3)
    lines = []
    for r in range(150):
        d = random_line(rng, fx["users"], fx["items"], TEMPLATES)
        d["num"] = 1000 + r
        lines.append(dump(d))
    check(ctx, log, ev, index, "\n".join(lines) + "\n")


def test_event_name_subsets_cross_blacklist_events(ctx, hand):
    log, ev, index = hand
    names = ["purchase", "view", "category-pref"]
    subsets = [[a] for a in names] + [[a, b] for a in names for b in names if a != b] + [names[::-1], ["view", "view"]]
    lines = [json.dumps({"user": u, "eventNames": s}) for s in subsets for u in ("u1", "U 2", "u-3", "u5", "xyz")]
    for black in (None, ["view"], ["purchase", "category-pref"], []):
        check(ctx, log, ev, index, "\n".join(lines), handmade_params(blacklistEvents=black) if black is not None else None)


def test_blacklist_items_overlap_at_warp_lanes(ctx, hand):
    log, ev, index = hand
    u1_black = ["Iphone 6", "Iphone 5", "Iphone 4", "Ipad-retina", "Galaxy"]
    lines = []
    for lane in (0, 31, 32):
        fill = ["f%d" % k for k in range(lane)]
        for shared in u1_black[:2] + ["Surface", "Nexus"]:
            bl = fill + [shared] + ["g%d" % k for k in range(3)] + [shared]
            lines.append(json.dumps({"user": "u1", "item": "Surface", "itemSet": fill[:lane // 2] + ["Nexus", shared], "blacklistItems": bl}))
            lines.append(json.dumps({"item": shared, "itemSet": [shared] * 3, "blacklistItems": bl[::-1], "returnSelf": lane == 31}))
    check(ctx, log, ev, index, "\n".join(lines))


def test_more_lines_than_one_launch_has_warps(ctx, hand):
    log, ev, index = hand
    rng = random.Random(9)
    lines = [json.dumps({"user": rng.choice(["u1", "u-3", "xyz"]), "item": rng.choice(["Galaxy", "Nexus"])} if r % 3 else
                        {"itemSet": ["Galaxy"], "num": 2}) for r in range(12000)]
    body, off = check(ctx, log, ev, index, "\n".join(lines))
    assert len(off) == 12001


def test_empty_file(ctx, hand):
    log, ev, index = hand
    body, off = check(ctx, log, ev, index, b"")
    assert body == b"" and list(off) == [0]
    body, off = ctx.query_file(None, None, handmade_params(), b"", NOW)
    assert body == b"" and list(off) == [0]


def test_homogeneous_file_is_cco_mixed_queries(ctx, hand):
    log, ev, index = hand
    tpl = {"fields": [{"name": "categories", "values": ["Tablets"], "bias": 0}], "blacklistItems": ["Soap", "Galaxy"], "itemSetBias": 2}
    rows = [("u1", "Iphone 4", None), (None, None, ["Galaxy", "Soap"]), ("u-3", None, []), (None, "Galaxy", ["Nexus"]), (None, None, None)]
    lines = [json.dumps(dict(tpl, **{k: v for k, v in zip(("user", "item", "itemSet"), r) if v is not None})) for r in rows]
    got = ctx.query_file(log, index, handmade_params(), ("\n".join(lines) + "\n").encode(), NOW)
    want = ctx.mixed_queries(log, index, handmade_params(), Q.MixedQuery.from_json(tpl), [r[0] for r in rows], [r[1] for r in rows],
                             [r[2] for r in rows], NOW)
    assert got[0] == want[0] and np.array_equal(got[1], want[1])


def test_path_and_entry_point(ctx, hand, tmp_path):
    log, ev, index = hand
    fx = load_golden("query_file_handmade.json")
    p = tmp_path / "queries.json"
    p.write_text(fx["file"])
    want = Q.query_file(ev, index, handmade_params(), fx["file"].encode(), NOW)
    for got in (ctx.query_file(log, index, handmade_params(), str(p), NOW), ur.queries_from_file(p, handmade_export(), index, handmade_params(), NOW, ctx=ctx),
                ur.queries_from_file(memoryview(fx["file"].encode()), log, index, handmade_params(), NOW, ctx=ctx)):
        assert got[0] == want[0] and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("text, log_too, index_too, match", [
    ('{}\n\n{}\n', True, True, "line 1: not a JSON object"),
    ('{}\n{}\n {"item": 1}', True, True, 'line 2: "item" is not a string'),
    ('{}\n{"itemSet": [1]}\n', True, True, 'line 1: "itemSet" is not an array of strings'),
    ('{}\n{"blacklistItems": "a"}\n', True, True, 'line 1: "blacklistItems" is not an array of strings'),
    ('{}\n{"withRanks": 1}\n', True, True, 'line 1: "withRanks" is not true or false'),
    ('{}\n{"user": "a", "x": 1, "user": null}\n', True, True, 'line 1: the member "user" is repeated'),
    ('{}\n{"num": 1.5}\n', True, True, 'line 1: "num" is not an integer'),
    ('{}\n{"user": "a"\n', True, True, "line 1: not one JSON object"),
    ('{}\n{"user": 3}\n', True, True, 'line 1: "user" is not a string'),
    ('{}\n{}\n{"num": 1, "num": 2}\n', True, True, 'line 2: the member "num" is repeated'),
    ('{"item": "x"}\n[1]\n', True, True, "line 1: not a JSON object"),
    ('{}\n{"user": "u1", "eventNames": ["nope"]}\n', True, True, "line 1: key not found: nope"),
    ('{"item": "Galaxy"}\n{"user": "u1"}\n', False, True, "line 1: a row has a user"),
    ('{"user": "u1"}\n{"item": "Galaxy"}\n', True, False, "line 1: a row has an item"),
])
def test_errors_name_the_line(ctx, hand, text, log_too, index_too, match):
    log, ev, index = hand
    for f in (lambda: ctx.query_file(log if log_too else None, index if index_too else None, handmade_params(), text.encode(), NOW),
              lambda: Q.query_file(ev if log_too else None, index if index_too else None, handmade_params(), text.encode(), NOW)):
        with pytest.raises(ValueError, match=match):
            f()


def test_set_without_model_name_names_the_line(ctx, hand):
    log, ev, index = hand
    ap = handmade_params(indicators=None, eventNames=[])
    for f in (ctx.query_file, lambda *a: Q.query_file(ev, *a[1:])):
        with pytest.raises(ValueError, match="line 1: an item-set query needs a model event name"):
            f(log, None, ap, b'{}\n{"itemSet": []}\n', NOW)

"""buildQuery for mixed queries (ur_query.mixed_plan / mixed_queries: a user, an item and an item set in one query) against
the reference's integration-test query derived by hand (tests/golden/mixed_queries_handmade.json), one assertion per quirk,
and a reduction: on the golden templates, a row with exactly one member is the record the user-, item- or item-set-query
mirror writes for it, and a row with no member is an unknown user's user query."""
import json
import os
import subprocess

import pytest

from conftest import ROOT, load_golden
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200 import ur_query as Q
from user_query_data import handmade_export, handmade_params, line

NOW = 1_700_000_000_000
CS = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'


@pytest.fixture(scope="module")
def fx():
    return load_golden("mixed_queries_handmade.json")


@pytest.fixture(scope="module")
def ev():
    return E.read_export(handmade_export())


@pytest.fixture(scope="module")
def index():
    return load_golden("item_queries_handmade.json")["index"].encode()


def rows(ev, index, rs, ap=None, q=None, header="{}"):
    """[(user, item, set)] -> the mirror's records as text, one per row"""
    users, items, sets = [r[0] for r in rs], [r[1] for r in rs], [r[2] for r in rs]
    body, off = Q.mixed_queries(ev, index, ap or handmade_params(), q, users, items, sets, NOW, header)
    assert len(off) == len(rs) + 1 and off[-1] == len(body)
    out = []
    for r in range(len(rs)):
        h, text, tail = body[off[r]:off[r + 1]].decode("utf-8", "surrogatepass").split("\n")
        assert h == header and tail == ""
        json.loads(text)
        out.append(text)
    return out


def one(ev, index, user=None, item=None, item_set=None, ap=None, q=None) -> str:
    return rows(ev, index, [(user, item, item_set)], ap, q)[0]


def bool_of(text):
    return json.loads(text)["query"]["bool"]


def test_integration_test_query_matches_the_hand_derived_one(fx, ev, index):
    assert one(ev, index, "u1", "Iphone 4") == fx["u1_iphone4_default"]
    texts = rows(ev, index, [tuple(r) for r in fx["rows"]])
    assert texts[0] == fx["u1_iphone4_default"]


def test_every_golden_template_is_json_for_every_row(fx, ev, index):
    for ap in (handmade_params(), handmade_params(userBias=-1, itemBias=-1)):
        for tpl in fx["queries"]:
            rows(ev, index, [tuple(r) for r in fx["rows"]], ap, Q.MixedQuery.from_json(tpl), header='{"index":"x"}')


def kinds(clauses):
    """each clause's terms name and values, or 'cs' / 'range'"""
    out = []
    for c in clauses:
        if "terms" in c:
            out.append(next((k, v) for k, v in c["terms"].items() if k != "boost"))
        else:
            out.append("cs" if "match_all" in json.dumps(c) else "range")
    return out


@pytest.mark.parametrize("user_bias", [None, -1])
@pytest.mark.parametrize("item_bias", [None, -1])
def test_should_and_must_order_for_every_bias_sign(ev, index, user_bias, item_bias):
    ap = handmade_params(userBias=user_bias, itemBias=item_bias)
    q = Q.MixedQuery(fields=[Q.Field("color", ["red"], 2), Q.Field("brand", ["A"], -1)], itemSetBias=3)
    b = bool_of(one(ev, index, "u1", "Iphone 4", ["s1", "s2"], ap, q))
    hist = [("purchase", ["Galaxy", "Ipad-retina", "Iphone 4", "Iphone 5", "Iphone 6"]), ("view", ["Soap", "Mobile-acc", "Phones"]),
            ("category-pref", ["tablets", "phones"])]
    sim = [("purchase", ["Iphone 6", "Ipad-retina"]), ("view", ["Soap", "Tablets"]), ("category-pref", ["tablets"])]
    should = ([] if user_bias else hist) + ([] if item_bias else sim) + [("color", ["red"]), ("purchase", ["s1", "s2"]), "cs"]
    must = (hist if user_bias else []) + (sim if item_bias else []) + [("brand", ["A"]), "range", "range"]
    assert kinds(b["should"]) == should
    assert kinds(b["must"]) == must
    for c in b["must"][:-3]:
        assert c["terms"]["boost"] == 0
    assert b["should"][-2]["terms"]["boost"] == 3.0


def test_distinct_across_the_four_sources_keeps_each_first_position():
    # u's blacklisted purchases, latest first: b, a (a also viewed, not blacklisted by view)
    export = "\n".join([line("u", "purchase", "a", 1000), line("u", "purchase", "b", 2000), line("u", "view", "z", 3000)]) + "\n"
    ev = E.read_export(export.encode())
    index = b'{"index":{"_id":"x"}}\n{"purchase":["p"]}\n'
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "purchase"}, {"name": "view"}], "recsModel": "collabFiltering"})
    q = Q.MixedQuery(blacklistItems=["c", "b", "d", "c"])
    ex = lambda t: bool_of(t)["must_not"][0]["ids"]["values"]
    # user x list (b), item x user (a), set x user (b), set x list (c, d), set x item (x), repeats in the set
    assert ex(one(ev, index, "u", "a", ["x", "b", "e", "c", "e", "a"], ap, q)) == ["b", "a", "c", "d", "x", "e"]
    # item x list: not repeated; the set's copy of the item neither
    assert ex(one(ev, index, "u", "d", ["d", "f", "f"], ap, q)) == ["b", "a", "c", "d", "f"]
    # item x set only: the item keeps its place before the set
    assert ex(one(ev, index, "u", "x", ["y", "x"], ap, q)) == ["b", "a", "c", "d", "x", "y"]
    # no user: the list, the item, the set
    assert ex(one(ev, index, None, "x", ["a", "x", "c"], ap, q)) == ["c", "b", "d", "x", "a"]
    # returnSelf: the item is not excluded, but a set element equal to it is
    assert ex(one(ev, index, "u", "x", ["x"], ap, Q.MixedQuery(returnSelf=True))) == ["b", "a", "x"]
    assert ex(one(ev, index, "u", "x", [], ap, Q.MixedQuery(returnSelf=True))) == ["b", "a"]


def test_unknown_user_is_a_row_without_user(ev, index):
    assert one(ev, index, "nobody", "Iphone 4", ["s"]) == one(ev, index, None, "Iphone 4", ["s"])
    t = one(ev, index, "nobody")
    assert '"should":[{"terms":{"purchase":[]}},{"terms":{"view":[]}},{"terms":{"category-pref":[]}},' + CS + "]" in t


def test_missing_document_and_empty_source_write_no_similar_items(ev):
    index = b'{"index":{"_id":"e"}}\n{}\n{"index":{"_id":"n"}}\n{"popRank":1}\n'
    for item in ("missing", "e"):
        b = bool_of(one(ev, index, "u1", item))
        assert len(b["should"]) == 4   # the history and constant_score only
    b = bool_of(one(ev, index, "u1", "n"))   # a source without the names: [] per model name
    assert kinds(b["should"])[3:6] == [("purchase", []), ("view", []), ("category-pref", [])]


def test_absent_set_and_empty_set(ev, index):
    assert '{"terms":{"purchase":[]}},' + CS not in one(ev, index, None, None, None).split('"purchase":[]}},', 1)[1]
    t = one(ev, index, None, None, [])
    assert '{"terms":{"category-pref":[]}},{"terms":{"purchase":[]}},' + CS in t
    assert kinds(bool_of(one(ev, index, None, None, None))["should"]) == [("purchase", []), ("view", []), ("category-pref", []), "cs"]


def test_item_set_bias_zero_drops_the_clause_and_still_excludes_the_set(ev, index):
    for zero in (0, -0.0):
        b = bool_of(one(ev, index, "u1", None, ["s", "Soap"], q=Q.MixedQuery(itemSetBias=zero)))
        assert ("purchase", ["s", "Soap"]) not in kinds(b["should"])
        assert b["must_not"][0]["ids"]["values"][-2:] == ["s", "Soap"]


def test_return_self(ev, index):
    ex = lambda t: bool_of(t)["must_not"][0]["ids"]["values"]
    assert ex(one(ev, index, None, "Nexus")) == ["Nexus"]
    assert ex(one(ev, index, None, "Nexus", q=Q.MixedQuery(returnSelf=True))) == []
    assert ex(one(ev, index, None, "Nexus", ap=handmade_params(returnSelf=True))) == []
    assert ex(one(ev, index, None, "Nexus", ap=handmade_params(returnSelf=True), q=Q.MixedQuery(returnSelf=False))) == ["Nexus"]


def test_reduction_to_the_single_builders(fx, ev, index):
    """rows with one member are the single builders' records; rows with none are an unknown user's user query"""
    users, items, sets = ["u1", "U 2", "xyz", "u5"], ["Iphone 4", "Nexus", "xyz", ""], [["Iphone 6", "Soap", "Iphone 6"], [], ["x"]]
    for ap in (handmade_params(), handmade_params(userBias=-1, itemBias=-1, recsModel="collabFiltering")):
        for tpl in fx["queries"]:
            q = Q.MixedQuery.from_json(tpl)
            try:
                Q.plan(ap, q, NOW)
            except KeyError:   # a query event name without limits: no user column here
                with pytest.raises(KeyError):
                    Q.mixed_queries(ev, index, ap, q, users, None, None, NOW)
                assert Q.mixed_queries(None, index, ap, q, None, items, None, NOW)[0] == Q.item_queries(index, ap, q, items, NOW)[0]
                continue
            assert Q.mixed_queries(ev, None, ap, q, users, None, None, NOW)[0] == Q.user_queries(ev, ap, q, users, NOW)[0]
            assert Q.mixed_queries(None, index, ap, q, None, items, None, NOW)[0] == Q.item_queries(index, ap, q, items, NOW)[0]
            assert Q.mixed_queries(None, None, ap, q, None, None, sets, NOW)[0] == Q.item_set_queries(sets, ap, q, NOW)[0]
            n = len(users)
            assert (Q.mixed_queries(ev, index, ap, q, [None] * n, [None] * n, [None] * n, NOW)[0]
                    == Q.user_queries(ev, ap, q, ["no such user"] * n, NOW)[0])
            mixed = Q.mixed_queries(ev, index, ap, q, [users[0], None, None], [None, items[0], None], [None, None, sets[0]], NOW)
            singles = [Q.user_queries(ev, ap, q, users[:1], NOW), Q.item_queries(index, ap, q, items[:1], NOW), Q.item_set_queries(sets[:1], ap, q, NOW)]
            assert mixed[0] == b"".join(s[0] for s in singles)


def test_limits_are_consulted_exactly_when_there_is_a_user_column(ev, index):
    q = Q.MixedQuery(eventNames=["purchase", "nowhere"])
    with pytest.raises(KeyError):
        Q.mixed_plan(handmade_params(), q, NOW, with_limits=True)
    with pytest.raises(KeyError):   # a user column whose rows have no user still consults them
        Q.mixed_queries(ev, index, handmade_params(), q, [None], ["Nexus"], None, NOW)
    body, _ = Q.mixed_queries(None, index, handmade_params(), q, None, ["Nexus"], [["s"]], NOW)   # no user column: not consulted
    assert b'{"terms":{"nowhere":[]}}' in body


def test_the_warning_for_item_sets_mixed_with_users_is_not_an_error(ev, index):
    b = bool_of(one(ev, index, "u1", "Iphone 4", ["AirPods"]))
    assert ("purchase", ["AirPods"]) in kinds(b["should"])


def test_mixed_query_from_json():
    q = Q.MixedQuery.from_json({"user": "u", "item": "i", "itemSet": ["a"], "itemSetBias": 1.5, "itemBias": 2, "returnSelf": True,
                                "userBias": -1, "num": 3, "blacklistItems": ["b"], "eventNames": ["view"]})
    assert (q.itemSetBias, q.itemBias, q.returnSelf, q.userBias, q.num, q.blacklistItems, q.eventNames) == (1.5, 2, True, -1, 3, ["b"], ["view"])
    assert Q.MixedQuery.from_json({}) == Q.MixedQuery()


def test_column_lengths_must_agree(ev, index):
    with pytest.raises(ValueError):
        Q.mixed_queries(ev, index, handmade_params(), None, ["u1"], ["a", "b"], None, NOW)


def test_c_declarations_compile():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "mixed_queries_abi_check.c")], check=True)

"""buildQuery for item-set queries (ur_query.item_set_plan / item_set_queries) against query strings derived by hand from
the reference's Scala code, on the sets of examples/multi-query-handmade-item-sets.sh (tests/golden/
item_set_queries_handmade.json), one assertion per quirk."""
import json
import os
import subprocess

import pytest

from conftest import ROOT, load_golden
from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200 import ur_query as Q
from user_query_data import handmade_params

NOW = 1_700_000_000_000
CS = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'


@pytest.fixture(scope="module")
def fx():
    return load_golden("item_set_queries_handmade.json")


def sets_params(**over):
    return ur.URAlgorithmParams.from_engine_json({**load_golden("item_set_queries_handmade.json")["params"], **over})


def one(item_set, ap=None, q=None) -> str:
    body, off = Q.item_set_queries([item_set], ap or sets_params(), q, NOW)
    header, text, tail = body.decode("utf-8", "surrogatepass").split("\n")
    assert header == "{}" and tail == "" and list(off) == [0, len(body)]
    json.loads(text)
    return text


def bool_of(text):
    return json.loads(text)["query"]["bool"]


def test_last_example_matches_the_hand_derived_query(fx):
    assert one(fx["sets"][-1]) == fx["last_set_default"]
    body, off = Q.item_set_queries(fx["sets"], sets_params(), None, NOW)
    assert len(off) == len(fx["sets"]) + 1
    assert body[off[-2]:off[-1]] == b"{}\n" + fx["last_set_default"].encode() + b"\n"


def test_every_golden_query_is_json_for_every_set(fx):
    for ap in (sets_params(), handmade_params()):
        for tpl in fx["queries"]:
            body, off = Q.item_set_queries(fx["sets"], ap, Q.ItemSetQuery.from_json(tpl), NOW, header='{"index":"x"}')
            for s in range(len(fx["sets"])):
                h, text, tail = body[off[s]:off[s + 1]].decode().split("\n")
                assert h == '{"index":"x"}' and tail == ""
                json.loads(text)


def test_item_set_bias_is_the_query_value_only_and_zero_drops_the_clause():
    s = ["a", "b"]
    clause = '{"terms":{"purchase":["a","b"]'
    assert clause + "]}}" not in one(s) and clause + "}}" in one(s)                                    # None: no boost
    assert clause + ',"boost":1.0}}' in one(s, q=Q.ItemSetQuery(itemSetBias=1))                       # no != 1 test
    assert clause + ',"boost":1.0499999523162842}}' in one(s, q=Q.ItemSetQuery(itemSetBias=1.05))     # Float widened
    assert clause + ',"boost":2.0}}' in one(s, q=Q.ItemSetQuery(itemSetBias=2))
    assert clause + ',"boost":-1.0}}' in one(s, q=Q.ItemSetQuery(itemSetBias=-1))                     # in should, negative
    assert bool_of(one(s, q=Q.ItemSetQuery(itemSetBias=-1)))["should"][1] == {"terms": {"purchase": ["a", "b"], "boost": -1.0}}
    for zero in (0, -0.0):
        t = one(s, q=Q.ItemSetQuery(itemSetBias=zero))
        assert t.startswith('{"from":0,"size":4,"query":{"bool":{"should":[{"terms":{"purchase":[]}},' + CS + "]")
        assert '"must_not":[{"ids":{"values":["a","b"],"boost":0}}]' in t   # the exclusion stays
    assert clause + "}}" in one(s, sets_params(itemBias=3, userBias=2))   # no algorithm-level fallback


def test_an_empty_set_still_writes_the_clause():
    t = one([])
    assert '"should":[{"terms":{"purchase":[]}},{"terms":{"purchase":[]}},' + CS + "]" in t
    assert '"must_not":[{"ids":{"values":[],"boost":0}}]' in t


def test_repeats_are_kept_in_the_clause_and_written_once_in_must_not():
    t = one(["x", "y", "x", "z", "y", "x"])
    assert bool_of(t)["should"][1] == {"terms": {"purchase": ["x", "y", "x", "z", "y", "x"]}}
    assert bool_of(t)["must_not"][0] == {"ids": {"values": ["x", "y", "z"], "boost": 0}}


def test_no_max_query_events_slice_on_the_set():
    ap = sets_params(indicators=None, eventNames=["purchase"], maxQueryEvents=2)
    s = [f"i{k}" for k in range(5)]
    assert bool_of(one(s, ap))["should"][1] == {"terms": {"purchase": s}}


def test_blacklist_items_come_first_each_once_and_set_elements_among_them_are_not_repeated():
    t = one(["b", "x", "a", "x"], q=Q.ItemSetQuery(blacklistItems=["a", "c", "a", "b"]))
    assert bool_of(t)["must_not"][0] == {"ids": {"values": ["a", "c", "b", "x"], "boost": 0}}
    assert bool_of(t)["should"][1] == {"terms": {"purchase": ["b", "x", "a", "x"]}}


def test_the_clause_uses_the_first_model_name_not_the_query_event_names():
    ap = handmade_params()   # model names purchase, view, category-pref
    t = one(["s"], ap, Q.ItemSetQuery(eventNames=["view", "nowhere"]))
    assert '"should":[{"terms":{"view":[]}},{"terms":{"nowhere":[]}},{"terms":{"purchase":["s"]}},' + CS + "]" in t
    t = one(["s"], sets_params(indicators=None, eventNames=["cart", "view"]), Q.ItemSetQuery(eventNames=["view"]))
    assert '"should":[{"terms":{"view":[]}},{"terms":{"cart":["s"]}},' in t


def test_negative_algorithm_user_bias_moves_the_empty_history_to_must_the_set_clause_stays_in_should():
    t = one(["s"], handmade_params(userBias=-1), Q.ItemSetQuery(itemSetBias=3))
    assert ('"should":[{"terms":{"purchase":["s"],"boost":3.0}},' + CS + '],"must":[{"terms":{"purchase":[],"boost":0}},'
            '{"terms":{"view":[],"boost":0}},{"terms":{"category-pref":[],"boost":0}},{"constant_score"') in t
    assert '{"terms":{"purchase":[],"boost":2.0}}' in one(["s"], q=Q.ItemSetQuery(userBias=2))   # the query's user boost


def test_boosted_metadata_sits_between_the_history_and_the_set_clause():
    q = Q.ItemSetQuery(fields=[Q.Field("color", ["red"], 2), Q.Field("brand", ["A"], -1), Q.Field("size", ["L"], 0)])
    b = bool_of(one(["s"], q=q))
    assert b["should"] == [{"terms": {"purchase": []}}, {"terms": {"color": ["red"], "boost": 2.0}}, {"terms": {"purchase": ["s"]}},
                           json.loads(CS)]
    assert b["must"] == [{"terms": {"brand": ["A"], "boost": 0}}]
    assert b["must_not"] == [{"ids": {"values": ["s"], "boost": 0}}, {"terms": {"size": ["L"]}}]


def test_sort_is_empty_under_collab_filtering_and_ranked_otherwise():
    assert one(["s"]).endswith('"sort":[]}')
    assert one(["s"], sets_params(recsModel="all")).endswith('"sort":[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]}')


def test_both_date_filter_forms():
    now = Q.iso_utc(NOW)
    t = one(["s"], handmade_params())
    assert ('"must":[{"constant_score":{"filter":{"range":{"available":{"lte":"' + now + '"}}},"boost":0}},'
            '{"constant_score":{"filter":{"range":{"expires":{"gt":"' + now + '"}}},"boost":0}}]') in t
    t = one(["s"], handmade_params(), Q.ItemSetQuery(dateRange=Q.DateRange("date", before="2020", after="")))
    assert '"must":[{"constant_score":{"filter":{"range":{"date":{"lt":"2020"}}},"boost":0}}]' in t


def test_no_model_event_name_raises():
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": [], "recsModel": "collabFiltering"})
    with pytest.raises(ValueError):
        Q.item_set_queries([["a"]], ap, None, NOW)


def test_item_set_query_from_json():
    q = Q.ItemSetQuery.from_json({"itemSet": ["a"], "itemSetBias": 1.5, "num": 2, "from": 3, "blacklistItems": ["b"], "userBias": -1,
                                  "eventNames": ["view"], "currentDate": "2020", "dateRange": {"name": "d", "after": "x"},
                                  "fields": [{"name": "f", "values": ["v"], "bias": 0}]})
    assert (q.itemSetBias, q.num, q.from_, q.blacklistItems, q.userBias, q.eventNames, q.currentDate) == (1.5, 2, 3, ["b"], -1, ["view"], "2020")
    assert q.dateRange == Q.DateRange("d", None, "x") and q.fields == [Q.Field("f", ["v"], 0.0)]
    assert Q.ItemSetQuery.from_json({}).itemSetBias is None


def test_existing_plans_are_unchanged_by_the_boosted_field():
    ap = handmade_params()
    q = Q.UserQuery(fields=[Q.Field("color", ["red"], 2)])
    p = Q.plan(ap, q, NOW)
    assert p.should == p.boosted + "," + CS and p.boosted == '{"terms":{"color":["red"],"boost":2.0}}'
    assert Q.plan(ap, Q.UserQuery(), NOW).boosted == ""


def test_c_declarations_compile():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "item_set_queries_abi_check.c")], check=True)

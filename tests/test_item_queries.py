"""buildQuery for item queries (ur_query.item_plan / item_queries) against query strings derived by hand from the
reference's Scala code, on the handmade model index (tests/golden/item_queries_handmade.json), one assertion per quirk."""
import json
import os
import subprocess

import pytest

from conftest import ROOT, load_golden
from universal_recommender_b200 import ur_query as Q
from user_query_data import handmade_params

NOW = 1_700_000_000_000
CS = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'
HIST = '{"terms":{"purchase":[]}},{"terms":{"view":[]}},{"terms":{"category-pref":[]}}'


@pytest.fixture(scope="module")
def fx():
    return load_golden("item_queries_handmade.json")


def doc(i, src) -> bytes:
    return (json.dumps({"index": {"_id": i}}) + "\n" + json.dumps(src) + "\n").encode()


def one(index, item, ap=None, q=None) -> str:
    body, off = Q.item_queries(index, ap or handmade_params(), q, [item], NOW)
    header, text, tail = body.decode("utf-8", "surrogatepass").split("\n")
    assert header == "{}" and tail == "" and list(off) == [0, len(body)]
    json.loads(text)
    return text


def bool_of(text):
    return json.loads(text)["query"]["bool"]


def test_iphone4_matches_the_hand_derived_query(fx):
    assert one(fx["index"].encode(), "Iphone 4") == fx["iphone4_default"]


def test_every_golden_query_is_json_for_every_item(fx):
    body = fx["index"].encode()
    for tpl in fx["queries"]:
        q = Q.ItemQuery.from_json(tpl)
        out, off, items = Q.item_queries(body, handmade_params(), q, None, NOW)
        assert items == ["Iphone 6", "Iphone 5", "Iphone 4", "Ipad-retina", "Nexus", "Galaxy", "Surface"]
        out, off = Q.item_queries(body, handmade_params(), q, fx["items"], NOW)
        assert len(off) == len(fx["items"]) + 1
        for r in range(len(fx["items"])):
            h, text, _ = out[off[r]:off[r + 1]].decode().split("\n")
            json.loads(text)


def test_the_mirror_reads_the_index_as_the_rerank_oracle_parses_it(fx):
    import rerank_oracle as ro
    body = fx["index"].encode() + doc("rep", {"purchase": ["a"], "purchase ": 1, "purchase": ["b"]})
    want = [(i, {name: json.loads(v) for _, name, v in ms}) for i, ms in ro.parse_body(body)]
    assert Q.index_documents(body) == want


def test_missing_document_vs_document_without_the_field_vs_empty_source(fx):
    body = doc("none", {}) + doc("bare", {"id": "bare"})
    missing, empty, bare = (one(body, i) for i in ("absent", "none", "bare"))
    assert missing == empty.replace('"none"', '"absent"')   # neither adds a similar-items clause
    assert bool_of(missing)["should"][3] == json.loads(CS)
    assert '"should":[' + HIST + ',{"terms":{"purchase":[]}},{"terms":{"view":[]}},{"terms":{"category-pref":[]}},' + CS in bare
    assert '{"terms":{"purchase":[]}},{"terms":{"view":[]}},{"terms":{"category-pref":[]}},' + CS in one(fx["index"].encode(), "Surface")


def test_slice_keeps_a_list_of_max_query_events_and_cuts_a_longer_one_to_max_minus_one():
    ap = handmade_params(indicators=None, eventNames=["buy"], maxQueryEvents=3)
    body = doc("a", {"buy": ["x1", "x2", "x3"]}) + doc("b", {"buy": ["x1", "x2", "x3", "x4"]})
    assert bool_of(one(body, "a", ap))["should"][1] == {"terms": {"buy": ["x1", "x2", "x3"]}}
    assert bool_of(one(body, "b", ap))["should"][1] == {"terms": {"buy": ["x1", "x2"]}}
    assert bool_of(one(doc("c", {"buy": ["x", "y", "x"]}), "c", ap))["should"][1] == {"terms": {"buy": ["x", "y", "x"]}}   # no distinct


def test_empty_history_per_query_name_in_should_or_must_by_the_algorithm_user_bias(fx):
    body = fx["index"].encode()
    assert one(body, "xyz").startswith('{"from":0,"size":4,"query":{"bool":{"should":[' + HIST + "," + CS + '],"must":[{"constant_score"')
    t = one(body, "xyz", handmade_params(userBias=-1))
    assert '"should":[' + CS + '],"must":[{"terms":{"purchase":[],"boost":0}},{"terms":{"view":[],"boost":0}},' \
           '{"terms":{"category-pref":[],"boost":0}},{"constant_score"' in t
    assert '{"terms":{"purchase":[],"boost":2.0}}' in one(body, "xyz", q=Q.ItemQuery(userBias=2))
    t = one(body, "xyz", handmade_params(maxQueryEvents=2, indicators=None, eventNames=["purchase", "view"]))
    assert '"should":[{"terms":{"purchase":[]}},' + CS in t   # the first maxQueryEvents - 1 names


def test_algorithm_item_bias_moves_similar_items_to_must_the_query_bias_only_changes_the_boost(fx):
    body = fx["index"].encode()
    p = '{"terms":{"purchase":["Iphone 6","Ipad-retina"]'
    assert p + ',"boost":2.0}}' in one(body, "Iphone 4", q=Q.ItemQuery(itemBias=2))
    assert p + ',"boost":1.0499999523162842}}' in one(body, "Iphone 4", q=Q.ItemQuery(itemBias=1.05))
    for b in (1, 0, -3):   # no boost written; the query's bias never moves them
        t = one(body, "Iphone 4", q=Q.ItemQuery(itemBias=b))
        assert '"should":[' + HIST + "," + p + "}}," in t
    assert p + ',"boost":3.0}}' in one(body, "Iphone 4", handmade_params(itemBias=3))
    t = one(body, "Iphone 4", handmade_params(itemBias=-1), Q.ItemQuery(itemBias=5))
    assert '"should":[' + HIST + "," + CS + '],"must":[' + p + ',"boost":0}},{"terms":{"view":["Soap","Tablets"],"boost":0}},' in t


def test_return_self_at_the_query_and_the_algorithm_level(fx):
    body = fx["index"].encode()
    self_out = '"must_not":[{"ids":{"values":["Nexus"],"boost":0}}]'
    assert self_out in one(body, "Nexus")
    assert '"must_not":[{"ids":{"values":[],"boost":0}}]' in one(body, "Nexus", q=Q.ItemQuery(returnSelf=True))
    assert '"must_not":[{"ids":{"values":[],"boost":0}}]' in one(body, "Nexus", handmade_params(returnSelf=True))
    assert self_out in one(body, "Nexus", handmade_params(returnSelf=True), Q.ItemQuery(returnSelf=False))


def test_an_item_inside_blacklist_items_is_written_once(fx):
    t = one(fx["index"].encode(), "Nexus", q=Q.ItemQuery(blacklistItems=["Galaxy", "Nexus", "Galaxy", "Soap"]))
    assert '"must_not":[{"ids":{"values":["Galaxy","Nexus","Soap"],"boost":0}}]' in t
    t = one(fx["index"].encode(), "Nexus", q=Q.ItemQuery(blacklistItems=["Galaxy"]))
    assert '"must_not":[{"ids":{"values":["Galaxy","Nexus"],"boost":0}}]' in t


def test_query_event_names_change_the_history_names_not_the_similar_item_names(fx):
    t = one(fx["index"].encode(), "Nexus", q=Q.ItemQuery(eventNames=["view", "nowhere"]))
    assert ('"should":[{"terms":{"view":[]}},{"terms":{"nowhere":[]}},{"terms":{"purchase":[]}},{"terms":{"view":["Tablets"]}},'
            '{"terms":{"category-pref":["tablets"]}},' + CS) in t


def test_a_repeated_model_field_member_the_last_one_wins():
    body = b'{"index":{"_id":"r"}}\n{"purchase":["old"],"view":[],"purchase":["new","newer"]}\n'
    assert '{"terms":{"purchase":["new","newer"]}}' in one(body, "r")


def test_bad_member_of_a_queried_document_raises_an_unqueried_one_is_accepted():
    body = doc("ok", {"purchase": ["a"]}) + doc("bad", {"purchase": ["a", 1]})
    one(body, "ok")
    with pytest.raises(ValueError, match='document 1: its "purchase" member'):
        one(body, "bad")
    with pytest.raises(ValueError, match="_id of document 0"):
        one(doc("x", {}) + doc("x", {}), "x")


def test_params_parse_the_item_keys():
    ap = handmade_params(itemBias=-2, returnSelf=True)
    assert ap.itemBias == -2 and ap.returnSelf is True
    q = Q.ItemQuery.from_json({"itemBias": 3, "returnSelf": False, "num": 2, "blacklistItems": ["a"]})
    assert (q.itemBias, q.returnSelf, q.num, q.blacklistItems) == (3, False, 2, ["a"])


def test_c_declarations_compile():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "item_queries_abi_check.c")], check=True)

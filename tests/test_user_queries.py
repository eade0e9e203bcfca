"""buildQuery for user queries (ur_query.py) against query strings derived by hand from the reference's Scala code, on the
handmade data (data/sample-handmade-data.txt as an export, examples/handmade-engine.json)."""
import json
import os
import subprocess

import pytest

from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_query as Q
from user_query_data import golden, handmade_export, handmade_params

NOW = 1_700_000_000_000
NOW_ISO = "2023-11-14T22:13:20.000Z"
DATES = ('{"constant_score":{"filter":{"range":{"available":{"lte":"%s"}}},"boost":0}},'
         '{"constant_score":{"filter":{"range":{"expires":{"gt":"%s"}}},"boost":0}}') % (NOW_ISO, NOW_ISO)
CS = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'
SORT = '[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]'


@pytest.fixture(scope="module")
def ev():
    return E.read_export(handmade_export())


def one(ev, user, ap=None, q=None):
    body, off = Q.user_queries(ev, ap or handmade_params(), q, [user], NOW)
    header, text, tail = body.decode().split("\n")
    assert header == "{}" and tail == ""
    json.loads(text)
    return text


def test_u1_matches_the_hand_derived_query(ev):
    assert one(ev, "u1") == golden()["u1_default"]


def test_every_golden_query_is_json_for_every_user(ev):
    g = golden()
    for q in g["queries"]:
        body, off, users = Q.user_queries(ev, handmade_params(), Q.UserQuery.from_json(q), None, NOW)
        assert users[:3] == ["u1", "U 2", "u-3"] and "xyz" not in users
        for r in range(len(users)):
            h, text, _ = body[off[r]:off[r + 1]].decode().split("\n")
            json.loads(text)
        body, off = Q.user_queries(ev, handmade_params(), Q.UserQuery.from_json(q), g["users"], NOW)
        assert len(off) == len(g["users"]) + 1


def test_absent_user_has_empty_history(ev):
    t = one(ev, "xyz")
    assert t.startswith('{"from":0,"size":4,"query":{"bool":{"should":[{"terms":{"purchase":[]}},{"terms":{"view":[]}},'
                        '{"terms":{"category-pref":[]}},' + CS + '],"must":[' + DATES + '],"must_not":[{"ids":{"values":[],"boost":0}}]')


def test_query_field_signs(ev):
    t = one(ev, "xyz", q=Q.UserQuery(fields=[Q.Field("categories", ["Tablets"], -1)]))
    assert '"must":[{"terms":{"categories":["Tablets"],"boost":0}},' + DATES + "]" in t   # query bias < 0: a filter
    t = one(ev, "xyz", q=Q.UserQuery(fields=[Q.Field("categories", ["Tablets"], 20)]))
    assert '{"terms":{"categories":["Tablets"],"boost":20.0}},' + CS in t
    t = one(ev, "xyz", q=Q.UserQuery(fields=[Q.Field("categories", ["Tablets"], 0)]))
    assert '"must_not":[{"ids":{"values":[],"boost":0}},{"terms":{"categories":["Tablets"]}}]' in t


def test_inverted_param_field_signs(ev):
    ap = handmade_params(fields=[{"name": "categories", "values": ["Tablets"], "bias": -1}, {"name": "countries", "values": ["MX"], "bias": 5}])
    t = one(ev, "xyz", ap)
    assert '{"terms":{"categories":["Tablets"],"boost":-1.0}},' + CS in t        # params bias < 0: a boost
    assert '"must":[{"terms":{"countries":["MX"],"boost":0}},' in t              # params bias > 0: a filter


def test_float_boost_text(ev):
    t = one(ev, "xyz", q=Q.UserQuery(fields=[Q.Field("categories", ["Tablets"], 1.05)]))
    assert '"boost":1.0499999523162842}}' in t
    assert Q.jfloat(2) == "2.0" and Q.jfloat(1.05) == "1.0499999523162842"


def test_user_bias_query_level_vs_algorithm_level(ev):
    t = one(ev, "u-4", q=Q.UserQuery(userBias=2))
    assert '{"terms":{"purchase":["Galaxy","Iphone 4","Iphone 5"],"boost":2.0}}' in t
    t = one(ev, "u-4", q=Q.UserQuery(userBias=1))
    assert '{"terms":{"purchase":["Galaxy","Iphone 4","Iphone 5"]}}' in t       # b == 1: no boost
    t = one(ev, "u-4", q=Q.UserQuery(userBias=-3))   # the query's bias never moves history into must
    assert '"should":[{"terms":{"purchase":["Galaxy","Iphone 4","Iphone 5"]}}' in t


def test_negative_algorithm_user_bias_puts_history_in_must(ev):
    t = one(ev, "u-4", handmade_params(userBias=-1))
    assert '"should":[' + CS + '],"must":[{"terms":{"purchase":["Galaxy","Iphone 4","Iphone 5"],"boost":0}},' in t


def test_limit_100_under_event_names_vs_500_under_indicators():
    lines = [json.dumps({"event": "buy", "entityType": "user", "entityId": "u", "targetEntityType": "item", "targetEntityId": f"i{k}",
                         "eventTime": Q.iso_utc(NOW - k * 1000)}) for k in range(600)]
    ev = E.read_export(("\n".join(lines) + "\n").encode())
    for params, n in (({"eventNames": ["buy"]}, 100), ({"indicators": [{"name": "buy"}]}, 500),
                      ({"eventNames": ["buy"], "indicators": [{"name": "buy", "maxItemsPerUser": 7}]}, 100),
                      ({"indicators": [{"name": "buy", "maxItemsPerUser": 7}]}, 7)):
        from universal_recommender_b200 import ur_algorithm as ur
        body, _ = Q.user_queries(ev, ur.URAlgorithmParams.from_engine_json(params), None, ["u"], NOW)
        hist = json.loads(body.decode().split("\n")[1])["query"]["bool"]["should"][0]["terms"]["buy"]
        assert hist == [f"i{k}" for k in range(n - 1, -1, -1)]   # the latest n, oldest first
    with pytest.raises(KeyError):
        Q.plan(ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy"]}), Q.UserQuery(eventNames=["view"]), NOW)


def test_max_query_events_slices_names(ev):
    t = one(ev, "u1", handmade_params(indicators=None, eventNames=["purchase", "view", "category-pref"], maxQueryEvents=2))
    assert '"should":[{"terms":{"purchase":["Galaxy","Ipad-retina","Iphone 4","Iphone 5","Iphone 6"]}},' + CS + "]" in t
    t = one(ev, "u1", handmade_params(indicators=None, eventNames=["purchase", "view"], maxQueryEvents=1))
    assert '"should":[' + CS + "]" in t


def test_blacklist_events(ev):
    t = one(ev, "u1", handmade_params(blacklistEvents=[]))
    assert '"must_not":[{"ids":{"values":[],"boost":0}}]' in t
    t = one(ev, "u1", handmade_params(blacklistEvents=["view", "purchase"]))
    assert ('"values":["Iphone 6","Iphone 5","Iphone 4","Ipad-retina","Phones","Mobile-acc","Galaxy","Soap"],"boost":0}}' in t)
    t = one(ev, "u1", q=Q.UserQuery(blacklistItems=["Nexus", "Galaxy", "Nexus"]))
    assert '"values":["Iphone 6","Iphone 5","Iphone 4","Ipad-retina","Galaxy","Nexus"],"boost":0}}' in t


def test_collab_filtering_sort_is_empty(ev):
    assert one(ev, "u1", handmade_params(recsModel="collabFiltering")).endswith('"sort":[]}')
    assert one(ev, "u1").endswith('"sort":' + SORT + "}")


def test_date_range_and_empty_strings(ev):
    t = one(ev, "xyz", q=Q.UserQuery(dateRange=Q.DateRange("date", before="b", after="a")))
    assert '"must":[{"constant_score":{"filter":{"range":{"date":{"gt":"a","lt":"b"}}},"boost":0}}]' in t
    t = one(ev, "xyz", q=Q.UserQuery(dateRange=Q.DateRange("date", after="")))   # Some(""): defined, bound left out
    assert '"must":[{"constant_score":{"filter":{"range":{"date":{}}},"boost":0}}]' in t
    t = one(ev, "xyz", q=Q.UserQuery(currentDate="2020-01-01T00:00:00.000Z"))
    assert '"lte":"2020-01-01T00:00:00.000Z"' in t and '"gt":"2020-01-01T00:00:00.000Z"' in t


def test_pagination(ev):
    assert one(ev, "u5", q=Q.UserQuery(from_=2, num=2)).startswith('{"from":2,"size":2,"query"')


def test_json4s_escaping():
    assert Q.json_string('a"\\\b\f\n\r\t\x01\x1f\x7f\u0080\u009f  €℀') == \
        '"a\\"\\\\\\b\\f\\n\\r\\t\\u0001\\u001f\x7f\\u0080\\u009f \\u2000\\u20ac℀"'


def test_train_ignores_query_keys():
    ap = handmade_params(blacklistEvents=["view"], maxQueryEvents=3, userBias=-2, fields=[{"name": "a", "values": ["b"], "bias": 1}])
    from universal_recommender_b200 import ur_algorithm as ur
    assert ur._indicator_params(ap, ["purchase", "view"]) == ur._indicator_params(handmade_params(), ["purchase", "view"])


SRC = r'''
#include <stddef.h>
#include "cco_b200.h"
int main(void) {
  cco_user_query_t q = {0};
  char *body = NULL; int64_t len = 0, n = 0, *off = NULL; cco_dictionary_t users;
  cco_event_log_t *log = NULL;
  if (cco_event_log_begin_ex(NULL, 1, NULL, CCO_LOG_KEEP_HISTORY, &log) != CCO_E_INVALID_ARG) return 1;
  if (cco_event_log_user_queries(NULL, NULL, &q, 0, NULL, NULL, &body, &len, &off, &n, &users) != CCO_E_INVALID_ARG) return 2;
  return 0;
}
'''


def test_c_declarations_compile(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "uq.c"
    src.write_text(SRC)
    subprocess.run(["cc", "-std=c99", "-Wall", "-Werror", "-c", "-I", os.path.join(root, "include"), str(src), "-o", str(tmp_path / "uq.o")],
                   check=True)

#!/usr/bin/env python
"""Writes tests/golden/query_file_handmade.json: a batchpredict query file (one Query JSON object per line) made of the
query bodies of the reference's example scripts -- examples/advanced-biz-rules-queries.sh, single-query-eventNames.sh,
multi-query-handmade.sh and multi-query-handmade-item-sets.sh, in that order (three bodies of multi-query-handmade.sh lack
the comma after "user": "u5"; they are written here with it) -- over the handmade data of the mixed-query fixture (the
events of tests/user_query_data.handmade_export and the index of item_queries_handmade.json, read at test time) under
examples/handmade-engine.json, and four records derived by hand from URAlgorithm.scala:
  u-3's events: purchase Surface (twice), view Mobile-acc (three times), category-pref tablets -> history purchase
    [Surface], view [Mobile-acc], category-pref [tablets] in should (userBias unset: no boost); blacklist (purchase, the
    first model name): [Surface]; dates: the available / expire pair at now (2023-11-14T22:13:20.000Z); sort: _score, popRank
  u-3, categories Tablets at bias -1: a filter, {"terms":{"categories":["Tablets"],"boost":0}} first in must (:844-867)
  u-3, categories Tablets at bias 20: a boost, {"terms":{"categories":["Tablets"],"boost":20.0}} in should after the
    history, before the constant_score clause
  u-3, categories Tablets at bias 0: an exclusion, {"terms":{"categories":["Tablets"]}} in must_not after the ids clause
  u1 with eventNames ["purchase"]: only the purchase history (user_queries_handmade.json's u1_default list); the blacklist
    is purchase again, so must_not is unchanged
The strings are written here by hand, not produced by ur_query.
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
NOW = "2023-11-14T22:13:20.000Z"
CS = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'
DATES = ('{"constant_score":{"filter":{"range":{"available":{"lte":"' + NOW + '"}}},"boost":0}},'
         '{"constant_score":{"filter":{"range":{"expires":{"gt":"' + NOW + '"}}},"boost":0}}')
SORT = '"sort":[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]}'
U3_HIST = '{"terms":{"purchase":["Surface"]}},{"terms":{"view":["Mobile-acc"]}},{"terms":{"category-pref":["tablets"]}}'
U3_IDS = '{"ids":{"values":["Surface"],"boost":0}}'


def record(should, must, must_not):
    return ('{"from":0,"size":4,"query":{"bool":{"should":[' + should + '],"must":[' + must + '],"must_not":[' + must_not
            + '],"minimum_should_match":1}},' + SORT)


BIZ = [{"user": "u-3"}] + [{"user": "u-3", "fields": f} for f in [
    [{"name": "categories", "values": ["Tablets"], "bias": -1}],
    [{"name": "categories", "values": ["Tablets"], "bias": 20}],
    [{"name": "categories", "values": ["Tablets"], "bias": 0}],
    [{"name": "categories", "values": ["Tablets"], "bias": 0}, {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 5}],
    [{"name": "categories", "values": ["Tablets", "Samsung"], "bias": 0}, {"name": "categories", "values": ["Phones"], "bias": -1},
     {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 5}],
    [{"name": "categories", "values": ["Tablets", "Samsung"], "bias": 5}, {"name": "categories", "values": ["Phones"], "bias": -1},
     {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 0}]]]
EVENT_NAMES = [{}, {"user": "u1"}, {"user": "u1", "eventNames": ["purchase"]}, {"user": "u1", "eventNames": ["view"]}]
TABLETS = {"name": "categories", "values": ["Tablets"]}
MULTI = ([{"user": u} for u in ("u1", "U 2", "u-3", "u-4", "u5")] + [{"item": i} for i in ("Iphone 4", "Ipad-retina", "Nexus", "Galaxy", "Surface")]
         + [{}, {"user": "xyz"}, {"item": "xyz"}, {"fields": [dict(TABLETS, bias=-1)]}, {"fields": [dict(TABLETS, bias=1.05)]},
            {"fields": [dict(TABLETS, bias=1.05), {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": -1}]},
            {"user": "u1", "item": "Iphone 4"}] + BIZ
         + [{"user": "u5", "from": 0, "num": 5}, {"user": "u5", "from": 0, "num": 2}, {"user": "u5", "from": 2, "num": 2}])
ITEM_SETS = [{"itemSet": s} for s in (["iPhone 6"], ["iPhone 7"], ["iPhone 6p"], ["AirPods"], ["USB type-C cable"], ["iPhone 6 charging cradle"],
                                      ["iPhone earbuds", "iPhone 6 case"])]
QUERIES = BIZ + EVENT_NAMES + MULTI + ITEM_SETS
HAND = {
    "1": record(U3_HIST + "," + CS, '{"terms":{"categories":["Tablets"],"boost":0}},' + DATES, U3_IDS),
    "2": record(U3_HIST + ',{"terms":{"categories":["Tablets"],"boost":20.0}},' + CS, DATES, U3_IDS),
    "3": record(U3_HIST + "," + CS, DATES, U3_IDS + ',{"terms":{"categories":["Tablets"]}}'),
    "9": record('{"terms":{"purchase":["Galaxy","Ipad-retina","Iphone 4","Iphone 5","Iphone 6"]}},' + CS, DATES,
                '{"ids":{"values":["Iphone 6","Iphone 5","Iphone 4","Ipad-retina","Galaxy"],"boost":0}}'),
}


def main():
    assert QUERIES[9] == {"user": "u1", "eventNames": ["purchase"]}
    fx = {"source": "the query bodies of the reference's example scripts as one file; records 1, 2, 3 and 9 derived by hand (see the generator)",
          "now_ms": 1_700_000_000_000, "file": "".join(json.dumps(q) + "\n" for q in QUERIES), "hand": HAND}
    json.dump(fx, open(os.path.join(HERE, "query_file_handmade.json"), "w"), indent=0)
    print("written", os.path.join(HERE, "query_file_handmade.json"))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Writes tests/golden/item_set_queries_handmade.json: the item-set queries of examples/multi-query-handmade-item-sets.sh
(its seven sets transcribed as written, "iPhone 6p" included) under examples/handmade-engine-item-sets.json's algorithm
params, a list of query templates, and the default query of the last set derived by hand from URAlgorithm.scala:
  history: no user, so the one query event name (the model name purchase) writes an empty terms clause in should
    (maxQueryEvents = 100 * 10, userBias unset: no boost)
  the set clause: the first model name, the set as given, no boost (itemSetBias unset)
  should ends in the constant_score clause; must: empty (no fields, no date filter)
  must_not: blacklistItems (none) ++ the set, distinct; sort: [] under recsModel "collabFiltering"
The string is written here by hand, not produced by ur_query.
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))

SETS = [["iPhone 6"], ["iPhone 7"], ["iPhone 6p"], ["AirPods"], ["USB type-C cable"], ["iPhone 6 charging cradle"],
        ["iPhone earbuds", "iPhone 6 case"]]
PARAMS = {"appName": "handmade-item-sets", "indexName": "ur-item-sets-index", "typeName": "items",
          "indicators": [{"name": "purchase"}], "recsModel": "collabFiltering", "num": 4}
QUERIES = [{}, {"itemSetBias": 2}, {"itemSetBias": 1.05}, {"itemSetBias": 0}, {"itemSetBias": -1, "num": 2, "from": 1},
           {"blacklistItems": ["iPhone 6", "AirPods", "iPhone 6"]}, {"userBias": 3, "eventNames": ["view", "purchase"]},
           {"userBias": -1, "itemSetBias": 1},
           {"fields": [{"name": "categories", "values": ["Phones", "Accessories"], "bias": 1.2},
                       {"name": "brand", "values": ["Apple"], "bias": -1}, {"name": "color", "values": ["red"], "bias": 0}]},
           {"dateRange": {"name": "date", "after": "2017-01-01T00:00:00.000Z", "before": "2018-01-01T00:00:00.000Z"}},
           {"currentDate": "2017-06-01T00:00:00.000Z"}]
LAST_SET_DEFAULT = ('{"from":0,"size":4,"query":{"bool":{"should":[{"terms":{"purchase":[]}},'
                    '{"terms":{"purchase":["iPhone earbuds","iPhone 6 case"]}},{"constant_score":{"filter":{"match_all":{}},"boost":0}}],'
                    '"must":[],"must_not":[{"ids":{"values":["iPhone earbuds","iPhone 6 case"],"boost":0}}],"minimum_should_match":1}},'
                    '"sort":[]}')


def main():
    fx = {"source": "examples/multi-query-handmade-item-sets.sh under examples/handmade-engine-item-sets.json (see the generator)",
          "now_ms": 1_700_000_000_000, "sets": SETS, "params": PARAMS, "queries": QUERIES, "last_set_default": LAST_SET_DEFAULT}
    json.dump(fx, open(os.path.join(HERE, "item_set_queries_handmade.json"), "w"), indent=0)
    print("written", os.path.join(HERE, "item_set_queries_handmade.json"))


if __name__ == "__main__":
    main()

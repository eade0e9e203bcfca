#!/usr/bin/env python
"""Writes tests/golden/user_queries_handmade.json: the user queries of examples/multi-query-handmade.sh (transcribed:
users u1, U 2, u-3, u-4, u5 and the absent xyz; field biases -1, 20, 0, 5; pagination) plus the quirk templates of
tests/test_user_queries.py, and the query of user u1 under examples/handmade-engine.json derived by hand from
data/sample-handmade-data.txt (times as examples/import_handmade.py spaces them, tests/golden/model_handmade.json):
  purchase, latest first: Iphone 6, Iphone 5, Iphone 4, Ipad-retina, Iphone 6, Iphone 5, Iphone 4, Ipad-retina, Galaxy x4
    -> prepended (oldest first) and distinct: Galaxy, Ipad-retina, Iphone 4, Iphone 5, Iphone 6
  view: Phones x6, Mobile-acc, Phones, Mobile-acc, Soap x2 -> Soap, Mobile-acc, Phones
  category-pref: phones x3, tablets -> tablets, phones
  blacklist (purchase), latest first, distinct: Iphone 6, Iphone 5, Iphone 4, Ipad-retina, Galaxy
  dates: availableDateName "available", expireDateName "expires", now 1700000000000 = 2023-11-14T22:13:20.000Z
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
NOW = "2023-11-14T22:13:20.000Z"
U1 = ('{"from":0,"size":4,"query":{"bool":{"should":['
      '{"terms":{"purchase":["Galaxy","Ipad-retina","Iphone 4","Iphone 5","Iphone 6"]}},'
      '{"terms":{"view":["Soap","Mobile-acc","Phones"]}},'
      '{"terms":{"category-pref":["tablets","phones"]}},'
      '{"constant_score":{"filter":{"match_all":{}},"boost":0}}],'
      '"must":[{"constant_score":{"filter":{"range":{"available":{"lte":"' + NOW + '"}}},"boost":0}},'
      '{"constant_score":{"filter":{"range":{"expires":{"gt":"' + NOW + '"}}},"boost":0}}],'
      '"must_not":[{"ids":{"values":["Iphone 6","Iphone 5","Iphone 4","Ipad-retina","Galaxy"],"boost":0}}],'
      '"minimum_should_match":1}},"sort":[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]}')
TABLETS = {"name": "categories", "values": ["Tablets"]}
QUERIES = [
    {},
    {"fields": [dict(TABLETS, bias=-1)]},
    {"fields": [dict(TABLETS, bias=1.05)]},
    {"fields": [dict(TABLETS, bias=20)]},
    {"fields": [dict(TABLETS, bias=0)]},
    {"fields": [dict(TABLETS, bias=0), {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 5}]},
    {"fields": [{"name": "categories", "values": ["Tablets", "Samsung"], "bias": 0}, {"name": "categories", "values": ["Phones"], "bias": -1},
                {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 5}]},
    {"fields": [{"name": "categories", "values": ["Tablets", "Samsung"], "bias": 5}, {"name": "categories", "values": ["Phones"], "bias": -1},
                {"name": "countries", "values": ["Estados Unidos Mexicanos"], "bias": 0}]},
    {"from": 0, "num": 5},
    {"from": 0, "num": 2},
    {"from": 2, "num": 2},
    {"dateRange": {"name": "date", "after": "2023-11-01T00:00:00.000Z", "before": "2023-11-20T00:00:00.000Z"}},
    {"dateRange": {"name": "date", "after": ""}},
    {"currentDate": "2023-11-10T00:00:00.000Z"},
    {"userBias": 2},
    {"userBias": 1.05, "blacklistItems": ["Iphone 4", "Nexus", "Nexus", "Soap"]},
    {"eventNames": ["view", "purchase"]},
]


def main():
    fx = {"source": "examples/multi-query-handmade.sh user queries + quirk templates; u1 derived by hand (see the generator)",
          "now_ms": 1_700_000_000_000, "users": ["u1", "U 2", "u-3", "u-4", "u5", "xyz"], "queries": QUERIES, "u1_default": U1}
    json.dump(fx, open(f"{HERE}/user_queries_handmade.json", "w"), indent=0)
    print("written", f"{HERE}/user_queries_handmade.json")


if __name__ == "__main__":
    main()

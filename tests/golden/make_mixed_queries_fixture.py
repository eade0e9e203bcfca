#!/usr/bin/env python
"""Writes tests/golden/mixed_queries_handmade.json: mixed queries (user, item and item set in one query) over the handmade
data -- the events of tests/user_query_data.handmade_export and the model index of item_queries_handmade.json, both read
at test time -- under examples/handmade-engine.json's algorithm params: rows of every member combination, the query
templates of the user-, item- and item-set-query fixtures plus mixed ones, and the query of the reference's integration
test, {"user": "u1", "item": "Iphone 4"} (examples/multi-query-handmade.sh), derived by hand from URAlgorithm.scala:
  history: u1's three lists, exactly as its user query (user_queries_handmade.json's u1_default): purchase Galaxy,
    Ipad-retina, Iphone 4, Iphone 5, Iphone 6; view Soap, Mobile-acc, Phones; category-pref tablets, phones -- in should
    (userBias unset: no boost)
  similar items: Iphone 4's document, as its item query (item_queries_handmade.json's iphone4_default): purchase Iphone 6,
    Ipad-retina; view Soap, Tablets; category-pref tablets -- in should after the history (itemBias unset: no boost)
  should ends in the constant_score clause; no set clause (no itemSet)
  must: the available / expire pair at now (2023-11-14T22:13:20.000Z)
  must_not: u1's blacklisted purchases, latest first (Iphone 6, Iphone 5, Iphone 4, Ipad-retina, Galaxy), then no
    blacklistItems, then the item itself (returnSelf false): Iphone 4 is already there, so it is not repeated
  sort: _score, then popRank
The string is written here by hand, not produced by ur_query.
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
NOW = "2023-11-14T22:13:20.000Z"
U1_IPHONE4 = ('{"from":0,"size":4,"query":{"bool":{"should":['
              '{"terms":{"purchase":["Galaxy","Ipad-retina","Iphone 4","Iphone 5","Iphone 6"]}},'
              '{"terms":{"view":["Soap","Mobile-acc","Phones"]}},'
              '{"terms":{"category-pref":["tablets","phones"]}},'
              '{"terms":{"purchase":["Iphone 6","Ipad-retina"]}},'
              '{"terms":{"view":["Soap","Tablets"]}},'
              '{"terms":{"category-pref":["tablets"]}},'
              '{"constant_score":{"filter":{"match_all":{}},"boost":0}}],'
              '"must":[{"constant_score":{"filter":{"range":{"available":{"lte":"' + NOW + '"}}},"boost":0}},'
              '{"constant_score":{"filter":{"range":{"expires":{"gt":"' + NOW + '"}}},"boost":0}}],'
              '"must_not":[{"ids":{"values":["Iphone 6","Iphone 5","Iphone 4","Ipad-retina","Galaxy"],"boost":0}}],'
              '"minimum_should_match":1}},"sort":[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]}')
# [user, item, item set]; null: the row does not have the member
ROWS = [["u1", "Iphone 4", None], ["u1", None, None], [None, "Iphone 4", None], [None, None, ["Iphone 6", "Soap"]], [None, None, None],
        ["U 2", "Nexus", ["Galaxy", "Iphone 4", "Galaxy"]], ["u-3", None, []], [None, "Galaxy", ["Galaxy", "Surface"]],
        ["xyz", "xyz", None], ["u5", "Surface", ["Iphone 5", "Iphone 6"]], ["u-4", "Ipad-retina", ["Ipad-retina", "Nexus"]]]
MIXED = [{"itemSetBias": 0}, {"itemSetBias": 2, "returnSelf": True}, {"itemSetBias": -1, "itemBias": 3, "userBias": 2},
         {"blacklistItems": ["Iphone 4", "Galaxy", "Soap", "Iphone 4"], "itemSetBias": 1.05},
         {"returnSelf": True, "blacklistItems": ["Nexus"]}, {"eventNames": ["view"], "itemBias": 0.5}]


def main():
    from make_item_queries_fixture import ITEMS
    from make_item_set_queries_fixture import QUERIES as SET_QUERIES
    from make_user_queries_fixture import QUERIES as USER_QUERIES
    item_queries = json.load(open(os.path.join(HERE, "item_queries_handmade.json")))["queries"]
    queries = list(USER_QUERIES) + [q for q in item_queries if q not in USER_QUERIES] + [q for q in SET_QUERIES if q not in USER_QUERIES] + MIXED
    fx = {"source": "the handmade export and index under examples/handmade-engine.json; u1 + Iphone 4 derived by hand (see the generator)",
          "now_ms": 1_700_000_000_000, "rows": ROWS, "users": ["u1", "U 2", "u-3", "u-4", "u5", "xyz"], "items": ITEMS,
          "queries": queries, "u1_iphone4_default": U1_IPHONE4}
    json.dump(fx, open(os.path.join(HERE, "mixed_queries_handmade.json"), "w"), indent=0)
    print("written", os.path.join(HERE, "mixed_queries_handmade.json"))


if __name__ == "__main__":
    import sys
    sys.path.insert(0, HERE)
    main()

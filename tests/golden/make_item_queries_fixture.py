#!/usr/bin/env python
"""Writes tests/golden/item_queries_handmade.json: the handmade model index and the item queries of
examples/multi-query-handmade.sh (transcribed: items Iphone 4, Ipad-retina, Nexus, Galaxy, Surface and the unknown xyz).
The index is written on the CPU by tests/model_oracle.model_bulk from tests/golden/model_handmade.json's inputs under
examples/handmade-engine.json's parameters (the default popRank ranking, now = the fixture's now_ms), the correlators
trained by the CPU oracle (oracle/), so the GPU tests need neither.  The templates are the user-query fixture's plus the
item-query keys; iphone4_default is the default query of Iphone 4 derived by hand from its document:
  history: no user, so the query event names purchase, view, category-pref each write an empty terms clause in should
  similar items: one clause per model name with the document's list (every list here is shorter than maxQueryEvents =
    (100 + 100 + 100) * 10), no boost (itemBias 1)
  must: the available / expire pair at now; must_not: the item itself (returnSelf false); sort: _score, popRank
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

NOW = "2023-11-14T22:13:20.000Z"
ITEMS = ["Iphone 4", "Ipad-retina", "Nexus", "Galaxy", "Surface", "xyz"]


def hand_query(purchase, view, cat):
    q = lambda xs: "[" + ",".join('"%s"' % x for x in xs) + "]"
    return ('{"from":0,"size":4,"query":{"bool":{"should":['
            '{"terms":{"purchase":[]}},{"terms":{"view":[]}},{"terms":{"category-pref":[]}},'
            '{"terms":{"purchase":' + q(purchase) + '}},{"terms":{"view":' + q(view) + '}},{"terms":{"category-pref":' + q(cat) + '}},'
            '{"constant_score":{"filter":{"match_all":{}},"boost":0}}],'
            '"must":[{"constant_score":{"filter":{"range":{"available":{"lte":"' + NOW + '"}}},"boost":0}},'
            '{"constant_score":{"filter":{"range":{"expires":{"gt":"' + NOW + '"}}},"boost":0}}],'
            '"must_not":[{"ids":{"values":["Iphone 4"],"boost":0}}],'
            '"minimum_should_match":1}},"sort":[{"_score":{"order":"desc"}},{"popRank":{"unmapped_type":"double","order":"desc"}}]}')


def index_body() -> bytes:
    import model_oracle as mo
    from oracle import oracle as orc
    from universal_recommender_b200 import preparator
    from universal_recommender_b200 import ur_model as um
    from user_query_data import handmade_params
    fx = json.load(open(os.path.join(HERE, "model_handmade.json")))
    ap = handmade_params()
    names = ap.model_event_names()
    actions = [(n, [(u, i) for (u, e, i, _) in fx["events"] if e == n]) for n in names]
    prepared = preparator.prepare([(n, p) for n, p in actions if p], fx["min_events_per_user"])
    orc.build()
    mats = [orc.Csr(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    ref = orc.train(mats, [orc.Params(500, 50, None)] * len(mats), 1)
    triples = [(i, f, um.extract_jvalue(f, v)) for i, f, v in um.aggregate_properties((s[0], s[1]) for s in fx["set_events"])]
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    by_name: dict = {}
    for _, e, i, t in fx["events"]:
        by_name.setdefault(e, []).append((i, t))
    rankings = um.rankings_for(um.rankings_params(ap.rankings, names), by_name, fx["now_ms"], names)
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    return mo.model_bulk([(r.row_ptr, r.col_idx) for r in ref], [n for n, _ in prepared], rows, cols, fields,
                         [(i, fields.index(f), um.property_json(v)) for i, f, v in triples],
                         [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings])


def main():
    from make_user_queries_fixture import QUERIES
    body = index_body()
    docs = {json.loads(a)["index"]["_id"]: json.loads(s) for a, s in zip(*[iter(body.decode().split("\n")[:-1])] * 2)}
    hand = (["Iphone 6", "Ipad-retina"], ["Soap", "Tablets"], ["tablets"])   # read off the Iphone 4 document by hand
    assert tuple(docs["Iphone 4"][n] for n in ("purchase", "view", "category-pref")) == tuple(hand)
    fx = {"source": "examples/multi-query-handmade.sh item queries over the handmade model index (see the generator)",
          "now_ms": 1_700_000_000_000, "items": ITEMS, "index": body.decode(),
          "queries": QUERIES + [{"itemBias": 2}, {"itemBias": 0.5, "returnSelf": True}, {"returnSelf": False, "blacklistItems": ["Galaxy"]},
                                {"itemBias": -1, "userBias": 3, "eventNames": ["view"]}],
          "iphone4_default": hand_query(*hand)}
    json.dump(fx, open(os.path.join(HERE, "item_queries_handmade.json"), "w"), indent=0)
    print("written", os.path.join(HERE, "item_queries_handmade.json"))


if __name__ == "__main__":
    main()

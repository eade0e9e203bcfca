"""Inputs of the user-query tests: the handmade data as a PredictionIO export and seeded random exports."""
import json
import os
import random

from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200.ur_query import iso_utc

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ENGINE = {"indicators": [{"name": "purchase"}, {"name": "view", "maxCorrelatorsPerItem": 50},
                             {"name": "category-pref", "maxCorrelatorsPerItem": 50}],
              "availableDateName": "available", "expireDateName": "expires", "dateName": "date", "num": 4,
              "indexName": "urindex"}   # examples/handmade-engine.json's algorithm params


def golden():
    return json.load(open(os.path.join(HERE, "golden", "user_queries_handmade.json")))


def line(user, event, item, t_ms, extra=""):
    return json.dumps({"event": event, "entityType": "user", "entityId": user, "targetEntityType": "item", "targetEntityId": item,
                       "eventTime": iso_utc(t_ms)}, ensure_ascii=False) + extra


def handmade_export() -> bytes:
    fx = json.load(open(os.path.join(HERE, "golden", "model_handmade.json")))
    lines = [line(u, e, i, t) for u, e, i, t in fx["events"]]
    lines += [json.dumps({"event": "$set", "entityType": "item", "entityId": i, "properties": p, "eventTime": iso_utc(t)})
              for i, p, t in fx["set_events"]]
    return ("\n".join(lines) + "\n").encode("utf-8")


def handmade_params(**over):
    return ur.URAlgorithmParams.from_engine_json({**REF_ENGINE, **over})


ODD = ['"', "\\", "\b", "\f", "\n", "\r", "\t", "\x01", "\x1f", "\x7f", "\u0080", "\u009f", " ", " ", "€", "⃿",
       "℀", "\U0001f600", "é", " "]


def random_export(seed: int, n_events: int = 3000, n_users: int = 60, n_items: int = 80, names=("buy", "view", "like", "other")) -> bytes:
    """ids with quotes, backslashes, control bytes, U+0080..U+009F, U+2000..U+20FF and 4-byte UTF-8; eventTime ties within
    and across names; repeated items; heavy users above the per-name limits; a name outside the query names"""
    rng = random.Random(seed)
    mk = lambda p, k: p + "".join(rng.choice(ODD) for _ in range(rng.randrange(3))) + str(k)
    users = [mk("u", k) for k in range(n_users)]
    items = [mk("i", k) for k in range(n_items)]
    base = 1_600_000_000_000
    out = []
    for _ in range(n_events):
        u = users[min(int(rng.expovariate(1 / 8)), n_users - 1)]   # a few heavy users
        it = items[min(int(rng.expovariate(1 / 15)), n_items - 1)]
        out.append(line(u, rng.choice(names), it, base + rng.randrange(40) * 1000))   # many ties
        if rng.random() < 0.05:
            out.append(json.dumps({"event": "rate", "entityType": "user", "entityId": u, "targetEntityType": "movie", "targetEntityId": it,
                                   "eventTime": iso_utc(base)}))
    return ("\n".join(out) + "\n").encode("utf-8")

#!/usr/bin/env python
"""Writes tests/golden/model_*.json, the inputs of the complete-model tests (cco_format_model, ur_model), from the
reference's own data (run where the reference checkout is mounted; the JSON files are committed).

  * events and `$set` properties: data/sample-handmade-data.txt (43 `$set` lines: categories, countries, integer
    defaultRank) and data/sample-rank-data.txt (18 `$set` lines: colours, non-integer defaultRank such as 2.7 and 7.15),
    parsed like examples/import_handmade.py:30-61: "user,event,item" or "item,$set,name:v1:v2..." (defaultRank -> float)
  * event times follow the importers: a fixed "now", every line 0.8 days earlier than the one before
    (examples/import_handmade.py:22-24, 43, 61)
  * ranking configs: the `rankings` of examples/pop-engine.json, trend-engine.json, hot-3-day-engine.json and
    rank/rank-engine.json.  The `random` ranking of rank-engine.json (uniqueRank) is dropped: Random.nextDouble is not
    reproducible, so it is not part of the device model.
"""
import json
import os

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
NOW_MS = 1_700_000_000_000
STEP_MS = 69_120_000   # 0.8 days


def parse(path):
    events, sets = [], []
    for n, line in enumerate(open(path)):
        d = line.rstrip("\r\n").split(",")
        if len(d) < 3:
            continue
        t = NOW_MS - n * STEP_MS
        if d[1] == "$set":
            props = d[2].split(":")
            name = props.pop(0)
            sets.append([d[0], {name: float(props[0]) if name == "defaultRank" else props}, t])
        else:
            events.append([d[0], d[1], d[2], t])
    sets.sort(key=lambda s: s[2])   # event-time order: later sets win
    return events, sets


def rankings_of(path):
    rs = json.load(open(f"{REF}/examples/{path}"))["algorithms"][0]["params"].get("rankings")
    return [r for r in rs if r.get("type") != "random"]


def main():
    configs = {name: rankings_of(name) for name in ("pop-engine.json", "trend-engine.json", "hot-3-day-engine.json", "rank/rank-engine.json")}
    for out, data, engine in (("model_handmade.json", "sample-handmade-data.txt", "handmade-engine.json"),
                              ("model_rank.json", "sample-rank-data.txt", "rank/rank-engine.json")):
        eng = json.load(open(f"{REF}/examples/{engine}"))
        ap = eng["algorithms"][0]["params"]
        events, sets = parse(f"{REF}/data/{data}")
        fx = {"source": f"data/{data} + examples/{engine}, times as examples/import_handmade.py",
              "now_ms": NOW_MS, "event_names": ap.get("eventNames") or eng["datasource"]["params"]["eventNames"],
              "indicators": ap.get("indicators"),
              "min_events_per_user": eng["datasource"]["params"].get("minEventsPerUser"),
              "events": events, "set_events": sets, "rankings": configs}
        json.dump(fx, open(f"{HERE}/{out}", "w"), indent=0)
    print("model fixtures written to", HERE)


if __name__ == "__main__":
    main()

"""An independent restatement of events.clean_export for the tests: it works on json.loads objects, finds expiry and
duplicates itself and applies the fold rules, without going through events.clean_events.  Value texts are re-rendered
with json.dumps, so it holds for exports written by json.dumps with its default separators (as the tests write them)."""
import json

from universal_recommender_b200 import events as E
from universal_recommender_b200.ur_model import duration_ms
from universal_recommender_b200.ur_query import json_string


def _identity(o: dict) -> str:
    tags = o.get("tags")
    props = sorted((k, json.dumps(v)) for k, v in (o.get("properties") or {}).items())
    return json.dumps([o["event"], o["entityType"], o["entityId"], o.get("targetEntityType"), o.get("targetEntityId"),
                       o.get("prId"), json.dumps(tags) if tags is not None else "[]", props])


def _fold(objs: list) -> bytes:
    """objs: (time, line, object) of one entity, sorted"""
    if any(o["event"] == "$set" for _, _, o in objs):
        state = None
        for _, _, o in objs:
            p = o.get("properties") or {}
            if o["event"] == "$set":
                if state is None:
                    state = {}
                for k, v in p.items():
                    state[k] = v   # an existing name keeps its place
            elif state is not None:
                for k in p:
                    state.pop(k, None)
        name, props = "$set", state
    else:
        name, props = "$unset", {}
        for _, _, o in objs:
            props.update(o.get("properties") or {})
    last = objs[-1][2]
    members = ",".join(json_string(k) + ":" + json.dumps(v) for k, v in props.items())
    return ('{"event":%s,"entityType":%s,"entityId":%s,"properties":{%s},"eventTime":%s}\n'
            % (json_string(name), json_string(last["entityType"]), json_string(last["entityId"]), members,
               json.dumps(last["eventTime"]))).encode("utf-8", "surrogatepass")


def clean_ref(data: bytes, window, now_ms, compress: bool) -> bytes:
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    objs = [json.loads(x) for x in lines]
    times = [E.parse_event_time(o["eventTime"]) for o in objs]
    alive = list(range(len(objs)))
    if window is not None and window.duration is not None:
        cutoff = now_ms - duration_ms(window.duration)
        alive = [i for i in alive if times[i] > cutoff or objs[i]["event"] in ("$set", "$unset")]
    if window is not None and window.removeDuplicates:
        best = {}
        for i in alive:
            k = _identity(objs[i])
            if k not in best or (times[i], i) >= (times[best[k]], best[k]):
                best[k] = i
        alive = sorted(best.values())
    groups, pinned = {}, set()
    if compress:
        for i in alive:
            o = objs[i]
            if o["entityType"] != "item":
                continue
            ent = (o["entityType"], o["entityId"])
            if o["event"] == "$delete" or (o["event"] in ("$set", "$unset") and o.get("targetEntityId") is not None):
                pinned.add(ent)
            elif o["event"] in ("$set", "$unset"):
                groups.setdefault(ent, []).append(i)
        groups = {k: g for k, g in groups.items() if k not in pinned and len(g) > 1}
    folded = {i for g in groups.values() for i in g}
    out = [lines[i] + b"\n" for i in alive if i not in folded]
    out += [_fold(sorted((times[i], i, objs[i]) for i in g)) for g in groups.values()]
    return b"".join(out)

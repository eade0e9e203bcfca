"""The references and inputs of the query-builder edge tests, on the CPU: json4s_quote_ref against ur_query.json_string
over every code point, history_ref against ur_query.user_history on every directed history case, and every generated
index body and export accepted (or refused, naming the document) by the host parsers."""
import json
import random

import pytest

from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200 import ur_query as Q
import query_edges_ref as R
import rerank_oracle


def test_quote_every_code_point():
    for lo in range(0, 0x110000, 0x1000):
        chars = [chr(c) for c in range(lo, lo + 0x1000)]
        assert [Q.json_string(ch) for ch in chars] == [R.json4s_quote_ref(ch) for ch in chars], hex(lo)
    assert R.json4s_quote_ref("\u0085\u2000\u20ff\u2100\u009f\u00a0\x7f\x1f") == '"\\u0085\\u2000\\u20ff\u2100\\u009f\u00a0\x7f\\u001f"'
    assert R.json4s_quote_ref('"\\\b\f\n\r\t') == '"\\"\\\\\\b\\f\\n\\r\\t"'


def test_quote_random_strings():
    rng = random.Random(3)
    pools = [(0, 0x30), (0x7e, 0xa2), (0x1ffe, 0x2102), (0xd7ff, 0xe001), (0x10000, 0x110000), (0, 0x110000)]
    for _ in range(3000):
        s = "".join(chr(rng.randrange(*rng.choice(pools))) for _ in range(rng.randrange(40)))
        assert Q.json_string(s) == R.json4s_quote_ref(s)
    strings = R.codepoint_strings() + R.EDGE_STRINGS + R.names64()
    assert all(Q.json_string(s) == R.json4s_quote_ref(s) for s in strings)


def test_codepoint_inputs_cover_the_range():
    strings = R.codepoint_strings()
    joined = "".join(strings)
    assert len(joined) == 0x10FFFF and joined == "".join(map(chr, range(1, 0x110000)))
    assert all(not (0xD800 <= ord(a) <= 0xDBFF and 0xDC00 <= ord(b) <= 0xDFFF) for s in strings for a, b in zip(s, s[1:]))
    assert len(set(strings + R.EDGE_STRINGS)) == len(strings) + len(R.EDGE_STRINGS)
    for s in strings[:50] + R.EDGE_STRINGS:   # both literal forms decode back
        assert json.loads(R.jraw(s)) == s and json.loads(R.jesc(s)) == s


def user_events(ev):
    """events.read_export's training events -> {user: [(name, item, time, line)]}"""
    out = {}
    for line, (u, n, i, t) in enumerate(ev.events):
        out.setdefault(u, []).append((n, i, t, line))
    return out


def history_cases():
    data, engine, names, users = R.history_export()
    yield data, ur.URAlgorithmParams.from_engine_json(engine), Q.UserQuery(), users
    yield data, ur.URAlgorithmParams.from_engine_json(engine), Q.UserQuery(eventNames=names[::-1] + names[:2]), users
    data, engine, names, users = R.names64_export()
    yield data, ur.URAlgorithmParams.from_engine_json(engine), Q.UserQuery(eventNames=names), users
    names = R.names64()
    data = R.codepoint_export(names)
    yield data, ur.URAlgorithmParams.from_engine_json({"eventNames": names, "maxQueryEvents": 100}), Q.UserQuery(), ["u%d" % k for k in range(7)]


def test_history_ref_matches_the_mirror():
    n = 0
    for data, ap, q, users in history_cases():
        p = Q.plan(ap, q, 0)
        p.blacklist_items = ["i1", "out-u-32-33", "i0", "i1"]
        ev = user_events(E.read_export(data))
        for u in users + list(ev):
            mine = ev.get(u, [])
            # user_history takes the user's events of the query names, latest first (as ur_query.user_queries selects them)
            recent = [(name, item) for name, item, _, _ in sorted(mine, key=lambda e: (-e[2], -e[3])) if name in p.names]
            got = Q.user_history(recent, p)
            assert got == R.history_ref(mine, p.names, p.limits, p.blacklist, p.blacklist_items), u
            n += 1
    assert n > 100


def test_history_cases_reach_their_edges():
    data, engine, names, users = R.history_export()
    ev = user_events(E.read_export(data))
    limits = dict(zip(names, R.LIMITS))
    for L, name in zip(R.LIMITS, names):
        for size in (L - 1, L, L + 1):
            assert sum(e[0] == name for e in ev.get("u-%d-%d" % (L, size), [])) == size
    # some user has equal eventTimes on both sides of its limit
    def straddles(mine, name):
        times = sorted((e[2] for e in mine if e[0] == name), reverse=True)
        L = limits[name]
        return len(times) > L and times[L - 1] == times[L]
    assert sum(straddles(mine, n) for mine in ev.values() for n in names) >= 5
    assert all(e[0] == "other" for u in users if u.startswith("only-other") for e in ev[u])
    assert len(R.names64_export()[2]) == 64


def test_generated_index_bodies_are_accepted():
    bodies = [R.codepoint_index(["purchase", "view", "like"])[0], R.array_sweep_index()[0], R.list_index()[0], R.many_index(300)[0]]
    for body in bodies:
        docs = Q.index_documents(body)
        assert [i for i, _ in docs] == [i for i, _ in rerank_oracle.parse_body(body)]
    body, ids, expect = R.array_sweep_index()
    assert {i: {k: v for k, v in s.items()} for i, s in Q.index_documents(body)} == expect
    body, ids, expect = R.list_index()
    for i, src in Q.index_documents(body):
        if expect[i] is None:
            assert src == {}
        else:
            assert {n: src.get(n, []) for n in ("purchase", "view")} == expect[i]
    body, ids, expect = R.codepoint_index(["purchase", "view", "like"])
    assert [i for i, _ in Q.index_documents(body)] == ids
    assert all(src == expect[i] for i, src in Q.index_documents(body))


def test_generated_exports_are_accepted():
    for data in (R.history_export()[0], R.names64_export()[0], R.codepoint_export(R.names64()), R.many_export(500, 3000)):
        assert len(E.read_export(data).events) == data.count(b"\n")


@pytest.mark.parametrize("form,valid", R.MALFORMED)
def test_malformed_values_are_refused_by_the_mirror(form, valid):
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["purchase", "view"]})
    for at in (0, 17, 39):
        body = R.malformed_index(form, at, 5)
        with pytest.raises(ValueError) as e:
            Q.item_queries(body, ap, None, None, 0)
        if valid:
            assert f'document {at}: its "view" member is not an array of strings' in str(e.value)
        else:
            assert isinstance(e.value, json.JSONDecodeError)

"""A batchpredict query file (ur_query.query_file: one Query JSON object per line, each with its own template): the
extraction rules of json4s' extract[Query] as ur_query.parse_query_line restates them, the records derived by hand from
the reference's example queries (tests/golden/query_file_handmade.json), and a homogeneous file against
ur_query.mixed_queries with that template."""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_golden
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_query as Q
from user_query_data import handmade_export, handmade_params

NOW = 1_700_000_000_000


@pytest.fixture(scope="module")
def ev():
    return E.read_export(handmade_export())


@pytest.fixture(scope="module")
def index():
    return load_golden("item_queries_handmade.json")["index"].encode()


def records(body, off):
    return [body[off[r]:off[r + 1]].decode("utf-8", "surrogatepass").split("\n")[1] for r in range(len(off) - 1)]


def run(ev, index, text, ap=None):
    return Q.query_file(ev, index, ap or handmade_params(), text.encode("utf-8", "surrogatepass"), NOW)


def parse(line):
    return Q.parse_query_line(line.encode("utf-8", "surrogatepass"), 7)


def test_hand_derived_records(ev, index):
    fx = load_golden("query_file_handmade.json")
    body, off = Q.query_file(ev, index, handmade_params(), fx["file"].encode(), fx["now_ms"])
    recs = records(body, off)
    assert len(recs) == fx["file"].count("\n")
    for r, text in fx["hand"].items():
        assert recs[int(r)] == text


def test_every_line_is_its_one_row_mixed_query(ev, index):
    fx = load_golden("query_file_handmade.json")
    body, off = Q.query_file(ev, index, handmade_params(), fx["file"].encode(), NOW)
    for r, line in enumerate(fx["file"].splitlines()):
        d = json.loads(line)
        b1, o1 = Q.mixed_queries(ev, index, handmade_params(), Q.MixedQuery.from_json(d), None if "user" not in d else [d["user"]],
                                 None if "item" not in d else [d["item"]], [d.get("itemSet")], NOW)
        assert body[off[r]:off[r + 1]] == b1


def test_homogeneous_file_is_mixed_queries(ev, index):
    tpl = {"fields": [{"name": "categories", "values": ["Tablets"], "bias": 20}], "returnSelf": True, "itemSetBias": 2, "num": 7}
    rows = [("u1", None, None), (None, "Iphone 4", None), (None, None, ["Galaxy", "Soap"]), ("u-3", "Galaxy", ["Galaxy"])]
    lines = []
    for u, i, s in rows:
        d = dict(tpl)
        d.update({k: v for k, v in (("user", u), ("item", i), ("itemSet", s)) if v is not None})
        lines.append(json.dumps(d))
    got = run(ev, index, "\n".join(lines) + "\n")
    want = Q.mixed_queries(ev, index, handmade_params(), Q.MixedQuery.from_json(tpl), [r[0] for r in rows], [r[1] for r in rows],
                           [r[2] for r in rows], NOW)
    assert got[0] == want[0] and np.array_equal(got[1], want[1])


def test_lines_final_newline_crlf_and_empty_file(ev, index):
    assert Q.query_file_lines(b"") == []
    assert Q.query_file_lines(b"{}\n") == [b"{}"]
    assert Q.query_file_lines(b"{}\n{}") == [b"{}", b"{}"]
    a = run(ev, index, '{"user":"u1"}\n')
    assert run(ev, index, '{"user":"u1"}')[0] == a[0]
    assert run(ev, index, ' \t{"user":"u1"} \r\n')[0] == a[0]
    body, off = run(ev, index, "")
    assert body == b"" and list(off) == [0]


@pytest.mark.parametrize("text", ["", " ", "\r", " \t "])
def test_empty_or_blank_line_is_an_error(ev, index, text):
    with pytest.raises(ValueError, match="line 1: not a JSON object"):
        run(ev, index, "{}\n" + text + "\n{}\n")


@pytest.mark.parametrize("text, what", [
    ("[]", "not a JSON object"), ('"u1"', "not a JSON object"), ("{", "not one JSON object"), ('{"user":"u1"} {}', "not one JSON object"),
    ('{"num": NaN}', "not one JSON object"), ('{"user": 1}', '"user" is not a string'), ('{"item": ["a"]}', '"item" is not a string'),
    ('{"currentDate": 5}', '"currentDate" is not a string'), ('{"itemSet": "a"}', '"itemSet" is not an array of strings'),
    ('{"blacklistItems": [1]}', '"blacklistItems" is not an array of strings'), ('{"eventNames": [null]}', '"eventNames" is not an array'),
    ('{"userBias": "1"}', '"userBias" is not a number'), ('{"itemBias": true}', '"itemBias" is not a number'),
    ('{"itemSetBias": []}', '"itemSetBias" is not a number'), ('{"num": 1.0}', '"num" is not an integer'),
    ('{"from": 1e2}', '"from" is not an integer'), ('{"num": 2147483648}', '"num" is outside the Int32 range'),
    ('{"from": -2147483649}', '"from" is outside the Int32 range'), ('{"returnSelf": 1}', '"returnSelf" is not true or false'),
    ('{"withRanks": "yes"}', '"withRanks" is not true or false'), ('{"fields": {}}', '"fields" is not an array'),
    ('{"fields": [{"name": "c", "values": ["x"]}]}', '"fields" element'), ('{"fields": [{"name": "c", "values": "x", "bias": 1}]}', "fields.values"),
    ('{"fields": [{"name": "c", "values": ["x"], "bias": null}]}', '"fields" element'), ('{"dateRange": {"after": "x"}}', '"dateRange" is not'),
    ('{"dateRange": {"name": "d", "before": 3}}', "dateRange.before"), ('{"user": "a", "user": "b"}', '"user" is repeated'),
    ('{"num": 1, "x": 0, "num": null}', '"num" is repeated'), ('{"withRanks": true, "withRanks": true}', '"withRanks" is repeated'),
])
def test_extraction_errors_name_the_line_and_member(text, what):
    with pytest.raises(ValueError, match="line 7: .*" + __import__("re").escape(what)):
        parse(text)


def test_null_is_absent_and_unknown_members_are_ignored():
    plain = parse('{"user": "u1"}')
    for text in ['{"user": "u1", "item": null, "itemSet": null, "fields": null, "num": null, "dateRange": null, "userBias": null}',
                 '{"user": "u1", "engineInstanceId": 3, "x": {"y": [1, 2]}, "withRanks": true}', '{"user": "u1", "x": 1, "x": 2}']:
        key, q, u, it, s = parse(text)
        assert (key, q, u, it, s) == plain


def test_member_values():
    key, q, u, it, s = parse('{"user": "\\u00e9", "item": "i", "itemSet": [], "blacklistItems": ["a", "a"], "userBias": 1.05, '
                             '"itemBias": -3, "itemSetBias": 0, "num": -2147483648, "from": 2147483647, "returnSelf": false, '
                             '"eventNames": ["view"], "currentDate": "2020", "dateRange": {"name": "d", "after": "x", "before": null}, '
                             '"fields": [{"name": "c", "values": ["v"], "bias": 20, "extra": 1}]}')
    assert (u, it, s) == ("é", "i", [])
    assert q.blacklistItems == ["a", "a"] and q.userBias == 1.05 and q.itemBias == -3.0 and q.itemSetBias == 0.0
    assert (q.num, q.from_, q.returnSelf, q.eventNames, q.currentDate) == (-2**31, 2**31 - 1, False, ["view"], "2020")
    assert q.dateRange == Q.DateRange("d", None, "x") and q.fields == [Q.Field("c", ["v"], 20.0)]
    # the row members are not part of the template
    assert parse('{"user": "a", "num": 3}')[0] == parse('{"item": "b", "itemSet": ["c"], "num": 3}')[0]
    assert parse('{"num": 3}')[0] != parse('{"num": 4}')[0]


def test_per_line_templates_differ_as_their_members(ev, index):
    text = '{"user":"u1","eventNames":["purchase"]}\n{"user":"u1","eventNames":["view"]}\n{"user":"u1"}\n'
    a, b, c = records(*run(ev, index, text))
    assert '"view"' not in a and '"purchase":[' in a
    assert '{"terms":{"purchase"' not in b and '"view":[' in b
    assert '"purchase":[' in c and '"view":[' in c


def test_limits_and_missing_inputs_name_the_line(ev, index):
    with pytest.raises(ValueError, match="line 1: key not found: nope"):
        run(ev, index, '{"eventNames":["nope"]}\n{"user":"u1","eventNames":["nope"]}\n')
    run(ev, index, '{"eventNames":["nope"]}\n{"item":"Galaxy","eventNames":["nope"]}\n')   # no user: no limits consulted
    with pytest.raises(ValueError, match="line 1: a row has a user"):
        Q.query_file(None, index, handmade_params(), b'{}\n{"user":"u1"}\n', NOW)
    with pytest.raises(ValueError, match="line 2: a row has an item"):
        Q.query_file(ev, None, handmade_params(), b'{}\n{"user":"u1"}\n{"item":"x"}\n', NOW)
    with pytest.raises(ValueError, match="line 0: the available / expire date filter needs now_ms"):
        Q.query_file(ev, index, handmade_params(), b'{}\n', None)
    Q.query_file(ev, index, handmade_params(), b'{"currentDate":"2020-01-01T00:00:00.000Z"}\n', None)


def test_blacklist_items_are_a_row_member():
    a = parse('{"user": "u1", "blacklistItems": ["a"], "num": 3}')
    b = parse('{"user": "u1", "blacklistItems": ["b", "c"], "num": 3}')
    assert a[0] == b[0] and a[1].blacklistItems == ["a"] and b[1].blacklistItems == ["b", "c"]


def test_template_from_key_reads_the_raw_values():
    key = b"\0".join([b'[{"name":"c","values":["v"],"bias":-1}]', b'', b'"2020"', b'true', b'3', b'', b'["view"]', b'2', b'', b'0'])
    q = Q.template_from_key(key, 4)
    assert q.fields == [Q.Field("c", ["v"], -1.0)] and q.currentDate == "2020" and q.returnSelf is True and q.num == 3
    assert q.eventNames == ["view"] and q.userBias == 2.0 and q.itemSetBias == 0.0 and q.from_ is None and q.dateRange is None
    with pytest.raises(ValueError, match='line 4: "num" is not an integer'):
        Q.template_from_key(b"\0\0\0\0" + b"1.5", 4)
    with pytest.raises(ValueError, match='line 4: "fields" is not JSON'):
        Q.template_from_key(b"[1 2]", 4)


def test_c_declarations_compile():
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "query_file_abi_check.c")], check=True)

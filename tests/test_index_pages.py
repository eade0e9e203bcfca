"""The model index read back from Elasticsearch pages (cco_index_pages_*) on the CPU: the host mirror ur_model.index_from_pages
on hand-written pages with literal bodies, every error it raises, and the round trip of model index bodies through seeded
scroll pages, checked against an independent parse (ur_predict.loads keeps member order, repeats and number texts)."""
import os
import random
import subprocess

import pytest

import index_pages_data as D
from conftest import ROOT
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200 import ur_predict as P

SHARDS = '"_shards":{"total":1,"successful":1,"skipped":0,"failed":0}'


def one(page: bytes):
    return um.index_from_pages([page])


# ---- rules, with literal bodies -------------------------------------------------------------------------------------------
def test_es5_total_and_scroll_id():
    page = b'{"_scroll_id":"DnF1ZXJ5\\u0041","took":2,"timed_out":false,' + SHARDS.encode() + \
        b',"hits":{"total":2,"max_score":1.0,"hits":[{"_index":"urindex","_type":"items","_id":"a","_score":1.0,' \
        b'"_source":{"id":"a","purchase":["b","c"]}},{"_index":"urindex","_type":"items","_id":"b","_score":1.0,"_source":{"id":"b"}}]}}'
    body, n, sid, total = um.index_page(page)
    assert body == b'{"index":{"_id":"a"}}\n{"id":"a","purchase":["b","c"]}\n{"index":{"_id":"b"}}\n{"id":"b"}\n'
    assert (n, sid, total) == (2, "DnF1ZXJ5A", 2)


@pytest.mark.parametrize("total,want", [('{"value":3,"relation":"eq"}', 3), ('{"value":10000,"relation":"gte"}', -1),
                                        ('{"relation":"eq","value":7}', 7), ('{"value":3}', 3), ("null", -1), ("1.5", -1)])
def test_es7_total(total, want):
    page = ('{"hits":{"total":%s,"hits":[]}}' % total).encode()
    assert um.index_page(page) == (b"", 0, None, want)


def test_absent_total_and_hits():
    assert um.index_page(b'{"took":1}') == (b"", 0, None, -1)
    assert um.index_page(b'{"hits":{"hits":null}}') == (b"", 0, None, -1)


def test_null_score_extra_members_and_sort():
    page = b'{"hits":{"hits":[{"sort":[3,"x]"],"_score":null,"_source":{"id":"i"},"fields":{"a":[{"b":"}"}]},' \
        b'"_routing":"r","_id":"i","_index":"u"}]},"took":1}'
    assert one(page) == (b'{"index":{"_id":"i"}}\n{"id":"i"}\n', 1, -1)


def test_source_spellings_kept_verbatim():
    src = b'{"id":"x","n":1.0E7,"n":-0,"m":12345678901234567890,"s":"\\u00e9\\u0041\\/\\ud83d\\ude00","e":[],"o":{}}'
    page = b'{"hits":{"hits":[{"_id":"x","_source":' + src + b'}]}}'
    assert one(page)[0] == b'{"index":{"_id":"x"}}\n' + src + b"\n"


def test_whitespace_inside_strings_kept_and_outside_dropped():
    page = b'{\n  "hits" : {\n    "hits" : [ {\n      "_id" : "a b",\n      "_source" : {\n        "id" : "a b",\n' \
        b'        "t" : " x\\t y \\" { ",\n        "l" : [ 1 , 2 ]\r\n      }\n    } ]\n  }\n}\n'
    assert one(page)[0] == b'{"index":{"_id":"a b"}}\n{"id":"a b","t":" x\\t y \\" { ","l":[1,2]}\n'


def test_id_decoded_and_reescaped():
    page = '{"hits":{"hits":[{"_id":"q\\"\\\\\\/\\u0001\\u00e9\\ud83d\\ude00\\ud800","_source":{}}]}}'.encode()
    want = '{"index":{"_id":"q\\"\\\\/\\u0001é\U0001F600'.encode() + b"\xed\xa0\x80" + b'"}}\n{}\n'
    assert one(page)[0] == want


def test_empty_final_page_and_empty_index():
    first = b'{"_scroll_id":"s","hits":{"total":1,"hits":[{"_id":"a","_source":{"id":"a"}}]}}'
    last = b'{"_scroll_id":"s","hits":{"total":1,"hits":[]}}'
    assert um.index_from_pages([first, last]) == (b'{"index":{"_id":"a"}}\n{"id":"a"}\n', 1, 1)
    assert um.index_from_pages([b'{"hits":{"total":0,"hits":[]}}']) == (b"", 0, 0)
    assert um.index_from_pages([]) == (b"", 0, -1)


def test_total_is_the_first_pages():
    p0 = b'{"hits":{"total":{"value":2,"relation":"eq"},"hits":[{"_id":"a","_source":{}}]}}'
    p1 = b'{"hits":{"total":{"value":9,"relation":"gte"},"hits":[{"_id":"b","_source":{}}]}}'
    assert um.index_from_pages([p0, p1])[1:] == (2, 2)


def test_first_of_repeated_page_members():
    page = b'{"hits":{"hits":[{"_id":"a","_source":{"k":1},"_source":{"k":2}}]},"hits":{"hits":[{"_id":"b","_source":{}}]},' \
        b'"_scroll_id":"one","_scroll_id":"two","timed_out":false,"timed_out":true}'
    assert um.index_page(page) == (b'{"index":{"_id":"a"}}\n{"k":1}\n', 1, "one", -1)


# ---- errors -------------------------------------------------------------------------------------------------------------
def hits_page(*hits: str) -> bytes:
    return ('{"hits":{"hits":[' + ",".join(hits) + "]}}").encode("utf-8", "surrogatepass")


@pytest.mark.parametrize("page,msg", [
    (b'{"hits":{"hits":[}}', "page 1, byte 19: unbalanced or mismatched brackets"),
    (b'{"hits":{"hits":[]}}}', "page 1, byte 20: unbalanced or mismatched brackets"),
    (b'{"hits":{"hits":[]}', "page 1, byte 19: unbalanced or mismatched brackets"),
    (b'{"hits":{"hits":[{"_id":"a}]}}', "page 1, byte 30: a string is not closed"),
    (b'{"hits":{"hits":[]}} x', "page 1, byte 20: malformed JSON"),
    (b'{"hits" {"hits":[]}}', "page 1, byte 8: malformed JSON"),
    (b'{"took":tru,"hits":{"hits":[]}}', "page 1, byte 8: malformed JSON"),
    (b'[{"hits":{"hits":[]}}]', "page 1: the top level is not an object"),
    (b'', "page 1: the top level is not an object"),
    (b'{"error":{"root_cause":[],"type":"search_context_missing_exception"},"status":404}',
     "page 1: Elasticsearch returned an error (status 404)"),
    (b'{"error":"gone"}', "page 1: Elasticsearch returned an error"),
    (b'{"timed_out":true,"hits":{"hits":[]}}', "page 1: the search timed out (timed_out is true)"),
    (b'{"_shards":{"total":5,"failed":1},"hits":{"hits":[]}}', "page 1: _shards.failed is not 0"),
    (b'{"hits":{"hits":{}}}', "page 1: hits.hits is neither an array nor absent"),
    (b'{"hits":{"hits":[1]}}', "page 1, byte 17: a hits.hits element is not an object"),
    (hits_page('{"_source":{}}'), "page 1, hit 0: the hit has no string _id"),
    (hits_page('{"_id":"a","_source":{}}', '{"_id":7,"_source":{}}'), "page 1, hit 1: the hit has no string _id"),
    (hits_page('{"_id":"a","_id":"a","_source":{}}'), "page 1, hit 0: a repeated _id"),
    (hits_page('{"_id":"a"}'), "page 1, hit 0: the hit has no _source"),
    (hits_page('{"_id":"a","_source":null}'), "page 1, hit 0: _source is not an object"),
    (hits_page('{"_id":"a","_source":{}}', '{"_id":"b","_source":{"x":"\\q"}}'),
     "page 1, hit 1, byte 69: a _source string holds a bad escape or a raw byte < 0x20"),
    (hits_page('{"_id":"a","_source":{"x":"\x01"}}'), "page 1, hit 0, byte 44: a _source string holds a bad escape or a raw byte < 0x20"),
    (hits_page('{"_id":"a","_source":{"x":"\\u12g4"}}'), "page 1, hit 0, byte 44: a _source string holds a bad escape or a raw byte < 0x20"),
])
def test_errors(page, msg):
    good = b'{"hits":{"hits":[{"_id":"z","_source":{}}]}}'
    with pytest.raises(ValueError) as e:
        um.index_from_pages([good, page])
    assert str(e.value) == msg


def test_hit_structure_before_source_strings():
    page = hits_page('{"_id":"a","_source":{"x":"\\q"}}', '{"_id":"b"}')
    with pytest.raises(ValueError, match="hit 1: the hit has no _source"):
        um.index_page(page)


# ---- round trip ------------------------------------------------------------------------------------------------------------
LAYOUTS = [(h, pretty, es7) for h in (1, 2, 7, 0) for pretty, es7 in ((False, True), (True, False))]


def check_layout(body: bytes, pages: list):
    got, n, total = um.index_from_pages(pages)
    want = D.docs_of(body)
    assert (n, total) == (len(want), len(want))
    have = D.docs_of(got)
    assert [i for i, _ in have] == [i for i, _ in want]
    assert [P.loads(s) for _, s in have] == [P.loads(s) for _, s in want]
    return got


@pytest.mark.parametrize("page_hits,pretty,es7", LAYOUTS)
def test_round_trip_of_the_handmade_model(orc, page_hits, pretty, es7):
    for k, (_, body) in enumerate(D.handmade_bodies(orc)):
        # compact pages give the body back; so do pretty ones, which add whitespace outside strings only
        assert check_layout(body, D.pages_of(body, page_hits, seed=k, pretty=pretty, es7=es7)) == body


@pytest.mark.parametrize("page_hits,pretty,es7", LAYOUTS)
def test_round_trip_of_edge_ids(page_hits, pretty, es7):
    body = D.edge_body(random.Random(5))
    assert check_layout(body, D.pages_of(body, page_hits, seed=page_hits, pretty=pretty, es7=es7)) == body


def test_c_declarations_compile(tmp_path):
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "index_pages_abi_check.c"), "-o", str(tmp_path / "ip.o")], check=True)

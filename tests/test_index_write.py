"""The host side of the model index write (URModel.save -> EsClient.hotSwap) on the CPU: the mapping and _aliases bodies
against the golden bytes of tests/golden/make_index_write_fixture.py, and the mirrors of cco_index_write_* (esFields, the
_bulk request cuts, the reading of _bulk responses) against restatements written here."""
import json

import pytest

from conftest import load_golden
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200.ur_algorithm import URAlgorithmParams


def doc(item: str, source: str) -> bytes:
    return b'{"index":{"_id":' + um.json_string(item).encode("utf-8", "surrogatepass") + b'}}\n' + source.encode("utf-8", "surrogatepass") + b"\n"


def test_mapping_and_alias_bodies_are_the_reference_bytes():
    fx = load_golden("index_write_handmade.json")
    ap = URAlgorithmParams.from_engine_json(fx["algorithm_params"])
    assert ap.typeName == "items" and ap.indexName == "urindex"
    for case in fx["mappings"]:
        assert um.index_mapping(case["fields"], ap, ap.typeName) == case["body"].encode()
    for case in fx["aliases"]:
        assert um.alias_actions(case["alias"], case["new_index"], case["old_index"]) == case["body"].encode()
    assert um.new_index_name("urindex", 1700000000000) == "urindex_1700000000000"


def test_type_name_defaults_to_none():
    assert URAlgorithmParams.from_engine_json({"eventNames": ["purchase"]}).typeName is None


def test_mapping_types_follow_get_mappings_order():
    # a name that is a ranking, an event and a date at once is a date; an event and a ranking, a keyword
    ap = URAlgorithmParams(eventNames=["x", "y"], dateName="x", rankings=[um.RankingParams("y", "popular", ["x"], None, None, "1 day")])
    body = um.index_mapping(["x", "y", "z"], ap, "t").decode()
    assert '"x"    : {      "type": "date"    }' in body
    assert '"y"    : {      "type": "keyword"    }' in body
    ap2 = URAlgorithmParams(eventNames=["x"], rankings=[um.RankingParams("r", "popular", ["x"], None, None, "1 day")])
    assert '"r"    : {      "type": "float"    }' in um.index_mapping(["r"], ap2, "t").decode()


def test_mapping_of_no_fields_holds_only_last():
    ap = URAlgorithmParams(eventNames=["purchase"])
    body = um.index_mapping([], ap, "items").decode()
    assert body.count('"type"') == 1 and '"last"' in body
    assert json.loads(body) == {"mappings": {"items": {"properties": {"last": {"type": "keyword"}}}}}


def fields_restated(body: bytes) -> list:
    """esFields as Spark collects the distinct keys of save's maps, in first-appearance order: every document line's
    decoded member names, then "id" (save adds it to every map)"""
    out = []
    lines = body.split(b"\n")
    for k in range(1, len(lines) - 1, 2):
        for name, _ in json.loads(lines[k], object_pairs_hook=list):
            if name not in out:
                out.append(name)
    if len(lines) > 1 and "id" not in out:
        out.append("id")
    return [json.dumps(n, ensure_ascii=False)[1:-1] for n in out]


FIELD_BODIES = {
    "last and id": doc("a", '{"last":["b"],"id":"a"}') + doc("b", '{"view":["a"],"last":[],"id":"b"}'),
    "escaped spelling": doc("a", '{"a\\u0062":["x"],"purchase":[]}') + doc("b", '{"ab":1,"q\\"r":2}'),
    "no id members": doc("a", '{"purchase":["b"]}') + doc("b", '{"view":["a"],"purchase":[]}'),
    "empty source": doc("a", "{}"),
    "empty body": b"",
}


@pytest.mark.parametrize("name", list(FIELD_BODIES))
def test_index_fields_against_restatement(name):
    body = FIELD_BODIES[name]
    assert um.index_fields(body) == fields_restated(body)


def test_index_fields_spellings():
    assert um.index_fields(FIELD_BODIES["escaped spelling"]) == ["ab", "purchase", 'q\\"r', "id"]
    assert um.index_fields(FIELD_BODIES["no id members"]) == ["purchase", "view", "id"]
    assert um.index_fields(FIELD_BODIES["last and id"]) == ["last", "id", "view"]
    assert um.index_fields(b"") == []


def cuts_restated(sizes, max_docs, max_bytes):
    """requests as lists of document indexes: a new request when the current one is full in documents or would pass
    max_bytes; a document alone may pass it"""
    reqs = []
    for d, sz in enumerate(sizes):
        if reqs and len(reqs[-1]) < max_docs and sum(sizes[e] for e in reqs[-1]) + sz <= max_bytes:
            reqs[-1].append(d)
        else:
            reqs.append([d])
    return reqs


def body_of_sizes(sizes) -> bytes:
    out = b""
    for k, sz in enumerate(sizes):
        head = doc("d%04d" % k, "{}")
        pad = sz - len(head) - len('"p":""')
        assert pad >= 0
        out += doc("d%04d" % k, '{"p":"' + "x" * pad + '"}')
    return out


DOC = len(doc("d0000", '{"p":""}'))
CUT_CASES = [
    ("exactly max_bytes", [DOC + 10, DOC + 10, DOC + 10], 1000, DOC + 10),
    ("max_bytes + 1 alone", [DOC, DOC + 11, DOC], 1000, DOC + 10),
    ("sum lands on the limit", [DOC, DOC + 5, DOC, DOC + 5], 1000, 2 * DOC + 5),
    ("max_docs = 1", [DOC, DOC, DOC], 1, 1 << 20),
    ("max_docs bound", [DOC] * 7, 3, 1 << 20),
    ("zero documents", [], 1000, 1 << 20),
]


@pytest.mark.parametrize("name,sizes,max_docs,max_bytes", CUT_CASES, ids=[c[0] for c in CUT_CASES])
def test_bulk_requests_against_restatement(name, sizes, max_docs, max_bytes):
    body = body_of_sizes(sizes)
    db, bb = um.bulk_requests(body, max_docs, max_bytes)
    want = cuts_restated(sizes, max_docs, max_bytes)
    assert [list(range(db[q], db[q + 1])) for q in range(len(db) - 1)] == want
    offs = [0]
    for sz in sizes:
        offs.append(offs[-1] + sz)
    assert bb == [offs[r[0]] for r in want] + [offs[-1]]
    assert b"".join(body[bb[q]:bb[q + 1]] for q in range(len(bb) - 1)) == body


def test_zero_documents_give_zero_requests():
    assert um.bulk_requests(b"", 1000, 1 << 20) == ([0], [0])


def item(i, status, error=None, es5=False):
    m = {"_index": "urindex_1", "_id": i, "_version": 1, "result": "created", "status": status}
    if es5:
        m.update({"_type": "items", "created": True})
    if error:
        m["error"] = error
    return {"index": m}


def test_bulk_item_statuses_reads_errors():
    err = {"type": "mapper_parsing_exception", "reason": "failed to parse [\"x\"]", "caused_by": {"type": "x", "reason": "y"}}
    resp = json.dumps({"took": 1, "errors": False, "items": [item("a", 201), item("b", 400, err), item("c", 429, {"type": "t"})]})
    assert um.bulk_item_statuses(resp.encode(), ["a", "b", "c"]) == [
        (201, "", ""), (400, "mapper_parsing_exception", 'failed to parse ["x"]'), (429, "t", "")]


@pytest.mark.parametrize("resp,ids,msg", [
    ('{"items":[]}', ["a"], "0 items for 1 documents"),
    ('{"items":[{"index":{"_id":"b","status":201}}]}', ["a"], "not the document's _id"),
    ('{"items":[{"index":{"_id":"a","status":201,"status":201}}]}', ["a"], "a repeated status"),
    ('{"items":[{"index":{"_id":"a"}}]}', ["a"], "has no status"),
    ('{"error":{"type":"x"},"status":413}', ["a"], "error (status 413)"),
    ('{"items":[{"create":{"_id":"a","status":201}}]}', ["a"], "not {"),
])
def test_bulk_item_statuses_errors(resp, ids, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("{", r"\{")):
        um.bulk_item_statuses(resp.encode(), ids)

"""Item properties refreshed in the live index, on the CPU: the host mirror ur_model.refresh_documents against the
invariant that defines it (over seeded random models written by tests/model_oracle.model_bulk), directed cases of the
rule, and the host steps of ur_algorithm.update_index against an Elasticsearch fake kept in this file."""
import json
import random

import numpy as np
import pytest

from model_oracle import model_bulk
from universal_recommender_b200 import ur_algorithm as ua
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200.ur_algorithm import IndexWriteError, URAlgorithmParams

NAMES = ["purchase", "vi\"ew"]
RANKS = ["popRank", "trendRank"]
FIELDS = ["color", "price", "id", "cat\\egory", "new\tfield", "size", "userRank"]
ITEM_CHARS = ["a", "b", "é", "\"", "\\", "\n", "\u2028", "z"]


def docs_of(body: bytes) -> dict:
    """{decoded id: source line bytes} of a bulk body"""
    lines = body.split(b"\n")
    return {json.loads(lines[k])["index"]["_id"]: lines[k + 1] for k in range(0, len(lines) - 1, 2)}


def random_model(seed: int, n_rows: int = 12):
    """(indicators, row_ids, col_ids, rankings) of a random indicator model; ids need escapes"""
    rng = random.Random(seed)
    ids = list(dict.fromkeys("".join(rng.choice(ITEM_CHARS) for _ in range(rng.randint(1, 4))) for _ in range(60)))
    row_ids = ids[:n_rows]
    col_ids = [ids[:30], ids[5:40]]
    indicators = []
    for cols in col_ids:
        rp, ci = [0], []
        for _ in range(n_rows):
            ci += sorted(rng.sample(range(len(cols)), rng.randint(0, 4)))
            rp.append(len(ci))
        indicators.append((np.array(rp, np.int64), np.array(ci, np.int32)))
    rankings = []
    for name, mode in zip(RANKS, ["popular", "trending"]):
        items = [rng.choice(ids) for _ in range(50)]
        times = [rng.randrange(0, 100) for _ in items]
        rankings.append((name, mode, 0, 100, [(items, times)]))
    return indicators, row_ids, col_ids, rankings, ids


def random_props(seed: int, ids, n: int = 40):
    """(item, field, JSON text) triples over ids and FIELDS"""
    rng = random.Random(seed)
    vals = ['"red"', "1.5", "[\"a\",\"b\"]", "true", '"q\\"uote"', "null", '{"k":1}', "-7"]
    return [(rng.choice(ids), rng.choice(FIELDS), rng.choice(vals)) for _ in range(n)]


def by_field(triples):
    """the triples in FIELDS order (stable): first appearance of a field = its index, as model_bulk numbers them"""
    return sorted(triples, key=lambda t: FIELDS.index(t[1]))


def formatted(model, triples) -> bytes:
    indicators, row_ids, col_ids, rankings, _ = model
    return model_bulk(indicators, NAMES, row_ids, col_ids, FIELDS, [(i, FIELDS.index(f), v) for i, f, v in triples], rankings)


def refresh(body, triples, rankings=RANKS):
    return um.refresh_documents(body, NAMES, rankings, [(i, f, um.RawJson(v)) for i, f, v in by_field(triples)])


def check_invariant(model, p, p2):
    old = formatted(model, p)
    want = formatted(model, p2)
    got = refresh(old, p2)
    assert docs_of(got.body) == docs_of(want)
    old_docs, want_docs = docs_of(old), docs_of(want)
    differ = {i for i, s in want_docs.items() if old_docs.get(i) != s}
    assert set(docs_of(got.delta)) == differ
    assert {json.loads(ln)["delete"]["_id"] for ln in got.deletes.split(b"\n")[:-1]} == set(old_docs) - set(want_docs)
    assert got.n_docs == len(want_docs) and got.n_changed + got.n_new == len(differ)
    assert got.n_changed + got.n_deleted + got.n_unchanged == len(old_docs)
    assert got.changed_ids == [i for i in old_docs if i in differ]
    assert got.deleted_ids == [i for i in old_docs if i not in want_docs]
    return got


@pytest.mark.parametrize("seed", range(8))
def test_random_models_meet_the_invariant(seed):
    model = random_model(seed)
    ids = model[4]
    p, p2 = random_props(seed, ids), random_props(seed + 100, ids) + [(f"new{seed}", "size", '"S"')]
    got = check_invariant(model, p, p2)
    assert got.n_changed > 0 and got.n_new > 0 and got.n_deleted > 0


@pytest.mark.parametrize("seed", range(4))
def test_the_same_properties_are_a_fixed_point(seed):
    model = random_model(seed)
    p = random_props(seed, model[4])
    old = formatted(model, p)
    got = refresh(old, p)
    assert got.body == old and got.delta == b"" and got.deletes == b""
    assert (got.n_changed, got.n_new, got.n_deleted, got.n_unchanged) == (0, 0, 0, len(docs_of(old)))


def test_changed_values_new_fields_and_unset_fields():
    model = random_model(1, n_rows=3)
    rows = model[1]
    p = [(rows[0], "color", '"red"'), (rows[1], "price", "1"), (rows[1], "size", '"L"')]
    p2 = [(rows[0], "color", '"blue"'), (rows[0], "price", "2"), (rows[1], "price", "1")]   # changed, new field, size unset
    got = check_invariant(model, p, p2)
    assert got.changed == [0, 1] and got.n_new == 0 and got.n_deleted == 0


def test_deleted_and_new_items_and_fieldless_items():
    model = random_model(2, n_rows=2)
    p = [("gone", "color", '"red"'), ("kept", "id", "null"), ("moved", "price", "3")]
    p2 = [("kept", "color", '"red"'), ("moved", "id", "null"), ("fresh", "size", "4"), ("bare", "id", "null")]
    got = check_invariant(model, p, p2)
    assert "gone" in got.deleted_ids
    assert docs_of(got.body)["moved"] == b'{"id":"moved"}'   # an "id" triple only marks the item
    assert docs_of(got.delta)["bare"] == b'{"id":"bare"}'


def test_a_user_defined_field_is_an_ordinary_property():
    ap = URAlgorithmParams(eventNames=["purchase", "view"], rankings=[
        um.RankingParams("popRank", "popular", ["purchase"], None, None, "1 day"),
        um.RankingParams("userRank", "userDefined", None, None, None, None),
        um.RankingParams(None, "random", None, None, None, None)])
    assert ua._refresh_names(ap) == (["purchase", "view"], ["popRank", "uniqueRank"])
    body = (b'{"index":{"_id":"a"}}\n{"id":"a","purchase":["b"],"userRank":1.0,"popRank":2.0}\n')
    got = um.refresh_documents(body, *ua._refresh_names(ap), [("a", "userRank", 5)])
    assert got.body == b'{"index":{"_id":"a"}}\n{"id":"a","purchase":["b"],"userRank":5,"popRank":2.0}\n'
    model = random_model(3)
    check_invariant(model, random_props(3, model[4]), random_props(4, model[4]) + [(model[1][0], "userRank", "9")])


def test_repeated_and_id_members_follow_json4s():
    body = (b'{"index":{"_id":"a"}}\n{"id":"other","purchase":["x"],"color":"red","purchase":["y"],"popRank":1.0,"popRank":2.0}\n'
            b'{"index":{"_id":"b"}}\n{"color":"red","id":"b"}\n')
    got = um.refresh_documents(body, ["purchase"], ["popRank"], [("a", "color", "red")])
    assert got.body == b'{"index":{"_id":"a"}}\n{"id":"a","purchase":["y"],"color":"red","popRank":2.0}\n'
    assert got.changed == [0] and got.deleted == [1] and got.deletes == b'{"delete":{"_id":"b"}}\n'


def test_escapes_in_ids_names_and_values_are_kept():
    item = 'q"\\\n\u00e9'
    esc = um.json_string(item).encode()
    body = b'{"index":{"_id":' + esc + b'}}\n{"id":' + esc + b',"vi\\"ew":["\\u0041"],"old":"x"}\n'
    got = um.refresh_documents(body, ['vi"ew'], [], [(item, "na\"me", "a\tb")])
    assert got.body == b'{"index":{"_id":' + esc + b'}}\n{"id":' + esc + b',"vi\\"ew":["\\u0041"],"na\\"me":"a\\u0009b"}\n'
    assert got.changed_ids == [item]
    gone = um.refresh_documents(body.replace(b',"vi\\"ew":["\\u0041"]', b""), ['vi"ew'], [], [])
    assert gone.deletes == b'{"delete":{"_id":' + esc + b'}}\n' and gone.deleted_ids == [item]


def test_a_property_named_like_a_correlator_is_refused():
    with pytest.raises(ValueError, match='"purchase" is named like a correlator'):
        um.refresh_documents(b"", ["purchase"], [], [("a", "purchase", "1")])


def test_a_repeated_id_is_refused():
    body = b'{"index":{"_id":"a"}}\n{"id":"a"}\n{"index":{"_id":"a"}}\n{"id":"a"}\n'
    with pytest.raises(ValueError, match="document 1: its _id is the _id of document 0"):
        um.refresh_documents(body, [], [], [])


def test_a_new_item_gets_no_random_rank_until_the_next_calc_pop():
    body = b'{"index":{"_id":"a"}}\n{"id":"a","purchase":[],"uniqueRank":0.5}\n'
    got = um.refresh_documents(body, ["purchase"], ["uniqueRank"], [("b", "color", "red"), ("a", "uniqueRank", 0.1)])
    assert got.body == body + b'{"index":{"_id":"b"}}\n{"id":"b","color":"red"}\n'
    assert got.n_changed == 0 and got.n_new == 1


def test_mapping_additions_type_as_index_mapping():
    ap = URAlgorithmParams(eventNames=["purchase"], availableDateName="available",
                           rankings=[um.RankingParams("popRank", "popular", None, None, None, "1 day")])
    assert json.loads(um.mapping_additions(["available", "popRank", "purchase", "color", "a\\\"b"], ap)) == {"properties": {
        "available": {"type": "date"}, "popRank": {"type": "float"}, "purchase": {"type": "keyword"}, "color": {"type": "keyword"},
        'a"b': {"type": "keyword"}}}


def test_bulk_item_statuses_reads_delete_items():
    resp = b'{"took":1,"errors":false,"items":[{"delete":{"_id":"a","status":200}},{"delete":{"_id":"b","status":404}}]}'
    assert um.bulk_item_statuses(resp, ["a", "b"], action="delete") == [(200, "", ""), (404, "", "")]
    with pytest.raises(ValueError, match='item 0: the item is not {"index":{...}}'):
        um.bulk_item_statuses(resp, ["a", "b"])


# ---- update_index against a fake Elasticsearch --------------------------------------------------------------------------
class FakeES:
    """An Elasticsearch 5 stand-in over one alias: indexes of {id: source}, mappings, and the requests it was sent.
    reject: ids whose first index action is answered 429."""

    def __init__(self, indexes: dict, alias: str = "urindex", type_name: str = "items", reject=()):
        self.docs = {name: dict(d) for name, d in indexes.items()}
        self.alias, self.type = alias, type_name
        self.props = {name: {f: {"type": "keyword"} for src in d.values() for f in json.loads(src)} for name, d in indexes.items()}
        self.reject = set(reject)
        self.log = []

    def __call__(self, method, path, body):
        self.log.append((method, path))
        parts = path.strip("/").split("/")
        if method == "GET" and parts[0] == "_alias":
            names = list(self.docs)
            if not names:
                return 404, b'{"error":"alias [urindex] missing","status":404}'
            return 200, json.dumps({n: {"aliases": {self.alias: {}}} for n in names}).encode()
        index = parts[0]
        if parts[1:] == ["_mapping", self.type]:
            if method == "GET":
                return 200, json.dumps({index: {"mappings": {self.type: {"properties": self.props[index]}}}}).encode()
            self.props[index].update(json.loads(body)["properties"])
            return 200, b'{"acknowledged":true}'
        if parts[1:] == ["_refresh"]:
            return 200, b'{"_shards":{"total":1,"successful":1,"failed":0}}'
        assert method == "POST" and parts[1:] == [self.type, "_bulk"], (method, path)
        lines = bytes(body).split(b"\n")[:-1]
        items, k = [], 0
        while k < len(lines):
            action = json.loads(lines[k])
            kind, meta = next(iter(action.items()))
            i = meta["_id"]
            if kind == "index":
                if i in self.reject:
                    self.reject.discard(i)
                    items.append({"index": {"_id": i, "status": 429, "error": {"type": "es_rejected_execution_exception"}}})
                else:
                    self.docs[index][i] = lines[k + 1].decode("utf-8", "surrogatepass")
                    items.append({"index": {"_id": i, "status": 200}})
                k += 2
            else:
                items.append({"delete": {"_id": i, "status": 200 if self.docs[index].pop(i, None) is not None else 404}})
                k += 1
        return 200, json.dumps({"took": 1, "errors": False, "items": items}).encode()


class HostIndexWrite:
    """CcoContext.index_write restated over the host mirrors (index_fields, bulk_requests, bulk_item_statuses), for the
    host steps of update_index; 429s are not retried here"""

    def __init__(self, body, max_docs, max_bytes):
        self.body, self.docs = body, um.bulk_documents(body)
        self.cut = um.bulk_requests(body, max_docs, max_bytes)
        self.status = [0] * len(self.docs)

    def fields(self):
        return um.index_fields(self.body)

    def requests(self):
        _, bb = self.cut
        return [self.body[bb[q]:bb[q + 1]] for q in range(len(bb) - 1)]

    def response(self, q, resp):
        db, _ = self.cut
        ids = [d[0] for d in self.docs[db[q]:db[q + 1]]]
        for k, (st, _, _) in enumerate(um.bulk_item_statuses(resp, ids)):
            self.status[db[q] + k] = st

    def retry(self):
        return len(self.cut[0]) - 1, []

    def finish(self):
        errors = [(d, "", "") for d, st in enumerate(self.status) if not 200 <= st < 300]
        return type("R", (), {"errors": errors, "n_rejected": sum(st == 429 for st in self.status), "n_failed": 0})()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass


class HostCtx:
    def index_write(self, body, max_docs, max_bytes):
        return HostIndexWrite(body, max_docs, max_bytes)


AP = URAlgorithmParams(eventNames=["purchase"], indexName="urindex", typeName="items",
                       rankings=[um.RankingParams("popRank", "popular", None, None, None, "1 day")])


def live_index():
    body = (b'{"index":{"_id":"a"}}\n{"id":"a","purchase":["b"],"color":"red","popRank":1.0}\n'
            b'{"index":{"_id":"b"}}\n{"id":"b","color":"blue"}\n'
            b'{"index":{"_id":"c"}}\n{"id":"c","purchase":[],"color":"red"}\n')
    return body, {"urindex_1": docs_of(body)}


def test_update_index_sends_the_mapping_the_delta_the_deletes_and_a_refresh():
    body, indexes = live_index()
    es = FakeES({n: {i: s.decode() for i, s in d.items()} for n, d in indexes.items()})
    r = um.refresh_documents(body, ["purchase"], ["popRank"], [("a", "color", "green"), ("a", "price", 3), ("c", "color", "red"),
                                                              ("d", "price", 1)])
    assert r.changed_ids == ["a"] and r.deleted_ids == ["b"] and r.n_new == 1
    r.deletes += b'{"delete":{"_id":"zz"}}\n'   # already gone: 404 is success
    index, _ = ua.update_index(r, AP, es, max_docs=1, ctx=HostCtx())
    assert index == "urindex_1"
    assert es.log == [("GET", "/_alias/urindex"), ("GET", "/urindex_1/_mapping/items"), ("PUT", "/urindex_1/_mapping/items"),
                      ("POST", "/urindex_1/items/_bulk"), ("POST", "/urindex_1/items/_bulk"),
                      ("POST", "/urindex_1/items/_bulk"), ("POST", "/urindex_1/items/_bulk"), ("POST", "/urindex_1/_refresh")]
    assert es.props["urindex_1"]["price"] == {"type": "keyword"}
    assert {i: s.encode() for i, s in es.docs["urindex_1"].items()} == docs_of(r.body)


def test_update_index_without_a_change_sends_no_bulk_request():
    body, indexes = live_index()
    es = FakeES({n: {i: s.decode() for i, s in d.items()} for n, d in indexes.items()})
    r = um.refresh_documents(body, ["purchase"], ["popRank"], [("a", "color", "red"), ("b", "color", "blue"), ("c", "color", "red")])
    assert r.delta == b"" and r.deletes == b""
    ua.update_index(r, AP, es, ctx=HostCtx())
    assert es.log == [("GET", "/_alias/urindex"), ("GET", "/urindex_1/_mapping/items"), ("POST", "/urindex_1/_refresh")]


@pytest.mark.parametrize("indexes", [{}, {"urindex_1": {}, "urindex_2": {}}])
def test_update_index_needs_an_alias_of_exactly_one_index(indexes):
    body, _ = live_index()
    r = um.refresh_documents(body, ["purchase"], ["popRank"], [])
    with pytest.raises(IndexWriteError):
        ua.update_index(r, AP, FakeES(indexes), ctx=HostCtx())


def test_update_index_raises_on_a_failed_delete():
    body, indexes = live_index()
    es = FakeES({n: {i: s.decode() for i, s in d.items()} for n, d in indexes.items()})
    r = um.refresh_documents(body, ["purchase"], ["popRank"], [("a", "color", "red"), ("c", "color", "red")])

    def broken(method, path, data):
        if data and data.startswith(b'{"delete"'):
            return 200, b'{"items":[{"delete":{"_id":"b","status":500}}]}'
        return es(method, path, data)
    with pytest.raises(IndexWriteError, match="1 deletes failed on urindex_1"):
        ua.update_index(r, AP, broken, ctx=HostCtx())


def build_abi_check(tmp_path) -> str:
    import os
    import subprocess
    from conftest import ROOT
    from universal_recommender_b200 import _native
    exe = str(tmp_path / "refresh_properties_abi_check")
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "refresh_properties_abi_check.c"), "-o", exe, "-L", libdir, "-lcco_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_c_program_builds_and_null_arguments_are_refused(tmp_path):
    import subprocess
    assert subprocess.run([build_abi_check(tmp_path)], capture_output=True, text=True, check=True).stdout == "ok\n"

"""cco_index_write on the H100.  Part 1: ur.write_index, hotSwap's whole sequence, against an in-process fake Elasticsearch
(no sockets, no threads): alias swaps, 429 retries, persistent item errors, the request order, and the stored index paged
back through ur.index_from_pages.  Part 2: the device session byte for byte against the ur_model mirrors (index_fields,
bulk_requests, bulk_item_statuses) over model bodies and edge bodies, _bulk responses of ES 5 and ES 8 shapes, and every
documented error."""
import dataclasses
import json
import random

import pytest

import index_pages_data as D
import search_results_data as SD
import universal_recommender_b200 as ur
from test_gpu_event_stream import AP, NOW
from test_gpu_events import random_export
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu

WAP = dataclasses.replace(AP, indexName="urindex", typeName="items")


def bulk_response(ids, statuses, rng, es5=False, pretty=False, errors_flag=None, reasons=None) -> bytes:
    """a _bulk response for the documents `ids`: ES 5 items carry _type and created, ES 8 ones _seq_no; members shuffled"""
    items = []
    for k, (i, st) in enumerate(zip(ids, statuses)):
        m = [('"_index"', '"urindex_1"'), ('"_id"', json.dumps(i, ensure_ascii=rng.random() < 0.5)), ('"status"', str(st))]
        if es5:
            m += [('"_type"', '"items"'), ('"created"', "true" if st == 201 else "false")]
        else:
            m += [('"_seq_no"', str(k)), ('"_primary_term"', "1")]
        if 200 <= st < 300:
            m += [('"_version"', "1"), ('"result"', '"created"'), ('"_shards"', '{"total":2,"successful":1,"failed":0}')]
        else:
            t, r = (reasons or {}).get(i, ("es_rejected_execution_exception" if st == 429 else "mapper_parsing_exception",
                                          "rejected execution of \"bulk\" \\ [x]\n" if st == 429 else "failed to parse [view]"))
            m.append(('"error"', '{"type":%s,"reason":%s,"caused_by":{"type":"illegal_argument_exception","reason":"a\\"b",'
                      '"caused_by":{"type":"x","reason":"y"}},"index":"urindex_1"}' % (json.dumps(t), json.dumps(r))))
        rng.shuffle(m)
        items.append('{"index":{' + ",".join(a + ":" + b for a, b in m) + "}}")
    flag = errors_flag if errors_flag is not None else any(not 200 <= s < 300 for s in statuses)
    top = [('"took"', str(rng.randrange(100))), ('"errors"', "true" if flag else "false"), ('"items"', "[" + ",".join(items) + "]")]
    rng.shuffle(top)
    text = "{" + ",".join(a + ":" + b for a, b in top) + "}"
    return (SD.pretty(text) + "\n" if pretty else text).encode("utf-8", "surrogatepass")


# ---- part 1: write_index against a fake Elasticsearch ---------------------------------------------------------------------
class FakeES:
    """indexes, aliases and _bulk in memory.  reject: {_id: rounds} answered 429 that many times; fail: _ids answered 400
    mapper_parsing_exception every time."""

    def __init__(self, reject=None, fail=(), seed=0, es5=True):
        self.indexes, self.aliases, self.log = {}, {}, []
        self.reject, self.fail, self.rng, self.es5 = dict(reject or {}), set(fail), random.Random(seed), es5

    def __call__(self, method, path, body):
        self.log.append((method, path))
        parts = path.strip("/").split("/")
        if method == "HEAD":
            if parts[0] == "_alias":
                return (200 if parts[1] in self.aliases else 404), b""
            return (200 if parts[0] in self.indexes else 404), b""
        if method == "PUT":
            self.indexes[parts[0]] = {"mapping": json.loads(body), "docs": {}, "order": {}}
            return 200, b'{"acknowledged":true}'
        if method == "POST" and parts[-1] == "_refresh":
            return 200, b'{"_shards":{"total":2,"successful":1,"failed":0}}'
        if method == "POST" and parts[-1] == "_bulk":
            return 200, self.bulk(self.indexes[parts[0]], body)
        if method == "GET" and parts[0] == "_alias":
            return 200, json.dumps({self.aliases[parts[1]]: {"aliases": {parts[1]: {}}}}).encode()
        if method == "POST" and parts[0] == "_aliases":
            for act in json.loads(body)["actions"]:
                if "add" in act:
                    self.aliases[act["add"]["alias"]] = act["add"]["index"]
                if "remove_index" in act:
                    self.indexes.pop(act["remove_index"]["index"], None)
            return 200, b'{"acknowledged":true}'
        if method == "DELETE":
            self.indexes.pop(parts[0])
            return 200, b'{"acknowledged":true}'
        raise AssertionError(f"unexpected {method} {path}")

    def bulk(self, index, body: bytes) -> bytes:
        lines = body.split(b"\n")[:-1]
        ids, statuses = [], []
        for k in range(0, len(lines), 2):
            i = json.loads(lines[k])["index"]["_id"]
            index["order"].setdefault(i, len(index["order"]))
            ids.append(i)
            if i in self.fail:
                statuses.append(400)
            elif self.reject.get(i, 0) > 0:
                self.reject[i] -= 1
                statuses.append(429)
            else:
                index["docs"][i] = lines[k + 1]
                statuses.append(201)
        return bulk_response(ids, statuses, self.rng, es5=self.es5)

    def pages(self, alias: str, page_hits: int) -> list:
        """the alias's index as a scroll returns it, in the order documents first arrived"""
        index = self.indexes[self.aliases[alias]]
        order = sorted(index["docs"], key=index["order"].get)
        body = b"".join(b'{"index":{"_id":' + um.json_string(i).encode("utf-8", "surrogatepass") + b"}}\n" + index["docs"][i] + b"\n"
                        for i in order)
        return D.pages_of(body, page_hits, seed=1)


@pytest.fixture(scope="module")
def export_body(ctx):
    return D.compact(ur.calc_all_from_events(random_export(11), WAP, 0, now_ms=NOW, ctx=ctx))


def expected_log(new, n_bulk, old=None, first=False):
    log = [("HEAD", f"/{new}"), ("PUT", f"/{new}"), ("POST", f"/{new}/_refresh")] + [("POST", f"/{new}/items/_bulk")] * n_bulk
    log.append(("HEAD", "/_alias/urindex"))
    if not first:
        log += [("GET", "/_alias/urindex"), ("HEAD", f"/{old}")]
    log.append(("POST", "/_aliases"))
    if not first:
        log.append(("HEAD", f"/{old}"))   # remove_index deleted it: deleteIndex finds nothing to delete
    return log


def test_two_writes_swap_the_alias_and_delete_the_first_index(ctx, export_body):
    es = FakeES()
    n_req = len(um.bulk_requests(export_body, 7, 1 << 20)[0]) - 1
    new1, res1 = ur.write_index(export_body, WAP, es, now_ms=NOW, max_docs=7, ctx=ctx)
    assert new1 == f"urindex_{NOW}" and es.aliases == {"urindex": new1} and res1.n_ok == len(res1.status)
    assert es.log == expected_log(new1, n_req, first=True)
    mapping = es.indexes[new1]["mapping"]["mappings"]["items"]["properties"]
    fields = um.index_fields(export_body)
    ranks = {"popRank", "uniqueRank"}   # WAP's rankings: float; the event names and the properties: keyword
    assert list(mapping) == fields + ["last"] and ranks <= set(fields)
    assert all(mapping[f] == {"type": "float" if f in ranks else "keyword"} for f in fields)
    es.log.clear()
    new2, _ = ur.write_index(export_body, WAP, es, now_ms=NOW + 1, max_docs=7, ctx=ctx)
    assert es.aliases == {"urindex": new2} and set(es.indexes) == {new2}
    assert es.log == expected_log(new2, n_req, old=new1)
    assert ur.index_from_pages(es.pages("urindex", 5), ctx=ctx) == export_body


def test_429s_within_retries_recover(ctx, export_body):
    ids = [i for i, _ in D.docs_of(export_body)]
    es = FakeES(reject={ids[0]: 3, ids[5]: 1, ids[-1]: 2}, es5=False)
    new, res = ur.write_index(export_body, WAP, es, now_ms=NOW, max_docs=4, retries=3, retry_wait_s=0, ctx=ctx)
    assert res.n_ok == len(ids) and res.n_rejected == res.n_failed == 0 and es.aliases == {"urindex": new}
    assert sum(1 for m, p in es.log if p.endswith("/_bulk")) == len(um.bulk_requests(export_body, 4, 1 << 20)[0]) - 1 + 3
    assert ur.index_from_pages(es.pages("urindex", 0), ctx=ctx) == export_body


@pytest.mark.parametrize("kind", ["429 past retries", "400"])
def test_failures_raise_with_ids_and_keep_the_alias(ctx, export_body, kind):
    ids = [i for i, _ in D.docs_of(export_body)]
    es = FakeES()
    old, _ = ur.write_index(export_body, WAP, es, now_ms=NOW, ctx=ctx)
    es.reject, es.fail = ({ids[3]: 5}, set()) if kind != "400" else ({}, {ids[3], ids[8]})
    with pytest.raises(ur.IndexWriteError) as e:
        ur.write_index(export_body, WAP, es, now_ms=NOW + 5, retries=2, retry_wait_s=0, ctx=ctx)
    msg = str(e.value)
    assert repr(ids[3]) in msg
    assert ("es_rejected_execution_exception" if kind != "400" else "mapper_parsing_exception: failed to parse [view]") in msg
    assert es.aliases == {"urindex": old} and f"urindex_{NOW + 5}" in es.indexes
    assert e.value.result.n_rejected == (1 if kind != "400" else 0) and e.value.result.n_failed == (0 if kind != "400" else 2)
    assert not any(p == "/_aliases" for _, p in es.log[-3:])


# ---- part 2: the device against the mirrors --------------------------------------------------------------------------------
def check_body(ctx, body, max_docs=1000, max_bytes=1 << 20):
    with ctx.index_write(body, max_docs, max_bytes) as w:
        assert w.fields() == um.index_fields(body)
        db, bb = w.cuts()
        assert (list(db), list(bb)) == um.bulk_requests(body, max_docs, max_bytes)
        assert b"".join(w.requests()) == body


NAME_EDGES = ["", "a\\\"b\x01\x1f", "\U0001F600\U0001F4A9", "\ud800x", "n" * 1500, "é"]


def edge_names_body() -> bytes:
    """names and ids of every escape class, 4-byte UTF-8, a lone surrogate, empty and 1 500 bytes at members 0, 31, 32, and
    documents of 0, 1, 31, 32, 33, 64 and 65 members"""
    out = b""
    for k, nm in enumerate(NAME_EDGES):
        members = ["m%d" % j for j in range(33)]
        for slot in (0, 31, 32):
            members[slot] = nm + str(slot)
        src = "{" + ",".join(um.json_string(m) + ":" + str(j) for j, m in enumerate(members)) + "}"
        out += b'{"index":{"_id":' + um.json_string(nm).encode("utf-8", "surrogatepass") + b'}}\n' + src.encode("utf-8", "surrogatepass") + b"\n"
    for n in (0, 1, 31, 32, 33, 64, 65):
        src = "{" + ",".join('"c%d\\u0041":[]' % j for j in range(n)) + "}"
        out += b'{"index":{"_id":"count%d"}}\n' % n + src.encode() + b"\n"
    return out


def test_member_counts_occur():
    counts = {len(m) for _, _, _, m in um.bulk_documents(edge_names_body())}
    assert {0, 1, 31, 32, 33, 64, 65} <= counts


def test_handmade_bodies(ctx, orc):
    for _, body in D.handmade_bodies(orc):
        check_body(ctx, body)
        check_body(ctx, body, max_docs=2, max_bytes=300)


@pytest.mark.parametrize("seed", [3, 11])
def test_export_bodies(ctx, seed):
    body = ur.calc_all_from_events(random_export(seed), WAP, 0, now_ms=NOW, ctx=ctx)
    pop = ur.calc_pop_from_events(body, random_export(seed + 1), WAP, now_ms=NOW, ctx=ctx)
    paged = ur.index_from_pages(D.pages_of(body, 9, seed=seed), ctx=ctx)
    for b in (body, pop, paged):
        check_body(ctx, b)
        check_body(ctx, b, max_docs=3, max_bytes=700)


def test_edge_bodies(ctx):
    for body in (edge_names_body(), D.edge_body(random.Random(5)), b""):
        for md, mb in ((1000, 1 << 20), (1, 1 << 20), (4, 2000), (1000, 1)):
            check_body(ctx, body, md, mb)


def test_1e5_distinct_fields(ctx):
    rng = random.Random(7)
    out = b""
    for d in range(1000):
        names = ["f%05d" % (d * 100 + k) for k in range(100)] + ["f%05d" % rng.randrange(100000) for _ in range(20)]
        rng.shuffle(names)
        out += b'{"index":{"_id":"d%d"}}\n' % d + ("{" + ",".join('"%s":1' % n for n in names) + "}").encode() + b"\n"
    fields = um.index_fields(out)
    assert len(fields) == 100001
    check_body(ctx, out)


def run_responses(ctx, body, max_docs, rng, es5, pretty, statuses_of, order=None):
    """answer every request (and the retry rounds) with the statuses statuses_of(round, ids) -> compare with the mirror"""
    docs = um.bulk_documents(body)
    ids = [d[0] for d in docs]
    want = [0] * len(ids)
    errs = {}
    with ctx.index_write(body, max_docs, 1 << 20) as w:
        db, _ = w.cuts()
        reqs = list(range(len(db) - 1))
        if order == "reversed":
            reqs.reverse()
        elif order == "shuffled":
            rng.shuffle(reqs)
        parts = w.requests()
        rnd = 0
        batch = [(q, list(range(db[q], db[q + 1])), parts[q]) for q in reqs]
        while batch:
            for q, dlist, part in batch:
                rid = [ids[d] for d in dlist]
                st = statuses_of(rnd, rid)
                resp = bulk_response(rid, st, rng, es5=es5, pretty=pretty, errors_flag=False if rnd == 0 else None)
                for d, (s, t, r) in zip(dlist, um.bulk_item_statuses(resp, rid)):
                    want[d] = s
                    errs[d] = (t, r)
                w.response(q, resp)
            first, rparts = w.retry()
            assert [list(dd) for dd, _ in rparts] == _chunks([d for d in range(len(ids)) if want[d] == 429], max_docs)
            rnd += 1
            batch = [(first + k, list(dd), p) for k, (dd, p) in enumerate(rparts)]
            if rnd > 4:
                break
        res = w.finish()
    assert list(res.status) == want
    assert res.n_ok == sum(200 <= s < 300 for s in want) and res.n_rejected == want.count(429)
    assert res.errors == [(d, *errs[d]) for d in range(len(ids)) if not 200 <= want[d] < 300]


def _chunks(xs, n):
    return [xs[k:k + n] for k in range(0, len(xs), n)]


@pytest.mark.parametrize("es5,pretty,order", [(True, False, None), (False, True, "reversed"), (True, True, "shuffled"),
                                              (False, False, "shuffled")])
def test_responses_against_mirror(ctx, export_body, es5, pretty, order):
    rng = random.Random(hash((es5, pretty, order)) & 0xffff)
    bad = {i for i, _ in D.docs_of(export_body)[::7]}

    def statuses(rnd, rid):
        return [429 if i in bad and rnd < 2 else 400 if i in bad and rnd == 2 and i.endswith("1") else 201 if rnd % 2 == 0 else 200
                for i in rid]
    run_responses(ctx, export_body, 5, rng, es5, pretty, statuses, order)


def test_edge_ids_and_reasons(ctx):
    body = D.edge_body(random.Random(5))
    rng = random.Random(2)
    reasons = {i: ("t\\\"é" + i[:3], "r\n😀" + i[:10]) for i in D.ID_EDGES}
    with ctx.index_write(body, 3, 1 << 20) as w:
        db, _ = w.cuts()
        ids = [d[0] for d in um.bulk_documents(body)]
        for q in range(len(db) - 1):
            rid = ids[db[q]:db[q + 1]]
            resp = bulk_response(rid, [500] * len(rid), rng, pretty=q % 2 == 1, reasons=reasons)
            w.response(q, resp)
        res = w.finish()
    assert res.n_failed == len(ids)
    assert [(t, r) for _, t, r in res.errors] == [reasons[i] for i in ids]


def test_more_items_than_warps(ctx):
    n = 20000
    body = b"".join(b'{"index":{"_id":"i%d"}}\n{"id":"i%d"}\n' % (k, k) for k in range(n))
    rng = random.Random(4)
    run_responses(ctx, body, n, rng, False, False, lambda rnd, rid: [429 if rnd == 0 and int(i[1:]) % 97 == 0 else 201 for i in rid])


ONE = b'{"index":{"_id":"a"}}\n{"id":"a"}\n'
ERRORS = [
    (b'{"items":[]}', 0, "request 0: 0 items for 1 documents"),
    (b'{"items":[{"index":{"_id":"b","status":201}}]}', 0, "request 0, item 0: the item's _id is not the document's _id"),
    (b'{"items":[{"index":{"_id":"a","status":201,"status":201}}]}', 0, "request 0, item 0: a repeated status"),
    (b'{"items":[{"index":{"_id":"a"}}]}', 0, "request 0, item 0: the item has no status"),
    (b'{"error":{"root_cause":[],"type":"x","reason":"y"},"status":413}', 0, "request 0: Elasticsearch returned an error (status 413)"),
    (b'{"items":[{"index":{"_id":"a","status":201}}]}', 5, "request 5 is out of range"),
    (b'{"items":[{"index":{"_id":"a","status":2.5}}]}', 0, "request 0, item 0: the status is not a 32-bit integer"),
    (b'{"items":[{"index":{"_id":"a","status":201}}', 0, "request 0, byte"),
]


@pytest.mark.parametrize("resp,q,msg", ERRORS)
def test_each_error(ctx, resp, q, msg):
    with ctx.index_write(ONE) as w:
        with pytest.raises(N.CcoInvalidArgument) as e:
            w.response(q, resp)
        assert msg in str(e.value)
        with pytest.raises(N.CcoInvalidArgument) as again:
            w.finish()
        assert str(again.value) == str(e.value)


def test_answered_twice(ctx):
    with ctx.index_write(ONE) as w:
        w.response(0, b'{"items":[{"index":{"_id":"a","status":201}}]}')
        with pytest.raises(N.CcoInvalidArgument, match="request 0 is answered twice"):
            w.response(0, b'{"items":[{"index":{"_id":"a","status":201}}]}')


@pytest.mark.parametrize("body,msg", [(b'{"index":{"id":"a"}}\n{}\n', "document 0: the action line"),
                                      (b'{"index":{"_id":"a"}}\n{}\n{"index":{"_id":"a"}}\n{}\n', "document 1: its _id is the _id of document 0"),
                                      (b'{"index":{"_id":"a"}}\n', "lines come in (action, source) pairs"),
                                      (b'{"index":{"_id":"a"}}\n{}', "does not end in a newline")])
def test_body_not_in_bulk_form(ctx, body, msg):
    with pytest.raises(N.CcoInvalidArgument) as e:
        ctx.index_write(body)
    assert msg in str(e.value)

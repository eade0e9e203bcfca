"""Elasticsearch _search / _search/scroll pages for the index-pages tests: model index bodies (the reference's handmade data
under every ranking engine, and documents with edge ids) rendered as the pages a scroll returns, seeded, with compact or
pretty-printed sources, ES 5 or ES 7 totals, and the members a real page carries around each hit."""
import json
import random
import re

import search_results_data as SD
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200 import ur_predict as P

CONFIGS = ["pop-engine.json", "trend-engine.json", "hot-3-day-engine.json", "rank/rank-engine.json"]
ID_EDGES = SD.ID_EDGES + ["\U0001F600\U0001F4A9", "\ud800lone", "x" * 1500 + "é"]


def handmade_bodies(orc) -> list:
    """[(engine, bulk body)]: model_oracle.model_bulk over tests/golden/model_handmade.json for every ranking engine"""
    from conftest import load_golden
    from test_model_docs import bulk_and_docs, model_inputs
    fx = load_golden("model_handmade.json")
    out = []
    for config in CONFIGS:
        prepared, triples, fields, rankings = model_inputs(fx, config)
        mats = [orc.Csr(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
        ref = orc.train(mats, [orc.Params(500, 50, None)] * len(mats), 1)
        body, _ = bulk_and_docs([(r.row_ptr, r.col_idx) for r in ref], prepared, triples, fields, rankings)
        out.append((config, body))
    return out


def edge_body(rng) -> bytes:
    """documents whose ids are the escape classes, 4-byte UTF-8, lone surrogates and 1 500-byte ids, with sources that
    hold escapes, nested arrays, repeated members and number spellings"""
    out = bytearray()
    for k, item in enumerate(ID_EDGES):
        q = um.json_string(item).encode("utf-8", "surrogatepass")
        src = b'{"id":' + q + b',"purchase":[' + b",".join(um.json_string(x).encode("utf-8", "surrogatepass")
                                                           for x in rng.sample(ID_EDGES, 3)) + b']'
        src += b',"n":' + rng.choice([b"1.0E7", b"-0", b"2.5e-3", b"12345678901234567890", b"0.0"])
        if k % 3 == 0:
            src += b',"n":[{"a":"\\u00e9 \\" ]} "},[]]'
        out += b'{"index":{"_id":' + q + b"}}\n" + src + b"}\n"
    return bytes(out)


_OUTSIDE_WS = re.compile(rb'("(?:[^"\\]|\\.)*")|[ \t\r]+', re.S)


def compact(body: bytes) -> bytes:
    """a bulk body with the whitespace outside strings dropped from its lines (an export's property values are spliced as
    spelled, `[1, 2]` included; a page reader gives them back as `[1,2]`)"""
    return _OUTSIDE_WS.sub(lambda m: m.group(1) or b"", body)


def docs_of(body: bytes) -> list:
    """[(decoded _id, _source bytes)] of a bulk body"""
    lines = body.split(b"\n")
    assert lines[-1] == b""
    return [(P.loads(lines[i]).get("index").get("_id"), lines[i + 1]) for i in range(0, len(lines) - 1, 2)]


def _id_text(item: str, rng) -> str:
    """the _id as Elasticsearch may spell it: raw UTF-8 or \\u escapes"""
    return json.dumps(item, ensure_ascii=rng.random() < 0.5)


def hit(item: str, source: bytes, rng) -> str:
    """one hit, its members in a random order with the ones ES adds around _id and _source"""
    members = [('"_id"', _id_text(item, rng)), ('"_source"', source.decode("utf-8", "surrogatepass"))]
    extra = [('"_index"', '"urindex"'), ('"_type"', '"items"'), ('"_score"', rng.choice(["null", "1.0", "0"])),
             ('"sort"', "[" + str(rng.randrange(10 ** 6)) + ',"x]"]'), ('"_routing"', '"r\\"1"'),
             ('"fields"', '{"a":[1,{"b":"}"}]}')]
    members += rng.sample(extra, rng.randrange(len(extra) + 1))
    rng.shuffle(members)
    return "{" + ",".join(k + ":" + v for k, v in members) + "}"


def page(hits: list, rng, total=None, scroll_id="c2Nyb2xs", es7=True, pretty=False) -> bytes:
    """one scroll page of hit texts; total: hits.total (None: absent)"""
    parts = []
    if scroll_id is not None:
        parts.append('"_scroll_id":' + json.dumps(scroll_id))
    parts += ['"took":' + str(rng.randrange(100)), '"timed_out":false',
              '"_shards":{"total":5,"successful":5,"skipped":0,"failed":0}']
    hp = []
    if total is not None:
        hp.append('"total":' + ('{"value":%d,"relation":"eq"}' % total if es7 else str(total)))
    hp += ['"max_score":null', '"hits":[' + ",".join(hits) + "]"]
    parts.append('"hits":{' + ",".join(hp) + "}")
    text = "{" + ",".join(parts) + "}"
    return ((SD.pretty(text) + "\n") if pretty else text).encode("utf-8", "surrogatepass")


def pages_of(body: bytes, page_hits: int, seed: int, pretty=False, es7=True) -> list:
    """the pages a scroll of page_hits (0: all in one) returns for the index `body`, ending with an empty page"""
    rng = random.Random(seed)
    docs = docs_of(body)
    n = page_hits or max(len(docs), 1)
    hits = [hit(i, s, rng) for i, s in docs]
    out = [page(hits[k:k + n], rng, total=len(docs), es7=es7, pretty=pretty) for k in range(0, len(hits), n)]
    return out + [page([], rng, total=len(docs), es7=es7, pretty=pretty)]

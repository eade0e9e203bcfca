"""TEST INFRASTRUCTURE: CPU restatement of cco_rerank_model, the rankings of an existing model index refreshed (calcPop).
Built on oracle/format_oracle.json_escape, model_oracle.java_double_int and random_rank_oracle.ranking_scores; the old
body is parsed with the json module, keeping the raw bytes of every top-level member's name and value.

Documents: the old ones in body order, then every item without an old document that has a property or a score, by first
appearance (property triples, then the ranking streams in order).  An old document:
    {"index":{"_id":"<decoded _id, escaped>"}}\\n{"id":"<same>"[,<old member>]*[,"<field>":<json>]*[,"<ranking>":<number>]*}\\n
old members in their order, spliced verbatim, except "id", those named like a ranking present for the item and those
followed by a member of the same (decoded) name; the properties in field index order except "id", those named like any old
member or like a present ranking; the rankings as model_oracle writes them.  A new document is model_bulk's."""
from __future__ import annotations

import json

import random_rank_oracle as ro
from oracle import format_oracle as fo

_ws = " \t\r\n"


def _skip(s: str, i: int) -> int:
    while i < len(s) and s[i] in _ws:
        i += 1
    return i


def members(line: str) -> list[tuple[bytes, str, bytes]]:
    """the top-level members of one JSON object line: (raw name bytes, decoded name, raw value bytes); ValueError if the line
    is not one object"""
    dec = json.JSONDecoder()
    i = _skip(line, 0)
    if not line.startswith("{", i):
        raise ValueError("not an object")
    i = _skip(line, i + 1)
    out = []
    if line.startswith("}", i):
        i += 1
    else:
        while True:
            if not line.startswith('"', i):
                raise ValueError("a member name must be a string")
            name, j = json.decoder.scanstring(line, i + 1, True)
            raw_name = line[i + 1:j - 1]
            i = _skip(line, j)
            if not line.startswith(":", i):
                raise ValueError("':' expected")
            i = _skip(line, i + 1)
            _, k = dec.raw_decode(line, i)
            out.append((raw_name.encode("utf-8"), name, line[i:k].encode("utf-8")))
            i = _skip(line, k)
            if line.startswith(",", i):
                i = _skip(line, i + 1)
            elif line.startswith("}", i):
                i += 1
                break
            else:
                raise ValueError("',' or '}' expected")
    if _skip(line, i) != len(line):
        raise ValueError("bytes after the object")
    return out


def parse_body(body: bytes) -> list[tuple[str, list[tuple[bytes, str, bytes]]]]:
    """a bulk body -> [(decoded _id, source members)]; ValueError for anything cco_rerank_model refuses"""
    if not body:
        return []
    if not body.endswith(b"\n"):
        raise ValueError("no final newline")
    lines = body[:-1].decode("utf-8").split("\n")
    if len(lines) % 2:
        raise ValueError("odd number of lines")
    docs, ids = [], set()
    for d in range(0, len(lines), 2):
        action = json.loads(lines[d], object_pairs_hook=list)
        if not isinstance(action, list) or len(action) != 1 or action[0][0] != "index" or not isinstance(action[0][1], list):
            raise ValueError(f"document {d // 2}: bad action")
        got = [v for k, v in action[0][1] if k == "_id"]
        if not got or not isinstance(got[-1], str):
            raise ValueError(f"document {d // 2}: no string _id")
        if got[-1] in ids:
            raise ValueError(f"document {d // 2}: repeated _id")
        ids.add(got[-1])
        docs.append((got[-1], members(lines[d + 1])))
    return docs


def old_documents(body: bytes) -> list[tuple[str, dict]]:
    """the body as ur_model.rerank_documents takes it: (id, {name: value}), the last of a repeated name winning"""
    return [(i, {name: json.loads(v) for _, name, v in ms}) for i, ms in parse_body(body)]


def rerank_bulk(body: bytes, field_names=(), triples=(), rankings=()) -> bytes:
    """triples = [(item id, field index, JSON text)], rankings = [(field name, mode, start_ms, end_ms, [(item ids, times)])]
    with mode popular / trending / hot / random, as random_rank_oracle.model_bulk takes them"""
    old = parse_body(body)
    props: dict = {}
    for item, f, text in triples:
        props.setdefault(item, {})[int(f)] = text
    property_items = [t[0] for t in triples]
    scored = [(name, ro.ranking_scores(mode, s, e, streams, property_items)) for name, mode, s, e, streams in rankings]
    rank_text = [ro.random_rank_text if mode == "random" else ro.mo.java_double_int for _, mode, *_ in rankings]
    order = list(old)
    have, seen = {i for i, _ in old}, set()
    for item in property_items + [i for *_, streams in rankings for s in streams for i in s[0]]:
        if item not in have and item not in seen:
            seen.add(item)
            if item in props or any(item in sc for _, sc in scored):
                order.append((item, []))
    out = bytearray()
    for item, ms in order:
        iid = fo.json_escape(item)
        have_props = props.get(item, {})
        have_ranks = [name for name, sc in scored if item in sc]
        names = {name for _, name, _ in ms}
        out += b'{"index":{"_id":"' + iid + b'"}}\n{"id":"' + iid + b'"'
        for j, (raw_name, name, raw_value) in enumerate(ms):
            if name == "id" or name in have_ranks or any(n == name for _, n, _ in ms[j + 1:]):
                continue
            out += b',"' + raw_name + b'":' + raw_value
        for f in sorted(have_props):
            if field_names[f] == "id" or field_names[f] in names or field_names[f] in have_ranks:
                continue
            out += b',"' + fo.json_escape(field_names[f]) + b'":' + have_props[f].encode("utf-8")
        for k, (name, sc) in enumerate(scored):
            if item not in sc or name == "id" or any(n == name and item in s for n, s in scored[k + 1:]):
                continue
            out += b',"' + fo.json_escape(name) + b'":' + rank_text[k](sc[item])
        out += b"}\n"
    return bytes(out)

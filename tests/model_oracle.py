"""TEST INFRASTRUCTURE: CPU restatement of the complete model index (cco_format_model), built on the conventions of
oracle/format_oracle.es_bulk and the PopModel restatement of oracle/pop_oracle.py.

    {"index":{"_id":"<id>"}}\\n{"id":"<id>"[,"<indicator>":[...]]*[,"<field>":<json>]*[,"<ranking>":<number>]*}\\n

Documents: the rows [row_begin, row_end) in row order; then, if row_begin == 0, every item without a row that has a property
or a score, by first appearance (property triples first, then the ranking streams in order).  Inside a document: "id", the
indicators in name order, the properties in field index order, the rankings in order; a field is dropped when a higher one
of the same name is in the document (indicators < properties < rankings, a later ranking over an earlier one, "id" over
everything but indicators, which are written as es_bulk writes them).  Rank numbers: Java's Double.toString of an integer."""
from __future__ import annotations

from oracle import format_oracle as fo
from oracle import pop_oracle as po


def java_double_int(v: int) -> bytes:
    s = str(abs(int(v)))
    sign = "-" if v < 0 else ""
    if len(s) <= 7:
        return (sign + s + ".0").encode()
    return (sign + s[0] + "." + (s[1:].rstrip("0") or "0") + "E" + str(len(s) - 1)).encode()


def ranking_scores(mode: str, start_ms: int, end_ms: int, streams) -> dict:
    """streams = [(item id strings, times)] -> {item id: integer score} through pop_oracle (ids numbered first)"""
    number: dict = {}
    items = [number.setdefault(i, len(number)) for s in streams for i in s[0]]
    times = [int(t) for s in streams for t in s[1]]
    ids = list(number)
    return {ids[j]: int(v) for j, v in po.pop_model(mode, items, times, start_ms, end_ms).items()}


def model_bulk(indicators, names, row_ids, col_ids, field_names=(), triples=(), rankings=(), row_begin: int = 0,
               row_end: int | None = None) -> bytes:
    """indicators / names / row_ids / col_ids / row_begin / row_end: as fo.es_bulk.  triples = [(item id, field index, JSON
    text)], the last of a repeated (item, field) wins.  rankings = [(field name, mode, start_ms, end_ms, [(item ids, times)])]."""
    n_rows = len(indicators[0][0]) - 1
    if row_end is None:
        row_end = row_begin + n_rows
    props: dict = {}
    for item, f, text in triples:
        assert text, "empty property value"
        props.setdefault(item, {})[int(f)] = text
    scored = [(name, ranking_scores(mode, s, e, streams)) for name, mode, s, e, streams in rankings]
    rows = set(row_ids)
    order = [(row_ids[row_begin + r], r) for r in range(n_rows)]
    if row_begin == 0:
        seen = set()
        for item in [t[0] for t in triples] + [i for *_, streams in rankings for s in streams for i in s[0]]:
            if item not in rows and item not in seen:
                seen.add(item)
                if item in props or any(item in sc for _, sc in scored):
                    order.append((item, -1))
    esc_cols = [[fo.json_escape(x) for x in ids] for ids in col_ids]
    out = bytearray()
    for item, r in order:
        iid = fo.json_escape(item)
        have_props = props.get(item, {})
        have_ranks = [name for name, sc in scored if item in sc]
        out += b'{"index":{"_id":"' + iid + b'"}}\n{"id":"' + iid + b'"'
        if r >= 0:
            for i, (rp, ci) in enumerate(indicators):
                if any(field_names[f] == names[i] for f in have_props) or names[i] in have_ranks:
                    continue
                out += b',"' + fo.json_escape(names[i]) + b'":['
                out += b",".join(b'"' + esc_cols[i][int(c)] + b'"' for c in ci[int(rp[r]) - int(rp[0]):int(rp[r + 1]) - int(rp[0])])
                out += b"]"
        for f in sorted(have_props):
            if field_names[f] == "id" or field_names[f] in have_ranks:
                continue
            out += b',"' + fo.json_escape(field_names[f]) + b'":' + have_props[f].encode("utf-8")
        for k, (name, sc) in enumerate(scored):
            if item not in sc or name == "id" or any(n == name and item in s for n, s in scored[k + 1:]):
                continue
            out += b',"' + fo.json_escape(name) + b'":' + java_double_int(sc[item])
        out += b"}\n"
    return bytes(out)

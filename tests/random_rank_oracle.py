"""TEST INFRASTRUCTURE: CPU restatement of the complete model index (cco_format_model) with random (uniqueRank) rankings.
It is tests/model_oracle.py's model_bulk with one more ranking mode; the popular / trending / hot scores and the integer
rank text are model_oracle's own, so for rankings of those modes both give the same bytes.

A random ranking scores the items of its events in [start_ms, end_ms) (every stream it is given) plus every property item,
with n from ur_model.random_rank, and its text is Java's Double.toString of n / 10^15 (random_rank_text)."""
from __future__ import annotations

import model_oracle as mo
from oracle import format_oracle as fo
from universal_recommender_b200 import ur_model as um


def random_rank_text(n: int) -> bytes:
    """Java's Double.toString of n / 10^15 (0 <= n < 10^15) from n's digits: 0.0; 0.ddd for n >= 10^12 (>= 10^-3), the 15
    fraction digits without trailing zeros; else d.ddd"E-"k"""
    if n == 0:
        return b"0.0"
    if n >= 10**12:
        return ("0." + str(n).zfill(15).rstrip("0")).encode()
    s = str(n)
    return (s[0] + "." + (s[1:].rstrip("0") or "0") + "E-" + str(16 - len(s))).encode()


def ranking_scores(mode: str, start_ms: int, end_ms: int, streams, property_items=()) -> dict:
    """{item id: integer score}: model_oracle.ranking_scores, or for random {item id: n} over the items of the events in
    [start_ms, end_ms) and the property items"""
    if mode != "random":
        return mo.ranking_scores(mode, start_ms, end_ms, streams)
    keep = [i for s in streams for i, t in zip(s[0], s[1]) if start_ms <= int(t) < end_ms] + list(property_items)
    return {i: um.random_rank(i, start_ms, end_ms) for i in dict.fromkeys(keep)}


def model_bulk(indicators, names, row_ids, col_ids, field_names=(), triples=(), rankings=(), row_begin: int = 0,
               row_end: int | None = None) -> bytes:
    """model_oracle.model_bulk's arguments and bytes; a ranking's mode may also be "random"."""
    n_rows = len(indicators[0][0]) - 1
    if row_end is None:
        row_end = row_begin + n_rows
    props: dict = {}
    for item, f, text in triples:
        assert text, "empty property value"
        props.setdefault(item, {})[int(f)] = text
    property_items = [t[0] for t in triples]
    scored = [(name, ranking_scores(mode, s, e, streams, property_items)) for name, mode, s, e, streams in rankings]
    rank_text = [random_rank_text if mode == "random" else mo.java_double_int for _, mode, *_ in rankings]
    rows = set(row_ids)
    order = [(row_ids[row_begin + r], r) for r in range(n_rows)]
    if row_begin == 0:
        seen = set()
        for item in property_items + [i for *_, streams in rankings for s in streams for i in s[0]]:
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
            out += b',"' + fo.json_escape(name) + b'":' + rank_text[k](sc[item])
        out += b"}\n"
    return bytes(out)

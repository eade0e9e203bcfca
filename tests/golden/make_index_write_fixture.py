#!/usr/bin/env python
"""Writes tests/golden/index_write_handmade.json: the bodies EsClient.createIndex PUTs and EsClient.hotSwap POSTs to
_aliases (EsClient.scala:168-246, 257-362) for examples/handmade-engine.json's algorithm params (indexName urindex,
typeName items, indicators purchase / view / category-pref, the default popRank ranking, the date names date, available
and expires).  The Scala string construction is restated here on its own terms: each template is the triple-quoted
literal as the source spells it, put through stripMargin and .replace("\n", ""), and the field types are getMappings'
Map built with `++` in the source's order (URAlgorithm.scala:955-967)."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))

ALGO = {"indexName": "urindex", "typeName": "items",
        "indicators": [{"name": "purchase"}, {"name": "view", "maxCorrelatorsPerItem": 50},
                       {"name": "category-pref", "maxCorrelatorsPerItem": 50}],
        "availableDateName": "available", "expireDateName": "expires", "dateName": "date", "num": 4}


def strip_margin(s: str) -> str:
    out = []
    for line in s.split("\n"):
        t = line.lstrip(" \t")
        out.append(t[1:] if t.startswith("|") else line)
    return "\n".join(out)


def create_index_body(index_type: str, field_names, type_mappings: dict) -> str:
    mappings = strip_margin('''
              |{ "mappings": {
              |    "%s": {
              |      "properties": {
            ''' % index_type).replace("\n", "")

    def mappings_field(t):
        return strip_margin('''
              |    : {
              |      "type": "%s"
              |    },
            ''' % t).replace("\n", "")

    tail = strip_margin('''
              |    "last": {
              |      "type": "keyword"
              |    }
              |}}}}
            ''').replace("\n", "")
    for f in field_names:
        mappings += '"%s"' % f + mappings_field(type_mappings.get(f, "keyword"))
    return mappings + tail


def alias_query(alias: str, new_index: str, old_index) -> str:
    delete_old = ',{ "remove_index": { "index": "%s"}}' % old_index if old_index is not None else ""
    return strip_margin('''
        |{
        |    "actions" : [
        |        { "add":  { "index": "%s", "alias": "%s" } }
        |        %s
        |    ]
        |}
      ''' % (new_index, alias, delete_old)).replace("\n", "")


def get_mappings() -> dict:
    ranking_field_names = ["popRank"]   # no rankings in the engine: the default popular ranking's field
    model_event_names = [i["name"] for i in ALGO["indicators"]]
    date_names = list(dict.fromkeys(d for d in (ALGO["dateName"], ALGO["availableDateName"], ALGO["expireDateName"]) if d))
    m = {}
    m.update({f: "float" for f in ranking_field_names})
    m.update({c: "keyword" for c in model_event_names})
    m.update({d: "date" for d in date_names})
    return m


FIELD_SETS = [
    ["purchase", "view", "category-pref", "popRank", "categories", "available", "expires", "date", "countries", "id"],
    ["id"],
    [],
    ["view", "last", "date", "id"],   # a property really named "last": the reference writes the key twice
    ["a\\\"b", "tab\\u0009", "id"],   # names needing escapes, spelled escaped
]


def main():
    tm = get_mappings()
    out = {"algorithm_params": ALGO, "mappings": [], "aliases": []}
    for fields in FIELD_SETS:
        out["mappings"].append({"fields": fields, "body": create_index_body(ALGO["typeName"], fields, tm)})
    for old in (None, "urindex_1699999999000"):
        out["aliases"].append({"alias": "urindex", "new_index": "urindex_1700000000000", "old_index": old,
                               "body": alias_query("urindex", "urindex_1700000000000", old)})
    with open(os.path.join(HERE, "index_write_handmade.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()

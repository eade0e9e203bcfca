"""calcPop on the CPU (recsModel "backfill"): the host mirror ur_model.rerank_documents against the byte-level restatement
tests/rerank_oracle.py, on the reference's data and on directed cases of every precedence rule."""
import os
import subprocess

import pytest

import rerank_oracle as rr
from conftest import ROOT, load_golden
from test_model_docs import CONFIGS, MODEL_FIXTURES, docs_of, model_inputs
from universal_recommender_b200 import ur_model as um


def fixture_rankings(fx, config, now_ms):
    """the fixture's rankings of a config with "now" at now_ms"""
    from universal_recommender_b200.ur_algorithm import URAlgorithmParams
    ap = URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"],
                                             "rankings": fx["rankings"][config]})
    by_name = {}
    for _, e, i, t in fx["events"]:
        by_name.setdefault(e, []).append((i, t))
    names = ap.model_event_names()
    return um.rankings_for(um.rankings_params(ap.rankings, names), by_name, now_ms, names)


def fixture_body(name, config):
    """(the fixture's fixture, its model body as the model restatement writes it, field names, JSON triples, oracle
    rankings, mirror triples, mirror rankings)"""
    import random_rank_oracle as ro
    from oracle import oracle as orc
    fx = load_golden(name)
    prepared, triples, fields, rankings = model_inputs(fx, config)
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    orc.build()
    res = orc.train([orc.Csr(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared], [orc.Params(500, 50, None)] * len(prepared), 1)
    jt = [(i, fields.index(f), um.property_json(v)) for i, f, v in triples]
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    body = ro.model_bulk([(r.row_ptr, r.col_idx) for r in res], names, rows, cols, fields, jt, rk)
    return fx, body, fields, jt, rk, triples, rankings


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_restatement_and_mirror_agree_on_the_reference_data(name, config):
    fx, body, fields, jt, rk, triples, rankings = fixture_body(name, config)
    got = rr.rerank_bulk(body, fields, jt, rk)
    assert got == body   # the fixed point: ranks already last and in order, old property members equal the fresh ones
    assert docs_of(got) == um.rerank_documents(rr.old_documents(body), triples, rankings)
    # a refresh: "now" two days later, half of the properties
    later = fixture_rankings(fx, config, fx["now_ms"] + 2 * 86_400_000)
    rk2 = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in later]
    again = rr.rerank_bulk(body, fields, jt[: len(jt) // 2], rk2)
    assert docs_of(again) == um.rerank_documents(rr.old_documents(body), triples[: len(triples) // 2], later)


def _rank(field, mode, items, times, start=0, end=100):
    return um.Ranking(field, mode, start, end, [(list(items), list(times))])


def _both(body, triples, rankings):
    """(restatement bytes, mirror documents) for mirror triples (item, field, value) and um.Rankings"""
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    jt = [(i, fields.index(f), um.property_json(v)) for i, f, v in triples]
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    got = rr.rerank_bulk(body, fields, jt, rk)
    assert docs_of(got) == um.rerank_documents(rr.old_documents(body), triples, rankings)
    return got


def test_a_fresh_set_loses_to_an_old_member():
    body = b'{"index":{"_id":"a"}}\n{"id":"a","color":"red","size":3}\n'
    got = _both(body, [("a", "color", "blue"), ("a", "shape", "round")], [])
    assert got == b'{"index":{"_id":"a"}}\n{"id":"a","color":"red","size":3,"shape":"round"}\n'


def test_a_stale_rank_survives_when_the_item_has_no_score():
    body = b'{"index":{"_id":"a"}}\n{"id":"a","popRank":7.0}\n{"index":{"_id":"b"}}\n{"id":"b","popRank":2.0}\n'
    got = _both(body, [], [_rank("popRank", "popular", ["b", "b"], [10, 20])])
    assert got == b'{"index":{"_id":"a"}}\n{"id":"a","popRank":7.0}\n{"index":{"_id":"b"}}\n{"id":"b","popRank":2.0}\n'
    got = _both(body, [], [_rank("popRank", "popular", ["b", "b", "b"], [10, 20, 30])])
    assert got.endswith(b'{"id":"b","popRank":3.0}\n') and b'"a","popRank":7.0' in got


def test_the_id_beats_a_different_id_member():
    body = b'{"index":{"_id":"real"}}\n{"id":"fake","x":1}\n'
    assert _both(body, [], []) == b'{"index":{"_id":"real"}}\n{"id":"real","x":1}\n'


def test_the_last_repeated_member_wins():
    body = b'{"index":{"_id":"a"}}\n{"x":1,"y":2,"x":3}\n'
    assert _both(body, [("a", "x", 9)], []) == b'{"index":{"_id":"a"}}\n{"id":"a","y":2,"x":3}\n'
    # repeated names are compared decoded
    body = b'{"index":{"_id":"a"}}\n{"\\u0078":1,"x":2}\n'
    assert rr.rerank_bulk(body) == b'{"index":{"_id":"a"}}\n{"id":"a","x":2}\n'


def test_new_items_are_appended_in_first_appearance_order():
    body = b'{"index":{"_id":"old"}}\n{"id":"old"}\n'
    triples = [("p2", "f", 1), ("old", "f", 2), ("p1", "f", 3)]
    got = _both(body, triples, [_rank("popRank", "popular", ["r1", "p1", "old", "r0"], [1, 2, 3, 4])])
    assert [d["id"] for d in docs_of(got)] == ["old", "p2", "p1", "r1", "r0"]
    assert docs_of(got)[0] == {"id": "old", "f": 2, "popRank": 1.0}


def test_old_documents_without_property_or_rank_are_kept():
    body = b'{"index":{"_id":"a"}}\n{"id":"a","buy":["x","y"]}\n{"index":{"_id":"b"}}\n{}\n'
    got = _both(body, [("c", "f", True)], [_rank("hotRank", "hot", ["c"], [50])])
    assert got == b'{"index":{"_id":"a"}}\n{"id":"a","buy":["x","y"]}\n{"index":{"_id":"b"}}\n{"id":"b"}\n' \
                  b'{"index":{"_id":"c"}}\n{"id":"c","f":true}\n'


def test_a_random_ranking_does_not_cover_items_only_in_the_index():
    body = b'{"index":{"_id":"a"}}\n{"id":"a"}\n{"index":{"_id":"b"}}\n{"id":"b"}\n'
    got = _both(body, [("c", "f", 1)], [_rank("uniqueRank", "random", ["b"], [5])])
    docs = docs_of(got)
    assert "uniqueRank" not in docs[0] and "uniqueRank" in docs[1] and "uniqueRank" in docs[2]


def test_the_restatement_refuses_what_the_device_refuses():
    for bad in [b'{"index":{"_id":"a"}}\n', b'{"index":{"_id":"a"}}\n{}', b'{"create":{"_id":"a"}}\n{}\n',
                b'{"index":{"_id":1}}\n{}\n', b'{"index":{"_id":"a"}}\n[]\n', b'{"index":{"_id":"a"}}\n{}\n{"index":{"_id":"a"}}\n{}\n',
                b'{"index":{"_id":"a"}}\n{"x":"\\q"}\n', b'{"index":{"_id":"a"}}\n{"x":[1}\n']:
        with pytest.raises(ValueError):
            rr.parse_body(bad)


def test_plain_c_program_compiles_against_the_rerank_entry(tmp_path):
    src = tmp_path / "rerank_abi_check.c"
    src.write_text(r'''
#include <stddef.h>
#include "cco_b200.h"
int rerank(cco_ctx_t *ctx, const char *body, int64_t len, char **out, int64_t *out_len) {
  static const int64_t ev_off[3] = {0, 6, 12}, ev_time[2] = {1000, 2000};
  cco_ranking_stream_t stream = {2, ev_off, "item-1item-3", ev_time};
  cco_ranking_t ranking = {"popRank", CCO_POP_POPULAR, 1, 0, 5000, &stream};
  return cco_rerank_model(ctx, body, len, NULL, 1, &ranking, out, out_len);
}
''')
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(tmp_path / "rerank_abi_check.o")], check=True)

"""The complete model index (SURVEY.md 8f-2 + 8f-3) on the CPU: the host mirror ur_model (ranking params, windows, the
property join and its precedence) against the byte-level restatement tests/model_oracle.py, on the reference's data."""
import json
import os
import subprocess

import pytest

from conftest import ROOT, load_golden
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200.ur_algorithm import URAlgorithmParams

MODEL_FIXTURES = ["model_handmade.json", "model_rank.json"]
CONFIGS = ["pop-engine.json", "trend-engine.json", "hot-3-day-engine.json", "rank/rank-engine.json"]


def docs_of(body: bytes):
    lines = body.decode("utf-8").split("\n")
    assert lines[-1] == "" and len(lines) % 2 == 1
    out = []
    for i in range(0, len(lines) - 1, 2):
        action, doc = json.loads(lines[i]), json.loads(lines[i + 1])
        assert action == {"index": {"_id": doc["id"]}}
        out.append(doc)
    return out


def model_inputs(fx, config):
    """a fixture + ranking config -> (event names, prepared actions, JSON triples, field names, Rankings)"""
    from universal_recommender_b200 import preparator
    ap = URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"],
                                             "rankings": fx["rankings"][config]})
    names = ap.model_event_names()
    actions = [(n, [(u, i) for (u, e, i, _) in fx["events"] if e == n]) for n in names]
    actions = [(n, p) for n, p in actions if p]
    prepared = preparator.prepare(actions, fx["min_events_per_user"])
    triples = [(i, f, um.extract_jvalue(f, v)) for i, f, v in um.aggregate_properties((s[0], s[1]) for s in fx["set_events"])]
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    by_name = {}
    for _, e, i, t in fx["events"]:
        by_name.setdefault(e, []).append((i, t))
    rankings = um.rankings_for(um.rankings_params(ap.rankings, names), by_name, fx["now_ms"], names)
    return prepared, triples, fields, rankings


def bulk_and_docs(indicators, prepared, triples, fields, rankings):
    import model_oracle as mo
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    body = mo.model_bulk(indicators, names, rows, cols, fields, [(i, fields.index(f), um.property_json(v)) for i, f, v in triples],
                         [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings])
    per_row = [(n, [[cols[t][int(c)] for c in ci[rp[r]:rp[r + 1]]] for r in range(len(rows))]) for t, (n, (rp, ci)) in enumerate(zip(names, indicators))]
    return body, um.model_documents(rows, per_row, triples, rankings)


# ---- Java's Double.toString ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("v,text", [(0, "0.0"), (9_999_999, "9999999.0"), (-9_999_999, "-9999999.0"), (10_000_000, "1.0E7"),
                                    (12_345_678, "1.2345678E7"), (2**53 - 1, "9.007199254740991E15"), (-3, "-3.0"),
                                    (-12_000_000, "-1.2E7"), (120_000_000, "1.2E8"), (1_000_000_000_000_000, "1.0E15")])
def test_java_double_of_integers(v, text):
    import model_oracle as mo
    assert mo.java_double_int(v) == text.encode()
    assert um.java_double(float(v)) == text


def test_java_double_of_fractions():
    for x, text in [(2.7, "2.7"), (7.15, "7.15"), (1.0, "1.0"), (0.001, "0.001"), (0.000999, "9.99E-4"), (1e21, "1.0E21"),
                    (-0.0, "-0.0"), (123.456, "123.456")]:
        assert um.java_double(x) == text
    assert um.property_json([2.7, "a\"b", 3, True, None]) == '[2.7,"a\\"b",3,true,null]'


# ---- params, window, values ------------------------------------------------------------------------------------------------
def test_ranking_params_default_and_one_per_type():
    d = um.rankings_params(None, ["purchase", "view"])
    assert [(r.field_name(), r.ranking_type(), list(r.eventNames), r.duration) for r in d] == [("popRank", "popular", ["purchase"], "3650 days")]
    rs = [um.RankingParams("a", "popular"), um.RankingParams("b", "trending"), um.RankingParams("c", "popular"), um.RankingParams(None, "hot")]
    assert [r.field_name() for r in um.rankings_params(rs, ["x"])] == ["a", "b", "hotRank"]
    assert um.RankingParams(None, None).field_name() == "popRank" and um.RankingParams(None, "odd").field_name() == "unknownRank"
    ap = URAlgorithmParams.from_engine_json({"eventNames": ["buy"], "rankings": [{"name": "t", "type": "trending", "duration": "2 days"}]})
    assert ap.rankings == [um.RankingParams("t", "trending", None, None, None, "2 days")]


def test_ranking_window():
    now = 1_700_000_000_000
    assert um.ranking_window(um.RankingParams(duration="3650 days"), now) == (now - 3650 * 86_400_000, now)
    assert um.ranking_window(um.RankingParams(duration=259200), now) == (now - 259_200_000, now)
    assert um.ranking_window(um.RankingParams(duration="259200"), now) == (now - 259_200_000, now)
    assert um.ranking_window(um.RankingParams(duration="3 hours"), now) == (now - 3 * 3_600_000, now)
    assert um.ranking_window(um.RankingParams(duration="90 seconds", offsetDate="2020-01-01T00:00:00Z"), now) == (1577836800000 - 90_000, 1577836800000)
    assert um.ranking_window(um.RankingParams(duration="1 day", offsetDate="ISO8601-date"), now) == (now - 86_400_000, now)   # unparsable: now
    with pytest.raises(ValueError):
        um.duration_seconds("3 fortnights")


def test_ranking_field_strings_become_doubles():
    assert um.extract_jvalue("popRank", "2.5") == 2.5 and um.extract_jvalue("hotRank", ["1", "2"]) == [1.0, 2.0]
    assert um.extract_jvalue("defaultRank", "2.5") == "2.5" and um.extract_jvalue("popRank", 3) == 3
    assert um.aggregate_properties([("a", {"x": 1, "y": 2}), ("b", {"x": 3}), ("a", {"x": 4})]) == [("a", "x", 4), ("a", "y", 2), ("b", "x", 3)]


def test_pop_scores_by_item_id_match_the_restatement():
    from oracle import pop_oracle as po
    items = ["a", "a", "a", "b", "b", "b", "b", "c", "c", "d"]
    times = [5, 35, 65, 10, 50, 70, 80, 40, 89, 90]
    for mode in ("popular", "trending", "hot"):
        want = po.pop_model(mode, [ord(i) for i in items], times, 0, 90)
        assert um.pop_scores(mode, items, times, 0, 90) == {chr(j): v for j, v in want.items()}


# ---- the join and its precedence -------------------------------------------------------------------------------------------
def _one_ranking(field, scores_items, mode="popular"):
    return um.Ranking(field, mode, 0, 100, [(scores_items, [1] * len(scores_items))])


def test_join_cases_row_property_rank_and_all_three():
    rows = ["r1", "r2"]
    inds = [("buy", [["r2"], []])]
    triples = [("r1", "color", ["red"]), ("p", "color", ["blue"]), ("both", "size", 3)]
    ranks = [_one_ranking("popRank", ["r1", "k", "k", "both", "ghost-late"])]
    docs = um.model_documents(rows, inds, triples, ranks)
    assert docs == [{"id": "r1", "buy": ["r2"], "color": ["red"], "popRank": 1.0},     # row + property + rank
                    {"id": "r2", "buy": []},                                            # row only
                    {"id": "p", "color": ["blue"]},                                     # property only
                    {"id": "both", "size": 3, "popRank": 1.0},                          # property + rank
                    {"id": "k", "popRank": 2.0},                                        # rank only
                    {"id": "ghost-late", "popRank": 1.0}]
    # an item seen only in a ranking stream without a score gets no document
    docs = um.model_documents(rows, inds, [], [_one_ranking("trendRank", ["z"], mode="trending")])
    assert [d["id"] for d in docs] == rows


def test_precedence_rules_byte_level_and_mirror_agree():
    import model_oracle as mo
    rows = ["r1", "r2"]
    names = ["buy", "view"]
    inds = [([0, 1, 1], [1]), ([0, 0, 1], [0])]
    fields = ["buy", "id", "popRank", "plain"]
    triples = [("r1", 0, '["p"]'), ("r1", 1, '"fake"'), ("r2", 2, "7"), ("r2", 3, "1"), ("r2", 3, "2"), ("x", 3, "5")]
    rankings = [("view", "popular", 0, 100, [(["r2"], [1])]), ("popRank", "popular", 0, 100, [(["r2", "r2", "x"], [1, 2, 3])]),
                ("popRank", "popular", 0, 100, [(["x"], [4])]), ("id", "popular", 0, 100, [(["r1"], [4])])]
    body = mo.model_bulk(inds, names, rows, [rows, rows], fields, triples, rankings)
    assert body.split(b"\n")[1] == b'{"id":"r1","view":[],"buy":["p"]}'                         # property beats indicator; "id" beats all
    assert body.split(b"\n")[3] == b'{"id":"r2","buy":[],"plain":2,"view":1.0,"popRank":2.0}'   # rank beats property and indicator
    assert body.split(b"\n")[5] == b'{"id":"x","plain":5,"popRank":1.0}'                          # the later popRank wins
    mirror = um.model_documents(rows, [("buy", [["r2"], []]), ("view", [[], ["r1"]])],
                                [(i, fields[f], json.loads(v)) for i, f, v in triples],
                                [um.Ranking(n, m, s, e, st) for n, m, s, e, st in rankings])
    assert docs_of(body) == mirror


# ---- the reference's data ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_model_bulk_equals_the_mirror_on_the_reference_data(orc, name, config):
    fx = load_golden(name)
    prepared, triples, fields, rankings = model_inputs(fx, config)
    mats = [orc.Csr(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    ref = orc.train(mats, [orc.Params(500, 50, None)] * len(mats), 1)
    body, mirror = bulk_and_docs([(r.row_ptr, r.col_idx) for r in ref], prepared, triples, fields, rankings)
    assert docs_of(body) == mirror
    assert len(mirror) >= prepared[0][1].n_cols


def test_fixture_sources():
    hm, rk = load_golden("model_handmade.json"), load_golden("model_rank.json")
    assert len(hm["set_events"]) == 43 and len(rk["set_events"]) == 18
    assert {s[1]["defaultRank"] for s in rk["set_events"] if "defaultRank" in s[1]} >= {2.7, 7.15}
    t = sorted(e[3] for e in hm["events"])
    assert hm["now_ms"] - t[0] == 111 * 69_120_000 or hm["now_ms"] >= t[-1]


def test_c_program_compiles_against_the_model_structs(tmp_path):
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "model_abi_check.c")], check=True)

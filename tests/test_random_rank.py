"""Random rankings (uniqueRank, PopModel.calcRandom) on the CPU: the text rule of n · 10^-15 against Java's Double.toString
of the double, the host mirror's item set and values, and the byte-level restatement against the mirror on the reference's
data with the rank engine's own `random` entry."""
import random

import numpy as np
import pytest

from conftest import load_golden
from test_model_docs import CONFIGS, MODEL_FIXTURES, docs_of, model_inputs
from universal_recommender_b200 import ur_model as um

RANDOM_ENTRY = {"name": "uniqueRank", "type": "random"}   # examples/rank/rank-engine.json


def with_random(fx, config="rank/rank-engine.json"):
    """the fixture with the rank engine's `random` entry put back after its other rankings"""
    fx = dict(fx)
    fx["rankings"] = dict(fx["rankings"], **{config: list(fx["rankings"][config]) + [RANDOM_ENTRY]})
    return fx


def test_text_rule_is_java_double_of_the_value():
    import random_rank_oracle as ro
    rng = random.Random(15)
    edges = {0, 10**12 - 1, 10**12, 10**12 + 1, 10**15 - 1}
    for k in range(16):
        edges |= {10**k, 10**k - 1, 10**k + 1} - {10**15, 10**15 + 1}
    vals = sorted(edges)
    vals += [rng.randrange(10**15) for _ in range(1_400_000)]              # uniform: ~1 in 1000 below 10^-3
    vals += [rng.randrange(10**12) for _ in range(400_000)]                # below 10^-3: E notation
    vals += [rng.randrange(10**rng.randrange(1, 12)) for _ in range(200_000)]   # every exponent down to 10^-15
    assert len(vals) >= 2_000_000
    bad = [n for n in vals if ro.random_rank_text(n).decode() != um.java_double(n / 1e15)]
    assert bad == []
    assert ro.random_rank_text(0) == b"0.0" and ro.random_rank_text(1) == b"1.0E-15" and ro.random_rank_text(123) == b"1.23E-13"
    assert ro.random_rank_text(10**12) == b"0.001" and ro.random_rank_text(999_999_999_999) == b"9.99999999999E-4"
    assert ro.random_rank_text(500_000_000_000_000) == b"0.5"


def test_value_restatement():
    import synth
    z = np.array([0, 1, 2**63, 2**64 - 1, 0x243F6A8885A308D3], np.uint64)
    assert [um._mix64(int(x)) for x in z] == [int(x) for x in synth._mix64(z)]
    # the hash reads 8-byte words: ids across the word boundary and multi-byte UTF-8 differ from their prefixes
    ids = ["", "a", "abcdefg", "abcdefgh", "abcdefghi", "é", "☃\x00", "\x00"]
    assert len({um.id_hash(i) for i in ids}) == len(ids)
    n = [um.random_rank(f"item-{j}", 0, 10**9) for j in range(20_000)]
    assert all(0 <= x < 10**15 for x in n)
    assert 0.48 < np.mean(n) / 1e15 < 0.52
    assert um.random_rank("a", 0, 10**9) == um.random_rank("a", 0, 10**9) != um.random_rank("a", 0, 10**9 + 1)
    assert um.random_rank("a", -5, 10**9) != um.random_rank("a", 0, 10**9)


def test_rankings_for_builds_the_random_item_set():
    start, end = 1_000, 5_000
    rp = um.RankingParams("uniqueRank", "random", ["buy"], None, None, "4 seconds")
    by_name = {"buy": [("in", 1_000), ("late", 5_000), ("mid", 3_000)],
               "view": [("early", 999), ("mid", 4_999), ("viewed", 4_999)],
               "not-a-model-event": [("other", 2_000)]}
    [r] = um.rankings_for(um.rankings_params([rp], ["buy"]), by_name, end, ["buy"])
    assert (r.field, r.mode, r.start_ms, r.end_ms) == ("uniqueRank", "random", start, end)
    assert [s[0] for s in r.streams] == [["in", "late", "mid"], ["early", "mid", "viewed"], ["other"]]   # every event name
    sc = r.scores(["prop-only", "in"])
    # start inclusive, end exclusive; any event name; property items; no duplicates; out of window without a property: none
    assert list(sc) == ["in", "mid", "viewed", "other", "prop-only"]
    assert all(sc[i] == um.random_rank(i, start, end) / 1e15 for i in sc)
    docs = um.model_documents(["in"], [("buy", [[]])], [("prop-only", "color", "red"), ("early", "color", "blue")], [r])
    assert [d["id"] for d in docs] == ["in", "prop-only", "early", "mid", "viewed", "other"]
    assert docs[2] == {"id": "early", "color": "blue", "uniqueRank": um.random_rank("early", start, end) / 1e15}
    # one ranking per type: the first random entry stays, next to the others
    rs = [um.RankingParams("p", "popular"), um.RankingParams("u", "random"), um.RankingParams("u2", "random")]
    assert [r.field_name() for r in um.rankings_params(rs, ["buy"])] == ["p", "u"]
    assert um.RankingParams(None, "random").field_name() == "uniqueRank"


def test_restatement_bytes_and_precedence_for_a_random_ranking():
    import random_rank_oracle as ro
    rows = ["r1", "r2"]
    inds = [([0, 1, 1], [1])]
    fields = ["uniqueRank", "plain"]
    triples = [("r1", 0, '"prop"'), ("p", 1, "1")]
    # named like the indicator; like the property; a later one of the same name (another window, property items only)
    rank = [("buy", "random", 0, 100, [(["r2", "late"], [5, 100])]), ("uniqueRank", "random", 0, 100, [(["r2"], [1])]),
            ("uniqueRank", "random", 0, 101, [([], [])])]
    body = ro.model_bulk(inds, ["buy"], rows, [rows], fields, triples, rank)
    t = lambda i, end=100: ro.random_rank_text(um.random_rank(i, 0, end)).decode()
    lines = body.decode().split("\n")
    assert lines[1] == '{"id":"r1","buy":%s,"uniqueRank":%s}' % (t("r1"), t("r1", 101))   # property items are in every set
    assert lines[3] == '{"id":"r2","buy":%s,"uniqueRank":%s}' % (t("r2"), t("r2"))
    assert lines[5] == '{"id":"p","plain":1,"buy":%s,"uniqueRank":%s}' % (t("p"), t("p", 101))
    assert len(lines) == 7                                                                  # "late" is outside the window
    mirror = um.model_documents(rows, [("buy", [["r2"], []])], [("r1", "uniqueRank", "prop"), ("p", "plain", 1)],
                                [um.Ranking(n, m, s, e, st) for n, m, s, e, st in rank])
    assert docs_of(body) == mirror
    named_id = ro.model_bulk(inds, ["buy"], rows, [rows], fields, triples, [("id", "random", 0, 100, [(["r2"], [1])])])
    assert docs_of(named_id)[1] == {"id": "r2", "buy": []} and b'"id":0.' not in named_id


def _bulk_inputs(orc, prepared, triples, fields, rankings):
    mats = [orc.Csr(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    ref = orc.train(mats, [orc.Params(500, 50, None)] * len(mats), 1)
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    return ([(r.row_ptr, r.col_idx) for r in ref], names, rows, cols, fields,
            [(i, fields.index(f), um.property_json(v)) for i, f, v in triples],
            [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings])


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_restatement_without_random_rankings_is_model_oracle(orc, name, config):
    import model_oracle as mo
    import random_rank_oracle as ro
    args = _bulk_inputs(orc, *model_inputs(load_golden(name), config))
    assert ro.model_bulk(*args) == mo.model_bulk(*args)


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_model_bulk_equals_the_mirror_with_the_rank_engine_random_entry(orc, name):
    import random_rank_oracle as ro
    fx = with_random(load_golden(name))
    prepared, triples, fields, rankings = model_inputs(fx, "rank/rank-engine.json")
    assert [r.mode for r in rankings] == ["popular", "random"]
    inds, names, rows, cols, *_ = args = _bulk_inputs(orc, prepared, triples, fields, rankings)
    body = ro.model_bulk(*args)
    per_row = [(n, [[cols[t][int(c)] for c in ci[rp[r]:rp[r + 1]]] for r in range(len(rows))]) for t, (n, (rp, ci)) in enumerate(zip(names, inds))]
    mirror = um.model_documents(rows, per_row, triples, rankings)
    assert docs_of(body) == mirror
    ranked = [d for d in mirror if "uniqueRank" in d]
    assert len(ranked) >= len({s[0] for s in fx["set_events"]})

"""The ur_predict mirror (URAlgorithm.predict's reading of the search hits, URAlgorithm.scala:484-529): the reference's
served PredictedResult lines, one case per rule and deviation, the number normaliser's fast path against
java_double(float(text)), the batchpredict echo against a hand-written json4s restatement, the error messages, and the C
declarations."""
import math
import os
import random
import subprocess

import numpy as np
import pytest

import search_results_data as D
from conftest import ROOT
from universal_recommender_b200 import ur_predict as P
from universal_recommender_b200.ur_model import java_double


def el(hits, extra=""):
    return '{' + extra + '"hits":{"total":3,"hits":[' + ",".join(hits) + "]}}"


def test_golden_lines():
    g = D.golden_elements()
    assert len(g) == 53
    for x, e in g:
        assert P.predicted_result(e, [], False) == x["text"], (x["file"], x["line"])


def test_error_element_and_status_are_empty():
    for e in ['{"error":{"reason":"x"},"status":404}', '{"status":500,"hits":{"hits":[{"_id":"a","_score":1}]}}',
              '{"error":null,"hits":{"hits":[{"_id":"a","_score":1}]}}']:
        assert P.predicted_result(e, [], False) == '{"itemScores":[]}'
    p = P.prediction(P.loads('{"status":503}'), [], False)
    assert (p.status, p.total) == (503, -1)


def test_totals():
    assert P.prediction(P.loads(el([])), [], False).total == 3
    assert P.prediction(P.loads('{"hits":{"total":{"value":7,"relation":"eq"},"hits":[]}}'), [], False).total == 7
    assert P.prediction(P.loads('{"hits":{"hits":[]}}'), [], False).total == -1


def test_integer_score_is_a_double():
    assert P.predicted_result(el(['{"_id":"a","_score":1}', '{"_id":"b","_score":-0}']), [], False) == \
        '{"itemScores":[{"item":"a","score":1.0},{"item":"b","score":0.0}]}'


def test_ranks_present_absent_null():
    hits = ['{"_id":"a","_score":2.5,"_source":{"trendRank":3,"popRank":1.5}}', '{"_id":"b","_score":1,"_source":{"popRank":null}}',
            '{"_id":"c","_score":1}', '{"_id":"d","_score":1,"_source":{"popRank":1e-5,"popRank":"x"}}']
    assert P.predicted_result(el(hits), ["popRank", "trendRank", "popRank"], True) == (
        '{"itemScores":[{"item":"a","score":2.5,"ranks":{"popRank":1.5,"trendRank":3.0}},{"item":"b","score":1.0},'
        '{"item":"c","score":1.0},{"item":"d","score":1.0,"ranks":{"popRank":1.0E-5}}]}')
    assert P.predicted_result(el(hits), ["popRank"], False).count("ranks") == 0


@pytest.mark.parametrize("hit,msg", [
    ('{"_score":1}', "record 0 hit 0: the hit has no string _id"),
    ('{"_id":7,"_score":1}', "no string _id"),
    ('{"_id":"a","_id":"a","_score":1}', "repeated"),
    ('{"_id":"a","_score":1,"_score":2}', "repeated"),
    ('{"_id":"a"}', "_score is missing"),
    ('{"_id":"a","_score":null}', "_score is missing"),
    ('{"_id":"a","_score":1,"_source":{"popRank":true}}', "rank 'popRank' is not a number"),
    ('{"_id":"a","_score":1e400}', "out of the range"),
])
def test_hit_errors(hit, msg):
    with pytest.raises(ValueError, match=msg):
        P.predictions('{"responses":[' + el([hit]) + "]}", ["popRank"], True)


def test_body_errors():
    with pytest.raises(ValueError, match="one responses array"):
        P.predictions('{"took":1}', [], False)
    with pytest.raises(ValueError, match="hits.hits is not an array"):
        P.predictions('{"responses":[{"hits":{"hits":{}}}]}', [], False)
    with pytest.raises(ValueError, match="2 response elements for 1 records"):
        P.predictions('{"responses":[{},{}]}', [], [True])
    with pytest.raises(ValueError):
        P.predictions('{"responses":[NaN]}', [], False)


def fast_path_text(text: str):
    """the device's fast path restated: the significant digits stripped of zeros, in Java's layout; None beyond it"""
    neg = text.startswith("-")
    t = text.lstrip("-")
    mant, _, exp = t.replace("E", "e").partition("e")
    ip, _, fp = mant.partition(".")
    digits = (ip + fp).lstrip("0")
    e10 = int(exp or 0) - len(fp)
    if not digits:
        return ("-" if neg and (fp or exp) else "") + "0.0"
    s = digits.rstrip("0")
    e10 += len(digits) - len(s)
    if len(s) > 15 or abs(e10) > 22:
        return None
    n, point = len(s), len(s) + e10
    sign = "-" if neg else ""
    if -2 <= point <= 7:
        if point <= 0:
            return sign + "0." + "0" * -point + s
        if point >= n:
            return sign + s + "0" * (point - n) + ".0"
        return sign + s[:point] + "." + s[point:]
    return sign + s[0] + "." + (s[1:] or "0") + "E" + str(point - 1)


def test_number_fast_path_matches_java_double():
    forms = ["0", "-0", "1", "-17", "120", "1e3", "1E+22", "1.5e-22", "123456789012345", "-1234567890.12345", "0.001",
             "0.0009990", "9999999", "10000000", "1.0E7", "0.10000000000000001", "1234567890123456", "12345678901234567",
             "3.14159265358979323", "0.3595937192440033", "4.9e-324", "1e23"]
    rng = random.Random(2024)
    f32 = np.frombuffer(np.random.default_rng(1).integers(0, 2 ** 32, 500000, dtype=np.uint64).astype(np.uint32).tobytes(), np.float32)
    f64 = np.random.default_rng(2).standard_normal(500000) * 10.0 ** np.random.default_rng(3).integers(-30, 30, 500000)
    texts = forms + [str(x) for x in f32 if np.isfinite(x)] + [repr(float(x)) for x in f64]   # ES writes float32 scores shortest
    texts += [str(rng.randint(-10 ** 18, 10 ** 18)) for _ in range(2000)]
    fast = 0
    for t in texts:
        want = java_double(float(int(t)) if t.lstrip("-").isdigit() else float(t))
        got = fast_path_text(t)
        if got is not None:
            fast += 1
            assert got == want, t
    assert fast > 300000   # random float32 bit patterns: many exponents lie beyond +-22


def json4s_render(v, out):
    """a hand-written json4s compact rendering for the echo test (independent of ur_predict.render)"""
    if isinstance(v, P.Num):
        out.append(str(int(v)) if v.lstrip("-").isdigit() else java_double(float(v)))
    elif isinstance(v, str):
        out.append(D.P.json_string(v))
    elif isinstance(v, list) and not hasattr(v, "count") or type(v) is list:
        out.append("[")
        for i, x in enumerate(v):
            out.append("," if i else "")
            json4s_render(x, out)
        out.append("]")
    elif v is None:
        out.append("null")
    elif v is True or v is False:
        out.append("true" if v else "false")
    else:
        out.append("{")
        for i, (k, x) in enumerate(v):
            out.append(("," if i else "") + D.P.json_string(k) + ":")
            json4s_render(x, out)
        out.append("}")


def test_batchpredict_echo():
    line = ' { "user" : "u\\u00e91", "num":-0, "bias": 1.50, "big": 12345678901234567890, "e":1E2, "f":[ "a" , null,true ], "user":"x"} '
    out = []
    json4s_render(P.loads(line), out)
    assert P.batchpredict_line(line, '{"itemScores":[]}') == '{"query":' + "".join(out) + ',"prediction":{"itemScores":[]}}'
    assert "".join(out) == '{"user":"ué1","num":0,"bias":1.5,"big":12345678901234567890,"e":100.0,"f":["a",null,true],"user":"x"}'


def test_c_declarations_compile(tmp_path):
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "search_results_abi_check.c"), "-o", str(tmp_path / "sr.o")], check=True)


def test_status_range():
    assert P.prediction(P.loads('{"status":-2147483648}'), [], False).status == -2 ** 31
    with pytest.raises(ValueError, match="status"):
        P.prediction(P.loads('{"status":2147483648}'), [], False)


def test_first_source_only():
    e = el(['{"_id":"a","_score":1,"_source":{"x":1},"_source":{"popRank":2}}'])
    assert P.predicted_result(e, ["popRank"], True) == '{"itemScores":[{"item":"a","score":1.0}]}'


def test_query_lines_and_with_ranks():
    assert P.query_file_lines(b'{"a":1}\n{"b":2}\n') == [b'{"a":1}', b'{"b":2}']
    assert P.query_file_lines(b'{"a":1}\n{"b":2}') == [b'{"a":1}', b'{"b":2}']
    assert [P.line_with_ranks(x) for x in ['{"withRanks":true}', '{"withRanks":false}', '{"withRanks":null}', '{}']] == [True, False, False, False]
    for bad, msg in [('{"withRanks":1}', "not true"), ('{"withRanks":null,"withRanks":true}', "repeats"), ('[]', "not one JSON object")]:
        with pytest.raises(ValueError, match=msg):
            P.line_with_ranks(bad)


def test_batchpredict_lines_pair_line_r_with_record_r():
    qf = b'{"user":"u1","withRanks":true}\n{"user":"u2"}\n'
    hit = '{"_id":"a","_score":2,"_source":{"popRank":1}}'
    b = '{"responses":[' + el([hit]) + "," + el([hit]) + "]}"
    assert P.batchpredict_lines(qf, [b], ["popRank"]) == [
        '{"query":{"user":"u1","withRanks":true},"prediction":{"itemScores":[{"item":"a","score":2.0,"ranks":{"popRank":1.0}}]}}',
        '{"query":{"user":"u2"},"prediction":{"itemScores":[{"item":"a","score":2.0}]}}']

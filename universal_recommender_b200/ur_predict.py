"""The second half of URAlgorithm.predict: Elasticsearch search hits turned into the engine's PredictedResult, restated on
the host as the mirror CcoContext.search_results is checked against.

For one query the reference (URAlgorithm.scala:484-529, EsClient.scala:370-385, Serving.scala:25-29) does this:
  * EsClient.search: a status other than 200 gives None, and None gives PredictedResult(Array.empty);
  * every element of hits.hits, in order, becomes ItemScore(item = hit \\ "_id", score = (hit \\ "_score").extract[Double]);
    a JSON integer is a JInt, so a score of 1 is 1.0;
  * with query.withRanks == Some(true) each ItemScore gets ranks: one entry per rankingsParams field name, from the hit's
    source, and ranks = Some(map) only when the map is non-empty;
  * Serving.serve returns the head of the predictions: the identity for one algorithm.
PredictionIO renders the result with json4s compact(render(Extraction.decompose(...))):
{"itemScores":[{"item":"...","score":<Double>,"ranks":{"<name>":<Double>,...}}]}, a None member left out, strings through
json4s' quote (ur_query.json_string) and doubles through Double.toString (ur_model.java_double).

Deviations (INTEGRATION.md lists them):
  1. withRanks reads "_source"; the reference reads hit \\ "source", a field that never exists, so every withRanks query
     of the reference throws;
  2. a ranking field absent from _source, or null, is left out of ranks (items without events in a ranking's window have
     no rank field); with no field left, ranks is omitted.  A rank that is present but not a JSON number is an error;
  3. ranks are in ur_model.rankings_params order (Scala's groupBy gives none); a name listed twice is one member;
  4. an _msearch response element with an "error" member, or a "status" other than 200, is the `case _ =>` branch: an
     empty itemScores.  Its status is reported, not raised.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Optional, Sequence

from .ur_model import java_double
from .ur_query import json_string


class Num(str):
    """the text of a JSON number, as the response spells it"""


def _constant(name):
    raise ValueError(f"{name} is not JSON")


class _Obj(list):
    """a JSON object as its (name, value) pairs, in order, repeated names kept"""

    def get(self, name, default=None):
        for k, v in self:
            if k == name:
                return v
        return default

    def count(self, name):   # noqa: A003 -- list.count by member name
        return sum(1 for k, _ in self if k == name)


def loads(text) -> object:
    """json.loads keeping number texts (Num) and objects as ordered pairs (_Obj); NaN and Infinity are refused"""
    if isinstance(text, (bytes, bytearray, memoryview)):
        text = bytes(text).decode("utf-8", "surrogatepass")
    return json.loads(text, parse_float=Num, parse_int=Num, parse_constant=_constant, object_pairs_hook=_Obj)


def number_value(text: str) -> float:
    """the double nearest to a JSON number's text (Python's float() rounds exactly, integer literals of any length
    included); an integer literal is a JInt, so -0 is 0.0; out of range is a ValueError"""
    v = float(text)
    if v == 0 and _is_integer(text):
        v = 0.0
    if v in (float("inf"), float("-inf")):
        raise ValueError(f"{text} is out of the range of a double")
    return v


def _is_integer(text: str) -> bool:
    return not any(ch in text for ch in ".eE")


def number_text(text: str) -> str:
    """Double.toString of a JSON number's value: json4s extract[Double] then render"""
    return java_double(number_value(text))


@dataclass
class Prediction:
    """one _msearch response element read as the reference reads its search result"""
    status: int                       # the element's "status", 0 when it has none
    total: int                        # hits.total (ES <= 6: a number, ES 7: {"value": ...}), -1 when absent
    items: list = field(default_factory=list)    # [(item id, score text)]
    scores: list = field(default_factory=list)   # [float]
    ranks: list = field(default_factory=list)    # [{name: float}] per hit, names in ranking order, {} without ranks
    rank_texts: list = field(default_factory=list)  # [{name: rank number text}]

    def text(self) -> str:
        """the PredictedResult as PredictionIO serves it"""
        parts = []
        for (item, score), rk in zip(self.items, self.rank_texts):
            s = '{"item":' + json_string(item) + ',"score":' + number_text(score)
            if rk:
                s += ',"ranks":{' + ",".join(json_string(n) + ":" + number_text(t) for n, t in rk.items()) + "}"
            parts.append(s + "}")
        return '{"itemScores":[' + ",".join(parts) + "]}"


def _unique(names: Sequence[str]) -> list[str]:
    return list(dict.fromkeys(names))


def prediction(element, ranking_names: Sequence[str], with_ranks: bool, where: str = "record 0") -> Prediction:
    """one parsed response element (loads) -> Prediction; ValueError names `where` and the hit"""
    if not isinstance(element, _Obj):
        raise ValueError(f"{where}: the response element is not an object")
    status = element.get("status")
    total = -1
    p = Prediction(status=0, total=-1)
    if status is not None:
        if not isinstance(status, Num) or not _is_integer(status) or not -2 ** 31 <= int(status) < 2 ** 31:
            raise ValueError(f"{where}: status is not an integer")
        p.status = int(status)
    hits = element.get("hits")
    if isinstance(hits, _Obj):
        t = hits.get("total")
        if isinstance(t, _Obj):
            t = t.get("value")
        if isinstance(t, Num) and _is_integer(t) and -2 ** 63 < int(t) < 2 ** 63:
            total = int(t)
    p.total = total
    if element.count("error") or (status is not None and p.status != 200):
        return p
    arr = hits.get("hits") if isinstance(hits, _Obj) else None
    if arr is None:
        return p
    if not isinstance(arr, list) or isinstance(arr, _Obj):
        raise ValueError(f"{where}: hits.hits is not an array")
    names = _unique(ranking_names)
    for h, hit in enumerate(arr):
        at = f"{where} hit {h}"
        if not isinstance(hit, _Obj):
            raise ValueError(f"{at}: the hit is not an object")
        if hit.count("_id") > 1 or hit.count("_score") > 1:
            raise ValueError(f"{at}: a repeated _id or _score")
        item = hit.get("_id")
        if not isinstance(item, str) or isinstance(item, Num):
            raise ValueError(f"{at}: the hit has no string _id")
        score = hit.get("_score")
        if not isinstance(score, Num):
            raise ValueError(f"{at}: _score is missing, null or not a number")
        rk, rt = {}, {}
        source = hit.get("_source")
        if with_ranks and isinstance(source, _Obj):
            for n in names:
                vals = [v for k, v in source if k == n]
                if not vals or vals[0] is None:
                    continue
                v = vals[0]
                if not isinstance(v, Num):
                    raise ValueError(f"{at}: the rank {n!r} is not a number")
                rk[n], rt[n] = number_value(v), v
        p.items.append((item, score))
        p.scores.append(number_value(score))
        p.ranks.append(rk)
        p.rank_texts.append(rt)
    return p


def predicted_result(element, ranking_names: Sequence[str], with_ranks: bool) -> str:
    """the PredictedResult JSON of one _msearch response element (bytes, str or parsed)"""
    if isinstance(element, (bytes, bytearray, memoryview, str)):
        element = loads(element)
    return prediction(element, ranking_names, with_ranks).text()


def predictions(body, ranking_names: Sequence[str], with_ranks=False, first_record: int = 0) -> list[Prediction]:
    """every element of one _msearch response body, in order.  with_ranks: a bool for every record, or one per record.
    Errors name the record (numbered from first_record) and the hit."""
    top = loads(body)
    if not isinstance(top, _Obj) or top.count("responses") != 1 or not isinstance(top.get("responses"), list) \
            or isinstance(top.get("responses"), _Obj):
        raise ValueError("the top level is not an object with one responses array")
    els = top.get("responses")
    flags = [bool(with_ranks)] * len(els) if isinstance(with_ranks, bool) else list(with_ranks)
    if len(flags) != len(els):
        raise ValueError(f"{len(els)} response elements for {len(flags)} records")
    return [prediction(e, ranking_names, f, f"record {first_record + r}") for r, (e, f) in enumerate(zip(els, flags))]


def ranking_names(ap) -> list[str]:
    """the ranking field names of the algorithm params, in ur_model.rankings_params order, each once"""
    from .ur_model import rankings_params
    return _unique(rp.field_name() for rp in rankings_params(ap.rankings, ap.model_event_names()))


def query_file_lines(query_file) -> list[bytes]:
    """the lines of a batchpredict query file (bytes, or a path, or already a list of lines): a final newline opens no
    line, as cco_query_file_read splits them"""
    if isinstance(query_file, (list, tuple)):
        return [x.encode("utf-8", "surrogatepass") if isinstance(x, str) else bytes(x) for x in query_file]
    if isinstance(query_file, (str,)) or hasattr(query_file, "__fspath__"):
        with open(query_file, "rb") as f:
            query_file = f.read()
    data = bytes(query_file)
    lines = data.split(b"\n")
    return lines[:-1] if data.endswith(b"\n") else lines


def line_with_ranks(line, where: str = "record 0") -> bool:
    """a query line's withRanks as cco_query_file_read reads it: true or false, null = absent, at most once"""
    q = loads(line)
    if not isinstance(q, _Obj):
        raise ValueError(f"{where}: the query line is not one JSON object")
    if q.count("withRanks") > 1:
        raise ValueError(f"{where}: the query line repeats withRanks")
    w = q.get("withRanks")
    if w is not None and not isinstance(w, bool):
        raise ValueError(f"{where}: the query line's withRanks is not true, false or null")
    return bool(w)


def batchpredict_lines(query_file, bodies, ranking_names: Sequence[str]) -> list[str]:
    """the batchpredict output lines (without newlines) of a query file and the _msearch response bodies to its queries:
    line r pairs with record r, whose withRanks is its line's"""
    lines = query_file_lines(query_file)
    out, r = [], 0
    for body in bodies:
        n = len(loads(body).get("responses") or [])
        flags = [line_with_ranks(lines[r + k], f"record {r + k}") for k in range(n)]
        for k, p in enumerate(predictions(body, ranking_names, flags, first_record=r)):
            out.append(batchpredict_line(lines[r + k], p.text()))
        r += n
    return out


def batchpredict_line(line, prediction_text: str) -> str:
    """[RECALL] PredictionIO's BatchPredict output line, compact(render(("query" -> parse(line)) ~ ("prediction" ->
    decompose(prediction)))): the query re-rendered by json4s (insignificant whitespace dropped, strings decoded and
    re-quoted, integer literals as BigInt prints them, other numbers as Double.toString, member order and repeated members
    kept), without the final newline"""
    return '{"query":' + render(loads(line)) + ',"prediction":' + prediction_text + "}"


def render(v) -> str:
    """json4s compact rendering of a parsed value"""
    if isinstance(v, Num):
        return ("0" if v == "-0" else str(v)) if _is_integer(v) else number_text(v)   # BigInt prints a JSON integer as it is
    if isinstance(v, str):
        return json_string(v)
    if isinstance(v, _Obj):
        return "{" + ",".join(json_string(k) + ":" + render(x) for k, x in v) + "}"
    if isinstance(v, list):
        return "[" + ",".join(render(x) for x in v) + "]"
    if v is None:
        return "null"
    return "true" if v else "false"

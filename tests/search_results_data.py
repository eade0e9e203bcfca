"""Synthetic Elasticsearch _msearch responses for the search-results tests: the golden PredictedResult lines turned back
into response elements, and seeded random bodies that reach the reader's edges (escapes, pretty printing, unknown and
permuted members, ranks present / absent / null, error elements, ES 6 and ES 7 totals)."""
import json
import random

from conftest import load_golden
from universal_recommender_b200 import ur_predict as P


def index_sources() -> dict:
    """item id -> its _source text in the handmade model index"""
    body = load_golden("item_queries_handmade.json")["index"]
    src = {}
    for line in body.splitlines()[1::2]:
        d = json.loads(line)
        src[d["id"]] = line
    return src


def golden_elements():
    """[(fixture entry, element text)]: hits in the line's order, _score with the line's own text"""
    src = index_sources()
    out = []
    for g in load_golden("predicted_results_handmade.json")["results"]:
        hits = []
        for h in P.loads(g["text"]).get("itemScores"):
            item, score = h.get("item"), h.get("score")
            s = '{"_index":"urindex","_type":"items","_id":' + json.dumps(item) + ',"_score":' + score
            if item in src:
                s += ',"_source":' + src[item]
            hits.append(s + "}")
        el = '{"took":3,"timed_out":false,"hits":{"total":' + str(len(hits)) + ',"max_score":null,"hits":[' + ",".join(hits) + ']},"status":200}'
        out.append((g, el))
    return out


def pretty(text: str) -> str:
    """text re-indented as ES's ?pretty does (newlines and two-space indents, " : "), strings and numbers untouched"""
    out, depth, in_str, esc = [], 0, False, False
    for ch in text:
        if in_str:
            out.append(ch)
            if esc:
                esc = False
            elif ch == "\\":
                esc = True
            elif ch == '"':
                in_str = False
        elif ch == '"':
            in_str = True
            out.append(ch)
        elif ch in "{[":
            depth += 1
            out.append(ch + "\n" + "  " * depth)
        elif ch in "}]":
            depth -= 1
            out.append("\n" + "  " * depth + ch)
        elif ch == ",":
            out.append(",\n" + "  " * depth)
        elif ch == ":":
            out.append(" : ")
        else:
            out.append(ch)
    return "".join(out)


def body(elements, pretty_print=False) -> bytes:
    """one _msearch response body of element texts"""
    b = '{"took":5,"responses":[' + ",".join(elements) + "]}"
    return ((pretty(b) + "\n") if pretty_print else b).encode("utf-8", "surrogatepass")


ID_EDGES = ["", 'a"b', "back\\slash", "{}[]:,\"", "été", "\U0001F600 smile", "😀", "tab\tnl\n",
            "\u0085 ", "x" * 1500, "\\" * 33, "\\\\\\\"", "ctl\u0001"]


def _num_text(rng) -> str:
    k = rng.random()
    if k < 0.4:
        return repr(float(rng.random() * 10 ** rng.randint(-5, 5))) if rng.random() < 0.5 else str(float.__repr__(float(__import__("numpy").float32(rng.random() * 20))))
    if k < 0.55:
        return str(rng.randint(-1000, 10 ** 6))
    if k < 0.7:
        return f"{rng.randint(1, 999999)}e{rng.randint(-30, 30)}"
    if k < 0.85:
        return "0." + "".join(rng.choice("0123456789") for _ in range(rng.randint(1, 20))) + "1"
    return rng.choice(["0", "-0", "0.0", "-0.0", "1E+2", "1e-7", "123456789012345678901234567890", "0.10000000000000001",
                       "9007199254740993", "4.9e-324", "1.7976931348623157e308", "2.2250738585072014E-308"])


def random_element(rng, names, n_hits=None, pretty_ws=False, errors=True) -> str:
    """one response element with random hits; ranks present / absent / null; members permuted; unknown members"""
    if errors and rng.random() < 0.08:
        return rng.choice(['{"error":{"type":"index_not_found_exception","reason":"no such index [x]"},"status":404}',
                           '{"status":500,"error":"boom","hits":{"hits":[1,2]}}', '{"status":429,"hits":{"total":0,"hits":[]}}'])
    n = rng.choice([0, 1, 2, 3, 20, 31, 32, 33]) if n_hits is None else n_hits
    hits = []
    for h in range(n):
        iid = rng.choice(ID_EDGES) if rng.random() < 0.3 else f"item-{rng.randint(0, 10 ** 6)}"
        src = [("id", json.dumps(iid)), ("purchase", json.dumps([f"p{rng.randint(0, 99)}" for _ in range(rng.randint(0, 30))])),
               ("categories", json.dumps(["a\\\"b", "{[,:]}"]))]
        for nm in names:
            k = rng.random()
            if k < 0.6:
                src.append((nm, _num_text(rng)))
            elif k < 0.75:
                src.append((nm, "null"))
        rng.shuffle(src)
        mem = [("_index", '"urindex"'), ("_type", '"items"'), ("_id", json.dumps(iid)), ("_score", _num_text(rng)),
               ("_source", "{" + ",".join(json.dumps(k) + ":" + v for k, v in src) + "}")]
        if rng.random() < 0.3:
            mem.append(("sort", "[1.5,\"x\"]"))
        if rng.random() < 0.2:
            mem.append(("_ignored", "[]"))
        rng.shuffle(mem)
        sep = "\n      " if pretty_ws else ""
        hits.append("{" + sep + ("," + sep).join(json.dumps(k) + " : " * pretty_ws + ":" * (not pretty_ws) + v for k, v in mem) + sep + "}")
    total = rng.choice([str(n), '{"value":' + str(n) + ',"relation":"eq"}', None])
    hm = [("max_score", "1.0"), ("hits", "[" + ",".join(hits) + "]")] + ([("total", total)] if total else [])
    rng.shuffle(hm)
    em = [("took", "1"), ("timed_out", "false"), ("hits", "{" + ",".join(json.dumps(k) + ":" + v for k, v in hm) + "}")]
    if rng.random() < 0.7:
        em.append(("status", "200"))
    rng.shuffle(em)
    return "{" + ",".join(json.dumps(k) + ":" + v for k, v in em) + "}"


def random_elements(seed, n, names):
    rng = random.Random(seed)
    return [random_element(rng, names, pretty_ws=rng.random() < 0.2) for _ in range(n)]

"""cco_search_results' number path on the H100 against the exact references of number_edges: every directed text as a
_score, as a rank beside ranks of the other path in the same hit, and as a value nested in batchpredict query lines split
over several bodies; the doubles bit for bit, the text byte for byte (against the ur_predict mirror and against
java_double directly), and n_exact equal to the texts the routing rule sends to the host.  Every text out of the range of
a double is an error in each position but a query line's integer literal, which is echoed verbatim.  A fuzz body of 10^6
numbers, and the integer fields of both readers (status, hits.total, _shards.failed) against their mirrors."""
import math
import random

import numpy as np
import pytest

import number_edges as E
import search_results_data as D
from test_gpu_predicted_results import expect_equal
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200 import ur_predict as P

pytestmark = pytest.mark.gpu
SETS = E.sets()
NAMES = ["r0", "r1", "r2", "r3", "r4"]   # r4 is never present: a NaN column


def in_range(name):
    return [t for t, _ in SETS[name] if E.value(t) is not None]


def n_exact(texts) -> int:
    return sum(E.route(t) == E.EXACT for t in texts)


def bits(xs) -> np.ndarray:
    return np.array(xs, np.float64).view(np.uint64)


def records_of(items, per=40):
    return [items[i:i + per] for i in range(0, len(items), per)]


def score_body(texts):
    els = ['{"hits":{"hits":[' + ",".join('{"_id":"h%d","_score":%s}' % (i, t) for i, t in enumerate(r)) + "]}}" for r in records_of(texts)]
    return D.body(els)


@pytest.mark.parametrize("name", list(SETS))
def test_scores(ctx, name):
    texts = in_range(name)
    b = score_body(texts)
    res = ctx.search_results(b, [])
    assert np.array_equal(res.scores.view(np.uint64), bits([E.value(t) for t in texts]))
    assert res.records() == ['{"itemScores":[' + ",".join('{"item":"h%d","score":%s}' % (i, E.java(t)) for i, t in enumerate(r)) + "]}"
                             for r in records_of(texts)]
    expect_equal(res, P.predictions(b, [], False))
    assert res.n_exact == n_exact(texts)


def rank_hits(texts, seed):
    """every text once as a rank r0..r3, shuffled so fast and exact ranks share hits; a slot with no text is null or
    absent -> [(source members, {name: text})]"""
    rng = random.Random(seed)
    items = texts + [None] * (len(texts) // 7 + 1)
    rng.shuffle(items)
    hits = []
    for i in range(0, len(items), 4):
        mem, got = [], {}
        for k, t in enumerate(items[i:i + 4]):
            if t is not None:
                mem.append('"r%d":%s' % (k, t))
                got["r%d" % k] = t
            elif rng.random() < 0.5:
                mem.append('"r%d":null' % k)
        rng.shuffle(mem)
        hits.append((mem, got))
    return hits


@pytest.mark.parametrize("name", list(SETS))
def test_ranks(ctx, name):
    texts = in_range(name)
    hits = rank_hits(texts, name)
    hit = '{"_id":"h","_score":1,"_source":{%s}}'
    b = D.body(['{"hits":{"hits":[' + ",".join(hit % ",".join(m) for m, _ in r) + "]}}" for r in records_of(hits)])
    res = ctx.search_results(b, NAMES, with_ranks=True)
    want = [[E.value(g[n]) if n in g else math.nan for n in NAMES] for _, g in hits]
    assert np.array_equal(res.ranks.view(np.uint64), bits(want))
    ranks_of = [",".join('"%s":%s' % (n, E.java(g[n])) for n in NAMES if n in g) for _, g in hits]
    item = ['{"item":"h","score":1.0' + (',"ranks":{%s}' % t if t else "") + "}" for t in ranks_of]
    assert res.records() == ['{"itemScores":[' + ",".join(r) + "]}" for r in records_of(item)]
    expect_equal(res, P.predictions(b, NAMES, True))
    assert res.n_exact == n_exact(texts)
    paths = [{E.route(t) for t in g.values()} for _, g in hits]
    if {p for _, p in SETS[name]} == {E.FAST, E.EXACT}:
        assert {E.FAST, E.EXACT} in paths, "no hit holds ranks of both paths"


def echo(t: str) -> str:
    """json4s' rendering of a number: an integer literal as BigInt prints it, anything else through Double.toString"""
    if E.parts(t)[4]:
        return "0" if t == "-0" else t
    return E.java(t)


def query_lines(texts, seed):
    """lines holding 1..6 texts each, nested in arrays and objects, with lines holding none between them; the first and
    the last line hold texts -> (lines, their echoes)"""
    rng = random.Random(seed)
    nest = ["%s", '{"b":%s}', "[[%s]]", '{"c":[1,{"d":%s}]}']
    lines, echoes, i, r = [], [], 0, 0
    while i < len(texts):
        if r % 3 == 1 and i + 1 < len(texts):
            mem = '{"user":"u%d","n":[1,2.5,-0.0,"x"],"withRanks":false}' % r   # fast-path numbers only
            lines.append(mem)
            echoes.append(mem)
        else:
            chunk = texts[i:i + rng.randint(1, 6)]
            i += len(chunk)
            fmt = [nest[(k + r) % len(nest)] for k in range(len(chunk) - 1)]
            for f in (lambda x: x, echo):
                line = '{"user":"u%d","a":[%s],"z":%s}' % (r, ",".join(p % f(t) for p, t in zip(fmt, chunk)), f(chunk[-1]))
                (lines if f is not echo else echoes).append(line)
        r += 1
    return lines, echoes


def line_texts(name):
    """a set's texts that a query line takes: those in range, and integer literals of any size"""
    return [t for t, _ in SETS[name] if E.value(t) is not None or E.parts(t)[4]]


@pytest.mark.parametrize("name", list(SETS))
def test_batchpredict_echo(ctx, name):
    texts = line_texts(name)
    lines, echoes = query_lines(texts, name)
    n = len(lines)
    cuts = sorted({0, n, n // 5, n // 2, n // 2 + 1, n - 1} & set(range(n + 1)))
    parts = [(a, b) for a, b in zip(cuts, cuts[1:]) if b > a]
    el = '{"hits":{"hits":[{"_id":"a","_score":1.5}]}}'
    bodies = [D.body([el] * (b - a)) for a, b in parts]
    qf = ("\n".join(lines) + "\n").encode()
    res = ctx.search_results(bodies, [], counts=[b - a for a, b in parts], query_lines=qf)
    want = ['{"query":%s,"prediction":{"itemScores":[{"item":"a","score":1.5}]}}' % e for e in echoes]
    assert res.records() == want
    assert res.text().decode().splitlines() == want
    assert P.batchpredict_lines(qf, bodies, []) == want
    assert res.n_exact == sum(E.route(t) == E.EXACT and not E.parts(t)[4] for t in texts)


@pytest.mark.parametrize("name", [k for k, v in SETS.items() if any(E.value(t) is None for t, _ in v)])
def test_out_of_range_is_an_error_in_every_position(ctx, name):
    for t in [t for t, _ in SETS[name] if E.value(t) is None]:
        b = score_body(["1.5", t, "2"])
        with pytest.raises(N.CcoInvalidArgument, match="range"):
            ctx.search_results(b, [])
        with pytest.raises(ValueError):
            P.predictions(b, [], False)
        b = D.body(['{"hits":{"hits":[{"_id":"h","_score":1,"_source":{"r0":0.3,"r1":%s,"r2":0.30000000000000004}}]}}' % t])
        with pytest.raises(N.CcoInvalidArgument, match="range"):
            ctx.search_results(b, NAMES, with_ranks=True)
        with pytest.raises(ValueError):
            P.predictions(b, NAMES, True)
        if E.parts(t)[4]:
            continue   # a query line's integer literal is a BigInt: test_batchpredict_echo
        qf = ('{"user":"ok","x":0.1}\n{"user":"u","a":[0.30000000000000004,{"b":%s}]}\n' % t).encode()
        b = D.body(['{"hits":{"hits":[]}}'] * 2)
        with pytest.raises(N.CcoInvalidArgument, match="record 1: the query line's .* is out of the range of a double"):
            ctx.search_results(b, [], query_lines=qf)
        with pytest.raises(ValueError, match="out of the range"):
            P.batchpredict_lines(qf, [b], [])


def test_fuzz_a_million_numbers_in_one_body(ctx):
    texts = E.fuzz(10 ** 6)
    K = 4
    hits = ['{"_id":"f","_score":%s,"_source":{%s}}' % (texts[i], ",".join('"r%d":%s' % (k, texts[i + 1 + k]) for k in range(K)))
            for i in range(0, len(texts), K + 1)]   # a score and K ranks each
    b = D.body(['{"hits":{"hits":[' + ",".join(r) + "]}}" for r in records_of(hits, 100)])
    res = ctx.search_results(b, NAMES[:K], with_ranks=True)
    vals = [E.value(t) for t in texts]
    assert np.array_equal(res.scores.view(np.uint64), bits(vals[0::K + 1]))
    assert np.array_equal(res.ranks.view(np.uint64), bits([vals[i + 1:i + K + 1] for i in range(0, len(vals), K + 1)]))
    assert res.n_exact == n_exact(texts) and 0 < res.n_exact < len(texts)
    expect_equal(res, P.predictions(b, NAMES[:K], True))


# ---- integer fields ----------------------------------------------------------------------------------------------------------
def expect_same_outcome(ctx, b, names=()):
    try:
        want = P.predictions(b, list(names), False)
    except ValueError:
        with pytest.raises(N.CcoInvalidArgument):
            ctx.search_results(b, list(names))
        return
    expect_equal(ctx.search_results(b, list(names)), want)


@pytest.mark.parametrize("s", E.STATUS)
def test_status_agrees_with_the_mirror(ctx, s):
    expect_same_outcome(ctx, D.body([E.status_element(s)]))


@pytest.mark.parametrize("t", E.TOTAL)
def test_hits_total_agrees_with_the_mirror(ctx, t):
    for el in E.total_elements(t):
        expect_same_outcome(ctx, D.body([el, '{"hits":{"total":5,"hits":[]}}']))


def index_outcome(ctx, page):
    """(body, n_docs, total) of the device and of the mirror, or the error's message"""
    try:
        want = um.index_from_pages([page])
    except ValueError as e:
        want = str(e).split(": ")[-1]
    try:
        with ctx.index_pages() as r:
            r.append(page)
            body = r.finish()
            got = (body, r.n_docs, r.total)
    except N.CcoInvalidArgument as e:
        got = str(e)
    return got, want


INDEX_PAGES = [E.shards_page(f) for f in E.SHARDS_FAILED] + [x.encode() for t in E.TOTAL for x in E.total_elements(t)]


@pytest.mark.parametrize("page", INDEX_PAGES, ids=range(len(INDEX_PAGES)))
def test_index_page_integers_agree_with_the_mirror(ctx, page):
    got, want = index_outcome(ctx, page)
    if isinstance(want, str):
        assert isinstance(got, str) and want in got, (got, want)
    else:
        assert got == want

"""The model index writer on the H100 at its edges (cco_pop_model, cco_format_model, cco_rerank_model; the kernels of
csrc/cco_format.cuh and k_member_info): events on PopModel's bucket edges through three routes, rank number text at every
magnitude, indicator arrays and old documents of 0, 1, 31, 32, 33, 64 and 65 elements, and the property sort at group
counts next to a power of two.  Every comparison is exact: bytes, or Python ints."""
import json
import time

import numpy as np
import pytest
import torch

import model_oracle as mo
import popmodel_ref as ref
import popmodel_shapes as shp
import universal_recommender_b200 as ur
from universal_recommender_b200 import _native
from test_gpu_format_model import format_both
from test_gpu_rerank_model import rerank_both
from test_model_docs import docs_of
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu

TINY = [(2, 3, np.array([0, 2, 3], np.int64), np.array([0, 1, 1], np.int32))]     # two users, three items
WARP_EDGES = (0, 1, 31, 32, 33, 64, 65)


# ---- 1. PopModel shapes through cco_pop_model, cco_format_model and cco_rerank_model ----------------------------------------
SHAPES = shp.shapes()
GROUPS = [SHAPES[q:q + _native.MAX_RANKINGS] for q in range(0, len(SHAPES), _native.MAX_RANKINGS)]   # one model call scores 8 rankings


def _string_route_inputs(group):
    """item j of every shape -> the id ids[j]; other ids come first in the row dictionary and the property section, and
    the last item is introduced there too, so that no item's group number in the key column is its index j"""
    n_max = max(s[4] for s in group)
    ids = [f"i{j}" for j in range(n_max)]
    rows = ["row-without-events", ids[min(1, n_max - 1)], "zz"]
    triples = [("p-first", "f", 1), (ids[n_max - 1], "f", 2), ("p-second", "f", 3)]
    rankings, wants = [], []
    for k, shape in enumerate(group):
        name, mode, start, end, n, items, times = shp.in_range(shape)
        half = len(items) // 2         # two streams per ranking, as two event names give
        rankings.append(um.Ranking(f"r{k}", mode, start, end, [([ids[j] for j in items[:half]], times[:half]),
                                                               ([ids[j] for j in items[half:]], times[half:])]))
        wants.append({ids[j]: v for j, v in ref.pop_model(mode, items, times, start, end).items()})
    return ids, rows, triples, rankings, wants


def _scores_in_body(body, n_rankings):
    got = [dict() for _ in range(n_rankings)]
    for doc in docs_of(body):
        for k in range(n_rankings):
            if f"r{k}" in doc:
                v = doc[f"r{k}"]
                assert isinstance(v, float) and v == int(v)
                got[k][doc["id"]] = int(v)
    return got


@pytest.mark.parametrize("group", GROUPS, ids=[f"{g[0][0]}..{g[-1][0]}" for g in GROUPS])
def test_popmodel_shapes_through_three_routes(ctx, group):
    for name, mode, start, end, n, items, times in group:
        want = ref.pop_model(mode, *shp.in_range((name, mode, start, end, n, items, times))[5:], start, end)
        got = ctx.pop_model(mode, items, times, n, start, end)
        assert all(v == int(v) for v in got.values()), name
        assert {j: int(v) for j, v in got.items()} == want, name
    ids, rows, triples, rankings, wants = _string_route_inputs(group)
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    jt = [(i, f, um.property_json(v)) for i, f, v in triples]
    got, want = format_both(ctx, TINY, [(500, 50, None)], ["buy"], rows, [rows], ["f"], jt, rk)
    assert got == want
    assert _scores_in_body(got, len(group)) == wants, [s[0] for s in group]
    old = (b'{"index":{"_id":"i0"}}\n{"id":"i0","keep":[1],"r0":-77.0}\n{"index":{"_id":"old-only"}}\n{"r1":5.0}\n')
    again = rerank_both(ctx, old, triples, rankings)
    fresh = _scores_in_body(again, len(group))
    for k, w in enumerate(wants):         # an old rank member stays where the new ranking has no score
        stale = {"i0": -77} if k == 0 and "i0" not in w else {"old-only": 5} if k == 1 else {}
        assert fresh[k] == {**w, **stale}, group[k][0]


# ---- 2. rank text end to end: items with ten million events --------------------------------------------------------------------
COUNTS = (9_999_999, 10_000_000, 10_000_001, 12_345_678)
# events of each item per bucket, oldest first; every mode's buckets add up to COUNTS
BUCKETS = {
    "popular": [(n,) for n in COUNTS],
    "trending": [(9_999_998, 1), (9_999_999, 1), (10_000_000, 1), (12_172_839, 172_839)],       # .., -9999999, -1.2E7
    "hot": [(9_999_997, 1, 1), (1, 9_999_998, 1), (1_666_667, 6_666_667, 1_666_667), (1, 12_345_676, 1)],
}


def check_rank_text(text: bytes, v: int):
    """the text against the restatement, and independently: it parses back to v, and it is Java's layout of the shortest
    digits of the double (Python's repr digits)"""
    assert text == mo.java_double_int(v), v
    assert float(text) == v and int(float(text)) == v, v
    assert text.decode() == um.java_double(float(v)), v
    assert len(text) <= 25


def test_rank_text_of_ten_million_event_items(ctx):
    if torch.cuda.mem_get_info(0)[0] < 8 << 30:
        pytest.skip("needs 8 GB of free device memory")
    item_bytes = np.frombuffer(b"abcd", np.uint8)
    total = sum(COUNTS)
    col = np.repeat(item_bytes, COUNTS)                  # one byte per id: a's events, then b's, c's, d's
    off = np.arange(total + 1, dtype=np.int64)
    rows = ["d", "row-without-events", "a"]              # b and c get documents of their own, after the rows
    order = rows + ["b", "c"]
    res, h = ctx.train_csr(TINY, [(500, 50, None)], 1, keep=True)
    try:
        plain = ctx.format_es_bulk(h, ["buy"], rows, [rows]).split(b"\n")
        for mode in ("popular", "trending", "hot"):
            nb = len(BUCKETS[mode][0])
            times = np.concatenate([np.repeat(np.arange(nb, dtype=np.int64), b) for b in BUCKETS[mode]])   # bucket b = [b, b + 1)
            assert len(times) == total and [sum(b) for b in BUCKETS[mode]] == list(COUNTS)
            t0 = time.perf_counter()
            got = ctx.format_model(h, ["buy"], rows, [rows], None, [("rank", mode, 0, nb, [(off, col, times)])])
            seconds = time.perf_counter() - t0
            want_scores = ref.pop_model(mode, [i for i in "abcd" for _ in range(nb)], list(range(nb)) * 4, 0, nb,
                                        [n for b in BUCKETS[mode] for n in b])
            assert len(want_scores) == 4 and (mode == "popular" or min(want_scores.values()) <= -10_000_000)
            want = bytearray()
            for d, item in enumerate(order):
                source = plain[2 * d + 1][:-1] if d < len(rows) else b'{"id":"%s"' % item.encode()
                rank = b',"rank":' + mo.java_double_int(want_scores[item]) if item in want_scores else b""
                want += b'{"index":{"_id":"%s"}}\n' % item.encode() + source + rank + b"}\n"
            assert got == bytes(want), mode
            for doc_line in got.split(b"\n")[1::2]:
                doc = json.loads(doc_line)
                if doc["id"] in want_scores:
                    text = doc_line[doc_line.index(b'"rank":') + 7:-1]
                    check_rank_text(text, want_scores[doc["id"]])
            print(f"[rank text] {mode}: {total} events, format_model {seconds:.2f} s")
    finally:
        ctx.free_result(h)


# ---- 3. rank text exhaustively: java_double_text once per value (cco_debug_rank_text) ---------------------------------------
def _texts(ctx, values, scale):
    off, b = ctx.debug_rank_text(values, scale)
    raw = b.tobytes()
    assert len(off) == len(values) + 1 and off[0] == 0
    return [raw[off[i]:off[i + 1]] for i in range(len(values))]


def test_rank_text_of_integers_at_every_magnitude(ctx):
    edge = [0, 2 ** 53 - 1, -(2 ** 53 - 1)]
    for k in range(16):
        edge += [s * (10 ** k + d) for s in (1, -1) for d in (-1, 0, 1)]
    zeros = [10_203_040, 100_000_001, 120_000_000, 1_000_000_100, 12_345_678_900_000, 9_007_199_254_740_990, 10_000_000_000_001,
             90_000_000, 1_230_000, 9_999_999_999_999_990, 1_000_000_000_000_001 * 9, 20_000_000_000_000, 5_050_505_050_505_050]
    zeros = [v for v in zeros if v < 2 ** 53]
    edge += zeros + [-v for v in zeros]
    rng = np.random.default_rng(3)
    mag = np.floor(10.0 ** rng.uniform(0, np.log10(2.0 ** 53), 1_000_000)).astype(np.int64)     # log-uniform in magnitude
    rand = (np.minimum(mag, 2 ** 53 - 1) * rng.choice([-1, 1], len(mag))).tolist()
    values = edge + rand
    texts = _texts(ctx, values, 0)
    assert {len(str(abs(v))) for v in rand} == set(range(1, 17))
    for v, text in zip(values, texts):
        check_rank_text(text, v)
    assert texts[:3] == [b"0.0", b"9.007199254740991E15", b"-9.007199254740991E15"]
    assert _texts(ctx, [9_999_999, 10_000_000, -12_000_000, 12_345_678], 0) == [b"9999999.0", b"1.0E7", b"-1.2E7", b"1.2345678E7"]


def test_rank_text_of_random_ranks_at_every_magnitude(ctx):
    edge = [0, 1, 10 ** 12 - 1, 10 ** 12, 10 ** 15 - 1]
    for k in range(15):
        edge += [10 ** k - 1, 10 ** k, 10 ** k + 1]
    rng = np.random.default_rng(4)
    rand = np.floor(10.0 ** rng.uniform(0, 15, 500_000)).astype(np.int64).tolist() + rng.integers(0, 10 ** 15, 500_000).tolist()
    values = [min(v, 10 ** 15 - 1) for v in edge + rand]
    texts = _texts(ctx, values, 15)
    for n, text in zip(values, texts):
        assert text.decode() == um.java_double(n / 1e15), n
        assert len(text) <= 25
    assert _texts(ctx, [0, 1, 10 ** 12 - 1, 10 ** 12, 120_000_000_000_000], 15) == [b"0.0", b"1.0E-15", b"9.99999999999E-4", b"0.001", b"0.12"]
    for bad, scale in (([2 ** 53], 0), ([-2 ** 53], 0), ([-1], 15), ([10 ** 15], 15), ([1], 7)):
        with pytest.raises(ur.CcoInvalidArgument):
            ctx.debug_rank_text(bad, scale)
    assert _texts(ctx, [], 0) == []


# ---- 4. k_doc_len / k_doc_write: arrays of 0, 1, 31, 32, 33, 64 and 65 elements ---------------------------------------------
LONG = "L" * 700 + '"\\\t' + "é" * 398 + "!"          # 1500 bytes of UTF-8, 1507 escaped


def _dense(rng, n_users, n_items, empty_cols=()):
    m = rng.random((n_users, n_items)) < 0.3
    m[:, list(empty_cols)] = False
    rp = np.zeros(n_users + 1, np.int64)
    np.cumsum(m.sum(1), out=rp[1:])
    return (n_users, n_items, rp, np.nonzero(m)[1].astype(np.int32))


def _column_ids(n, salt):
    kinds = ["x", "é", "☃", "\U0001f600", '"', "\\", "\t", "\x01q", "ab c", "名前"]
    return [kinds[c % len(kinds)] + (f"{salt}{c}" if c >= len(kinds) else "") for c in range(n)]


def test_indicator_arrays_around_a_warp(ctx):
    assert len(LONG.encode()) == 1500
    rng = np.random.default_rng(21)
    n_rows = 100
    mats = [_dense(rng, 400, n_rows, empty_cols=(n_rows - 1,)), _dense(rng, 400, 120)]
    rows = [f"item-{r}" for r in range(n_rows)]
    names = ["buy", "view"]
    seen = set()
    for top_k in (1, 31, 32, 33, 64, 65):
        params = [(500, top_k, None)] * 2
        res = ctx.train_csr(mats, params, 1)
        cols = [_column_ids(n_rows, "b"), _column_ids(120, "v")]
        # row 3: "", the 1500-byte id and a multi-byte id on lanes 0, 31 and 32 of the first chunks, the other way round in
        # the second indicator; row 5: the long id on the last lane of the second chunk and the empty one on lane 0 of the third
        for i, special in enumerate([{0: "", 31: LONG, 32: "☃☃"}, {0: LONG, 31: '"\\"', 32: ""}]):
            rp, ci = res[i][3], res[i][4]
            lengths = np.diff(rp)
            seen |= set(lengths.tolist())
            assert lengths[n_rows - 1] == 0 and (lengths[:n_rows - 1] == top_k).all(), (i, top_k)
            taken = {}
            for r, places in ((3, special), (5, {63: LONG, 64: ""})):
                for pos, text in places.items():
                    if pos < lengths[r]:
                        c = int(ci[rp[r] + pos])
                        assert taken.setdefault(c, text) == text
                        cols[i][c] = text
        got, want = format_both(ctx, mats, params, names, rows, cols, [], [], [])
        assert got == want, top_k
        assert got == ctx_es_bulk(ctx, mats, params, names, rows, cols)
        # the same items with properties and rankings: a field and a ranking named like an indicator drop its array
        fields = ["color", "view", "n"]
        triples = [(rows[r], fields[r % 3], '["%d"]' % r) for r in range(0, n_rows, 4)] + [("no-row", "color", "1")]
        events = ([rows[r] for r in range(0, n_rows, 3)] + ["no-row-2"], list(range(34)) + [5])
        rankings = [("popRank", "popular", 0, 50, [events]), ("buy", "popular", 0, 10, [events])]
        got, want = format_both(ctx, mats, params, names, rows, cols, fields, triples, rankings)
        assert got == want, top_k
    assert seen == set(WARP_EDGES), seen


def ctx_es_bulk(ctx, mats, params, names, rows, cols):
    _, h = ctx.train_csr(mats, params, 1, keep=True)
    try:
        return ctx.format_es_bulk(h, names, rows, cols)
    finally:
        ctx.free_result(h)


# ---- 5. the property sort: group counts next to a power of two, long runs of one (item, field) -----------------------------
@pytest.mark.parametrize("G", [255, 256, 257, 65_535, 65_536, 65_537])
def test_property_sort_keeps_the_last_triple(ctx, G):
    rows = ["a", "b", "c"]
    n_fields = 300
    fields = [f"f{f}" for f in range(n_fields)]
    fields[7], fields[290] = 'q"7', "id"
    extra = [f"x{q}" for q in range(G - len(rows))]
    item_of_group = rows + extra                       # first appearance: the rows, then the introductions below, in order
    text = lambda t: f'"{t}"'
    triples = [(x, fields[(q * 7) % n_fields], text(f"intro{q}")) for q, x in enumerate(extra)]
    marked = [item_of_group[g] for g in (0, G // 2, G - 2, G - 1)]
    last, before_last = item_of_group[G - 1], item_of_group[G - 2]
    for t in range(500):        # 500 triples compete for (last, f299) and (before_last, f256), among other items' and fields'
        triples.append((last, fields[299], text(f"last{t}")))
        triples.append((marked[t % 4], fields[(299 - t) % n_fields], text(f"m{t}")))
        triples.append((before_last, fields[256], str(t)))
        triples.append((item_of_group[(t * 37) % G], fields[299], "[%d]" % t))
    triples += [(before_last, fields[f], text(f"every{f}")) for f in reversed(range(n_fields))]     # every field, descending
    triples.append((last, fields[299], '"the last one"'))
    got, want = format_both(ctx, TINY, [(500, 50, None)], ["buy"], rows, [rows], fields, triples, [])
    assert got == want
    docs = {d["id"]: d for d in docs_of(got)}
    assert len(docs) == G and docs[last]["f299"] == "the last one"
    assert len(docs[before_last]) == n_fields and docs[before_last]["f256"] == "every256"     # 299 fields ("id" is dropped) + id


# ---- 6. old documents of 0 .. 65 members through cco_rerank_model ------------------------------------------------------------
def _old_doc(item, names_values):
    return b'{"index":{"_id":"%s"}}\n{' % item.encode() + b",".join(b'"%s":%s' % (n.encode(), v.encode()) for n, v in names_values) + b"}\n"


def _members(n):
    return [(f"m{k}", str(k)) for k in range(n)]


def test_old_documents_around_a_warp(ctx):
    body, scored = b"", []
    for n in WARP_EDGES:
        body += _old_doc(f"n{n}", _members(n))
        scored.append(f"n{n}")
    # one decoded name spelled twice, "dup" and "dup": in one chunk of 32 members, in adjacent chunks, 64 apart
    for a, b in ((3, 20), (20, 40), (0, 64), (31, 32), (64, 0)):
        ms = _members(65)
        ms[a], ms[b] = ("dup", '"plain"'), ("d\\u0075p", '"escaped"')
        body += _old_doc(f"dup{a}-{b}", ms)
        scored.append(f"dup{a}-{b}")
    # an old member named like a ranking the item has a score in: at positions 31 and 32, plain and escaped
    for pos, spelled in ((31, "popRank"), (32, "popRank"), (32, "pop\\u0052ank"), (64, "popRank")):
        ms = _members(65)
        ms[pos] = (spelled, "99.0")
        body += _old_doc(f"rank{pos}{len(spelled)}", ms)
        scored.append(f"rank{pos}{len(spelled)}")
    # the same on items the new ranking does not score: the old rank member survives
    for pos in (31, 32):
        ms = _members(65)
        ms[pos] = ("popRank", "42.0")
        body += _old_doc(f"unscored{pos}", ms)
    triples = []
    for item, _ in [(d, None) for d in scored] + [("unscored31", None), ("unscored32", None)]:
        triples.append((item, "m33", "fresh"))         # loses to the old member at position 33 where there is one
        triples.append((item, "m0", "fresh0"))
        triples.append((item, "color", "red"))
    triples.append(("brand-new", "m33", "fresh"))
    rankings = [um.Ranking("popRank", "popular", 0, 100, [(scored + ["brand-new-2"], list(range(len(scored) + 1)))]),
                um.Ranking("m64", "popular", 0, 100, [(scored[::2], [1] * len(scored[::2]))])]
    got = rerank_both(ctx, body, triples, rankings)
    docs = {d["id"]: d for d in docs_of(got)}
    assert docs["unscored31"]["popRank"] == 42.0 and docs["unscored32"]["popRank"] == 42.0
    assert docs["rank31" + "7"]["popRank"] == 1.0 and docs["n33"]["m33"] == "fresh" and docs["n64"]["m33"] == 33
    assert docs["dup0-64"]["dup"] == "escaped" and docs["dup64-0"]["dup"] == "plain" and docs["dup31-32"]["dup"] == "escaped"
    assert docs["n0"] == {"id": "n0", "m33": "fresh", "m0": "fresh0", "color": "red", "popRank": 1.0, "m64": 1.0}
    # and with no properties and no score anywhere, the body comes back member for member
    assert rerank_both(ctx, body, [], [um.Ranking("popRank", "popular", 0, 100, [(["elsewhere"], [500])])]) \
        == b"".join(_old_doc(i, [m for m in ms if m[0] != "id"]) .replace(b"\n{", b'\n{"id":"%s"%s' % (i.encode(), b"," if ms else b""), 1)
                    for i, ms in _documents(body))


def _documents(body):
    """(id, [(raw name, raw value)]) of a body built by _old_doc from unique names, the later of a repeated decoded name kept"""
    out = []
    lines = body.split(b"\n")
    for q in range(0, len(lines) - 1, 2):
        item = json.loads(lines[q])["index"]["_id"]
        inner = lines[q + 1][1:-1].decode()
        ms = [tuple(m.split(":", 1)) for m in inner.split(",")] if inner else []
        ms = [(n[1:-1], v) for n, v in ms]
        decoded = [json.loads(f'"{n}"') for n, _ in ms]
        out.append((item, [m for k, m in enumerate(ms) if decoded[k] not in decoded[k + 1:]]))
    return out

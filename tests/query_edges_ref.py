"""TEST INFRASTRUCTURE: references and input generators of the query-builder edge tests (test_query_edges.py on the CPU,
test_gpu_query_edges.py on the device).

json4s_quote_ref and history_ref restate, independently of ur_query, the two rules the device kernels implement on their
own: the json4s 3.2 quote (uq_escape on the device, uq_quote on the host) and one user's history lists and blacklist
(k_uq_hist_keys, k_uq_first, k_mq_record).  The generators write the directed index bodies and event exports; each returns
the body or export with the structure the queries must carry, which does not depend on the escaping."""
from __future__ import annotations

import json
import random

# ---- the json4s 3.2 quote, one table entry per code point below U+2100; every code point from U+2100 up passes through --
_SHORT = {0x22: '\\"', 0x5C: "\\\\", 0x08: "\\b", 0x0C: "\\f", 0x0A: "\\n", 0x0D: "\\r", 0x09: "\\t"}


def _entry(c: int) -> str:
    if c in _SHORT:
        return _SHORT[c]
    if c <= 0x1F or 0x80 <= c <= 0x9F or 0x2000 <= c <= 0x20FF:
        return "\\u" + format(c, "04x")
    return chr(c)


QUOTE_TABLE = [_entry(c) for c in range(0x2100)]


def json4s_quote_ref(s: str) -> str:
    """json4s 3.2's quote of s, quotes included"""
    return '"' + "".join(QUOTE_TABLE[ord(ch)] if ord(ch) < 0x2100 else ch for ch in s) + '"'


# ---- one user's history -------------------------------------------------------------------------------------------------
def history_ref(events, names, limits, blacklist, blacklist_items):
    """events: one user's training events [(event name, item, time ms, line)]; names / limits: the query event names and
    their per-name limits; blacklist: the blacklisted event names; blacklist_items: the query's list.
    -> ([the history list of each query name], blacklist): a name's list is its `limit` latest events (time descending, a
    later line first among equal times), oldest first, each item once at its oldest position; the blacklist is the items of
    every event of a name that is both a query name and blacklisted, newest first, then blacklist_items, each item once."""
    newest_first = sorted(events, key=lambda e: (e[2], e[3]), reverse=True)
    lists = []
    for name, limit in zip(names, limits):
        window = [item for ev, item, _, _ in newest_first if ev == name][:limit]
        window.reverse()
        out, seen = [], set()
        for item in window:
            if item not in seen:
                seen.add(item)
                out.append(item)
        lists.append(out)
    flagged = set(blacklist) & set(names)
    black, seen = [], set()
    for item in [item for ev, item, _, _ in newest_first if ev in flagged] + list(blacklist_items):
        if item not in seen:
            seen.add(item)
            black.append(item)
    return lists, black


# ---- what a record carries, read back with json.loads -------------------------------------------------------------------
def records(body: bytes, offsets):
    """the queries of an _msearch body, parsed: one (header, query) per record"""
    out = []
    for r in range(len(offsets) - 1):
        head, query, tail = body[offsets[r]:offsets[r + 1]].decode("utf-8", "surrogatepass").split("\n")
        assert tail == ""
        out.append((json.loads(head), json.loads(query)))
    return out


def clause_lists(query: dict, in_must: bool = False):
    """the [(name, values)] of the terms clauses in should (must when in_must), and the must_not ids"""
    b = query["query"]["bool"]
    terms = [c["terms"] for c in b["must" if in_must else "should"] if "terms" in c]
    pairs = [next((k, v) for k, v in t.items() if k != "boost") for t in terms]
    return pairs, b["must_not"][0]["ids"]["values"]


def expected_similar(names, members, slice_: int):
    """the similar-items clauses of a document's members (None: no source members)"""
    if members is None:
        return []
    out = []
    for n in names:
        v = members.get(n, [])
        out.append((n, v if len(v) <= slice_ else v[:slice_ - 1]))
    return out


# ---- JSON text of a string, two ways ------------------------------------------------------------------------------------
def jraw(s: str) -> str:
    """a JSON string literal with the bytes as they are, escaping only what JSON requires (and lone surrogates, which have no
    UTF-8 form)"""
    out = ['"']
    for ch in s:
        c = ord(ch)
        if ch == '"' or ch == "\\":
            out.append("\\" + ch)
        elif c < 0x20 or 0xD800 <= c <= 0xDFFF:
            out.append("\\u%04x" % c)
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)


def jesc(s: str) -> str:
    """a JSON string literal with every UTF-16 unit written as \\uXXXX"""
    out = ['"']
    for ch in s:
        c = ord(ch)
        if c > 0xFFFF:
            c -= 0x10000
            out.append("\\u%04x\\u%04X" % (0xD800 + (c >> 10), 0xDC00 + (c & 0x3FF)))
        else:
            out.append("\\u%04x" % c)
    out.append('"')
    return "".join(out)


def jlit(s: str, k: int) -> str:
    return jesc(s) if k % 2 else jraw(s)


# ---- every code point ---------------------------------------------------------------------------------------------------
def codepoint_strings(seed: int = 11) -> list:
    """U+0001..U+10FFFF in order, lone surrogates included, cut into strings of varied length (1 to about 1 500 code
    points).  A high surrogate is never followed by a low one inside a string: the pair would decode as one code point."""
    rng = random.Random(seed)
    out, c = [], 1
    while c <= 0x10FFFF:
        n = rng.choice([1, 2, 3, 5, 8, 31, 32, 33]) if rng.random() < 0.3 else rng.randrange(40, 1500)
        end = min(c + n, 0x110000)
        if c < 0xDC00 < end:
            end = 0xDC00
        out.append("".join(map(chr, range(c, end))))
        c = end
    return out


# each escape class at the last byte (and next to the last) of a string
EDGE_STRINGS = ["e\u0085", "e\u0080", "e\u009f", "e\u2000", "e\u20ff", "e\u2100", "e\u1fff", "e\u00a0", "e\u007f", "e\u00c2",
                "e\u2028\u0085", "\u0085", "\u20ff", "\u2100", "\u00a0", "\u007f", "e\u00e2\u0083", "e\\", 'e"', "e\t"]


def names64() -> list:
    """U+0001..U+10FFFF cut into 64 names: two short ones first (the control codes and C1), then 62 long ones"""
    cps = list(range(1, 0x110000))
    short = [cps[:0x7f], cps[0x7f:0xa0]]   # U+0001..U+007F, U+0080..U+00A0
    rest = cps[0xa0:]
    cut = [0xDC00 - 0xa1]                  # U+DBFF ends one name
    step = len(rest) // 62
    bounds = sorted(set([k * step for k in range(1, 62)] + cut))
    while len(bounds) > 61:
        bounds.remove(min(b for b in bounds if b not in cut))
    pieces, a = [], 0
    for b in bounds + [len(rest)]:
        pieces.append(rest[a:b])
        a = b
    names = ["".join(map(chr, p)) for p in short + pieces]
    assert len(names) == 64 and "".join(names) == "".join(map(chr, cps))
    return names


def index_body(docs, id_modes=None) -> bytes:
    """docs: [(id, source text)] -> a bulk body; the action's _id written raw or with \\u escapes, alternating"""
    lines = []
    for k, (i, src) in enumerate(docs):
        mode = k if id_modes is None else id_modes[k]
        lines.append('{"index":{"_index":"urindex","_id":' + jlit(i, mode) + "}}")
        lines.append(src)
    return ("\n".join(lines) + "\n").encode("utf-8")


def source(members, mode: int = 0) -> str:
    """[(name, [elements])] -> a source object, elements raw and \\u-escaped alternately (mode shifts the alternation)"""
    return "{" + ",".join(jlit(n, mode) + ":[" + ",".join(jlit(x, mode + j) for j, x in enumerate(v)) + "]" for n, v in members) + "}"


def codepoint_index(model_names, seed: int = 11):
    """every code point as array elements and as _ids: document k has _id strings[k] and, under each model name, the next
    1-3 strings -> (body, ids, {id: {name: elements}})"""
    strings = codepoint_strings(seed) + EDGE_STRINGS
    rng = random.Random(seed)
    docs, expect = [], {}
    n = len(strings)
    for k, s in enumerate(strings):
        members = [(nm, [strings[(k + 1 + j + t) % n] for j in range(rng.randrange(4))]) for t, nm in enumerate(model_names)]
        docs.append((s, source(members, k)))
        expect[s] = dict(members)
    return index_body(docs), strings, expect


def event_line(user, event, item, t_ms, mode: int = 0) -> str:
    from universal_recommender_b200.ur_query import iso_utc
    return ('{"event":' + jlit(event, mode) + ',"entityType":"user","entityId":' + jlit(user, mode + 1) +
            ',"targetEntityType":"item","targetEntityId":' + jlit(item, mode) + ',"eventTime":"' + iso_utc(t_ms) + '"}')


def export(lines) -> bytes:
    return ("\n".join(lines) + "\n").encode("utf-8")


def codepoint_export(names, seed: int = 11) -> bytes:
    """every code-point string as an item of users u0..u6, under the two short names of names64() (the first is the
    default blacklisted name) and a name outside the query"""
    strings = codepoint_strings(seed) + EDGE_STRINGS
    rng = random.Random(seed)
    base = 1_600_000_000_000
    lines = [event_line("u%d" % (k % 7), [names[0], names[1], "other"][k % 3], s, base + rng.randrange(50) * 1000, k)
             for k, s in enumerate(strings)]
    return export(lines)


# ---- k_iq_array: backslash runs, whitespace runs, brackets and commas inside strings ------------------------------------
def run_cases():
    """(offset, run, closer): runs of 0-66 escaped backslashes, with or without an escaped quote, at every offset 0-31 from
    the value's first byte"""
    return [(k, n, c) for n in range(67) for k in range(32) for c in ("", '\\"')]


WS = " \t\r"


def ws(n: int, k: int = 0) -> str:
    return "".join(WS[(k + j) % 3] for j in range(n))


def array_sweep_index():
    """-> (body, ids, {id: {name: elements}}): "purchase" holds a backslash run at every offset, "view" whitespace runs around
    every token, "like" brackets and commas inside strings"""
    docs, expect = [], {}
    tricky = ["]", ",", "[", '"]', '",', "a]b", "x,y", "\\", "\\]", "]\\", '\\",', "", " ", "[]", '["x"]', "}", "{"]
    for j, (k, n, c) in enumerate(run_cases()):
        elem_text = "a" + "\\\\" * n + c + "z%d" % j          # JSON text of the element
        elem = json.loads('"' + elem_text + '"')
        nxt = "t" + "\\\\" * (j % 5) + "%d" % j
        purchase = '["' + "p" * k + elem_text + '","' + nxt + '"]'   # the run starts k + 3 bytes into the value
        elem = "p" * k + elem
        w = [j % 41, (j * 7 + 3) % 41, (j * 13 + 5) % 41, (j * 17 + 11) % 41]
        view_elems = ["v%d" % j, tricky[j % len(tricky)], "w"]
        view = (ws(w[0], j) + "[" + ws(w[1], 1) + (ws(w[2], 2) + "," + ws(w[3], 0)).join(jlit(x, j + t) for t, x in enumerate(view_elems))
                + ws(w[2], 1) + "]" + ws(w[0], 2))
        like_elems = [tricky[(j + t) % len(tricky)] for t in range(j % 4)]
        like = "[" + ",".join(jraw(x) for x in like_elems) + "]"
        i = "doc%d" % j
        docs.append((i, '{"purchase":' + purchase + ',"view":' + view + ',' + ws(j % 7) + '"like":' + like + "}"))
        expect[i] = {"purchase": [elem, json.loads('"' + nxt + '"')], "view": view_elems, "like": like_elems}
    return index_body(docs), [i for i, _ in docs], expect


# a malformed "view" value: (text, valid JSON); each is refused by the device, the valid JSON ones by the mirror too
MALFORMED = [('["x",]', False), ('[,"x"]', False), ('["x",,"y"]', False), ('["x" "y"]', False), ('["x"]x', False),
             ('["x"}', False), ('["x",1]', True), ('[1]', True), ('["x",["y"]]', True), ('["x",{}]', True),
             ('{"a":["x"]}', True), ('"x"', True), ('null', True), ('[null]', True)]


def malformed_index(form: str, at: int, pad: int, n_docs: int = 40) -> bytes:
    """n_docs good documents, document `at`'s "view" member replaced by form, shifted by pad spaces inside the array (or
    before the value when form does not start with '[')"""
    docs = []
    for d in range(n_docs):
        if d == at:
            v = "[" + " " * pad + form[1:] if form.startswith("[") else " " * pad + form
        else:
            v = "[" + " " * pad + '"v%d","w"]' % d
        docs.append(("m%d" % d, '{"purchase":["p%d"],"view":%s}' % (d, v)))
    return index_body(docs)


# ---- list and slice boundaries ------------------------------------------------------------------------------------------
SIZES = [0, 1, 31, 32, 33, 63, 64, 65, 1000]


def list_element(j: int) -> str:
    odd = ["", "\u0085", "\u2000", '"', "\\", "\n", "\U0001f600", "\u00e9", "\ud800"]
    return "e%d" % j + odd[j % len(odd)] * (j % 3)


def list_index():
    """documents whose "purchase" and "view" arrays have SIZES elements, one whose model name is repeated (the last wins, one
    of them written with escapes), a source {} and a source without a model name -> (body, ids, expect, repeated-name id)"""
    docs, expect = [], {}
    for k, n in enumerate(SIZES):
        p = [list_element(j) for j in range(n)]
        v = [list_element(j + 7) for j in range(SIZES[-1 - k])]
        i = "s%d" % n
        docs.append((i, source([("purchase", p), ("view", v)], k)))
        expect[i] = {"purchase": p, "view": v}
    docs.append(("rep", '{"view":["a"],"purchase":["first"],"p\\u0075rchase":["second","x"],"view":' + "[" + ",".join(
        jraw(list_element(j)) for j in range(33)) + "]}"))
    expect["rep"] = {"purchase": ["second", "x"], "view": [list_element(j) for j in range(33)]}
    docs.append(("rep2", '{"\\u0070urchase":["first"],"purchase":["last"]}'))
    expect["rep2"] = {"purchase": ["last"], "view": []}
    docs.append(("empty", "{}"))
    expect["empty"] = None
    docs.append(("nomodel", '{"popRank":1.5,"category":["x"]}'))
    expect["nomodel"] = {"purchase": [], "view": []}
    return index_body(docs), [i for i, _ in docs], expect


# ---- history limits and ties --------------------------------------------------------------------------------------------
LIMITS = [1, 31, 32, 33, 64, 500]


def history_export(seed: int = 5):
    """users with limit - 1, limit and limit + 1 events of one name (limit in LIMITS), items repeated inside the window and
    just outside it, equal eventTimes within a name and across names (ties on the limit boundary), users with events of a
    name outside the query only; lines shuffled.  -> (export, engine json, users)"""
    rng = random.Random(seed)
    names = ["n%d" % L for L in LIMITS]
    base = 1_600_000_000_000
    ev = []
    users = []
    for L, name in zip(LIMITS, names):
        for size in (L - 1, L, L + 1):
            u = "u-%d-%d" % (L, size)
            users.append(u)
            pool = ["i%d" % j for j in range(max(2, L // 3))]
            for r in range(size):   # r = 0 is the newest
                t = base - r * 1000
                if L - 2 <= r <= L + 1:
                    t = base - (L - 2) * 1000   # ties across the limit
                item = rng.choice(pool)
                if r == L:
                    item = "out-%s" % u if size % 2 else pool[0]   # just outside: new, or also inside
                ev.append((u, name, item, t))
            for r in range(rng.randrange(1, 6)):   # other query names at the same times
                ev.append((u, rng.choice([x for x in names if x != name]), rng.choice(pool), base - rng.randrange(L + 2) * 1000))
    for k in range(4):
        u = "only-other-%d" % k
        users.append(u)
        for r in range(3):
            ev.append((u, "other", "i%d" % r, base))
    rng.shuffle(ev)
    lines = [event_line(u, n, i, t, k) for k, (u, n, i, t) in enumerate(ev)]
    engine = {"indicators": [{"name": n, "maxItemsPerUser": L} for n, L in zip(names, LIMITS)], "blacklistEvents": ["n31", "n1", "other"]}
    return export(lines), engine, names, users


def names64_export(seed: int = 6):
    """63 query names, q5 given twice (64 in all) and blacklisted once; users with events of all of them, ties across
    names -> (export, engine json, query names, users)"""
    rng = random.Random(seed)
    names = ["q%d" % k for k in range(63)]
    limits = [LIMITS[k % len(LIMITS)] for k in range(63)]
    base = 1_600_000_000_000
    ev, users = [], []
    for k in range(40):
        u = "w%d" % k
        users.append(u)
        for _ in range(rng.randrange(10, 200)):
            ev.append((u, rng.choice(names), "i%d" % rng.randrange(40), base - rng.randrange(30) * 1000))
    rng.shuffle(ev)
    lines = [event_line(u, n, i, t, k) for k, (u, n, i, t) in enumerate(ev)]
    engine = {"indicators": [{"name": n, "maxItemsPerUser": L} for n, L in zip(names, limits)], "blacklistEvents": ["q5", "q9"]}
    return export(lines), engine, names + ["q5"], users


# ---- many records per warp ----------------------------------------------------------------------------------------------
def many_index(n_docs: int, seed: int = 9):
    """n_docs documents with three model names -> (body, ids)"""
    rng = random.Random(seed)
    docs = []
    ids = ["d%d%s" % (k, "\u0085" if k % 5 == 0 else "") for k in range(n_docs)]
    for k, i in enumerate(ids):
        m = [(nm, [ids[rng.randrange(n_docs)] for _ in range(rng.randrange(6))]) for nm in ("purchase", "view", "like")]
        docs.append((i, source(m[:rng.randrange(4)], k)))
    return index_body(docs), ids


def many_export(n_users: int, n_events: int, seed: int = 10) -> bytes:
    """n_events events of n_users users, each user's first one a "view"; names outside the query among the rest"""
    rng = random.Random(seed)
    base = 1_600_000_000_000
    lines = []
    for k in range(n_events):
        u = k if k < n_users else rng.randrange(n_users)
        lines.append('{"event":"%s","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d\\u2028",'
                     '"eventTime":"%s"}' % ("view" if k < n_users else rng.choice(("buy", "view", "like", "other")), u, rng.randrange(5000),
                                            _iso(base + rng.randrange(100) * 1000)))
    return export(lines)


def _iso(ms: int) -> str:
    from universal_recommender_b200.ur_query import iso_utc
    return iso_utc(ms)

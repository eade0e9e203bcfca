"""The directed number texts of number_edges checked against exact arithmetic (fractions.Fraction), so the GPU tests can
trust them as a reference: every path label follows the routing rule, float() rounds every text correctly (ties to
even, overflow at the midpoint past DBL_MAX, underflow to a signed zero), java_double prints the shortest digits that
round back and the nearest of those, in Java's layout.  Then the ur_predict mirror's number contract: the reference
double for every text, and a ValueError for every text out of the range of a double, whatever its length; and the
mirror's reading of the integer fields (status, hits.total, _shards.failed) of both readers."""
import math
import re
from decimal import Decimal
from fractions import Fraction

import pytest

import number_edges as E
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200 import ur_predict as P
from universal_recommender_b200.ur_model import java_double

SETS = E.sets()
TOP = Fraction(2) ** 1024   # the virtual neighbour above DBL_MAX


def test_set_sizes():
    assert {k: len(v) for k, v in SETS.items()} == {"routing": 370, "powers_of_two": 25284, "ties": 4556, "zeros": 17,
                                                     "layout": 186, "saturation": 118, "integers": 54, "float32": 1654}


@pytest.mark.parametrize("name", list(SETS))
def test_labels_follow_the_routing_rule(name):
    for t, p in SETS[name]:
        assert E.route(t) == p, t[:80]


def check_rounding(text: str):
    """float(text) is the double nearest to the exact value, ties to the even one; infinity from the midpoint past
    DBL_MAX up; a zero keeps the text's sign unless the text is an integer"""
    v = E.value(text)
    q, side = E.exact_fraction(text)
    neg = text.startswith("-")
    if q is None:
        assert (v is None) if side > 0 else (v == 0 and math.copysign(1, v) == (-1 if neg else 1)), text[:80]
        return
    a = abs(q)
    if a >= E.OVERFLOW:
        assert v is None, text[:80]
        return
    assert v is not None and (v == 0 or (v < 0) == neg), text[:80]
    if v == 0:
        assert math.copysign(1, v) == (-1 if neg and not E.parts(text)[4] else 1), text[:80]
    x = abs(v)
    d = abs(a - Fraction(x))
    for n in ([Fraction(E.nextdown(x))] if x > 0 else []) + [Fraction(E.nextup(x)) if E.nextup(x) != math.inf else TOP]:
        dn = abs(a - n)
        assert d < dn or (d == dn and E.bits(x) % 2 == 0), (text[:80], x)


def decade(q: Fraction) -> int:
    """floor(log10(q)) of q > 0"""
    e = math.floor(math.log10(float(q))) if float(q) > 0 else -324
    while Fraction(10) ** e > q:
        e -= 1
    while Fraction(10) ** (e + 1) <= q:
        e += 1
    return e


PLAIN = re.compile(r"-?(0|[1-9][0-9]*)\.(0|[0-9]*[1-9])\Z")
SCI = re.compile(r"-?[1-9]\.(0|[0-9]*[1-9])E-?[1-9][0-9]{0,2}\Z")


def check_java(v: float):
    """java_double(v): the shortest digits that round back to v, the nearest to v of those, in Java's layout"""
    j = java_double(v)
    assert float(j) == v and (v != 0 or j == ("-0.0" if math.copysign(1, v) < 0 else "0.0")), (v, j)
    if v == 0:
        return
    x, J = abs(v), abs(Fraction(Decimal(j)))
    plain = Fraction(1, 1000) <= Fraction(x) < 10 ** 7
    assert (PLAIN if plain else SCI).match(j), (v, j)
    n = len(j.lstrip("-").partition("E")[0].replace(".", "").strip("0"))
    F = Fraction(x)
    e = decade(F)

    def near(p):   # the p-digit decimals on either side of v
        g = Fraction(10) ** (e - p + 1)
        return [math.floor(F / g) * g, math.ceil(F / g) * g]
    def back(c):   # c reads back as x (float() of a Fraction rounds correctly, but raises where it would overflow)
        return 0 < c < E.OVERFLOW and float(c) == x
    if n > 1:
        assert not any(back(c) for c in near(n - 1)), (v, j)
    ok = [c for c in near(n) if back(c)]
    assert J in ok and all(abs(J - F) <= abs(c - F) for c in ok), (v, j)


@pytest.mark.parametrize("name", list(SETS))
def test_float_rounds_every_text_correctly(name):
    for t, _ in SETS[name]:
        check_rounding(t)


@pytest.mark.parametrize("name", list(SETS))
def test_java_double_is_shortest_nearest_in_java_layout(name):
    for v in {E.bits(v): v for v in (E.value(t) for t, _ in SETS[name]) if v is not None}.values():
        check_java(v)


def test_references_cover_both_paths_and_every_outcome():
    allt = [x for v in SETS.values() for x in v]
    vals = [E.value(t) for t, _ in allt]
    assert sum(v is None for v in vals) == 60
    assert {p for _, p in allt} == {E.FAST, E.EXACT}
    assert any(v == 0 and math.copysign(1, v) < 0 for v in vals) and any(v == 0 and math.copysign(1, v) > 0 for v in vals)
    assert 5e-324 in vals and -1.7976931348623157e308 in vals


def test_the_two_defect_texts():
    z = "0" * 100000
    assert (E.route("1" + z + "e-200000"), E.value("1" + z + "e-200000")) == (E.EXACT, 0.0)
    assert (E.route("0." + z + "1e200000"), E.value("0." + z + "1e200000")) == (E.EXACT, None)
    assert E.value("-0") == 0.0 and math.copysign(1, E.value("-0")) == 1 and math.copysign(1, E.value("-0.0")) == -1


def test_java_digits_at_powers_of_two():
    """2^-24: the nearest 16-digit decimal lies outside the narrow lower half-gap, another 16-digit one inside the upper"""
    assert java_double(2.0 ** -24) == "5.960464477539063E-8"
    assert java_double(2.0 ** -44) == "5.684341886080802E-14"
    assert java_double(2.0 ** 89) == "6.189700196426902E26"


def test_fuzz_references():
    """a sample of the GPU fuzz texts: in range, and their references as exact as the directed ones"""
    texts = E.fuzz(3000, seed=2)
    assert len(texts) == 3000 and all(E.value(t) is not None for t in texts)
    for t in texts:
        check_rounding(t)
        check_java(E.value(t))


# ---- the mirror -----------------------------------------------------------------------------------------------------------
OUT_OF_RANGE = sorted({t for v in SETS.values() for t, _ in v if E.value(t) is None}
                      | {s + "1" * n for n in (310, 400, 4300, 4301, 10000, 100000) for s in ("", "-")}, key=len)


def test_mirror_number_value_is_the_reference():
    for v in SETS.values():
        for t, _ in v:
            want = E.value(t)
            if want is not None:
                got = P.number_value(t)
                assert E.bits(got) == E.bits(want), t[:80]
                assert P.number_text(t) == java_double(want)


@pytest.mark.parametrize("text", OUT_OF_RANGE, ids=lambda t: f"{t[:12]}..{len(t)}")
def test_mirror_out_of_range_is_a_value_error(text):
    with pytest.raises(ValueError, match="is out of the range of a double"):
        P.number_value(text)
    body = '{"responses":[{"hits":{"hits":[{"_id":"a","_score":%s}]}}]}' % text
    with pytest.raises(ValueError, match="out of the range"):
        P.predictions(body, [], False)
    body = '{"responses":[{"hits":{"hits":[{"_id":"a","_score":1,"_source":{"r":%s}}]}}]}' % text
    with pytest.raises(ValueError, match="out of the range"):
        P.predictions(body, ["r"], True)


def test_mirror_status():
    got = {}
    for s in E.STATUS:
        try:
            p = P.predictions('{"responses":[%s]}' % E.status_element(s), [], False)[0]
            got[s] = (p.status, len(p.items))
        except ValueError:
            got[s] = "error"
    assert got == {"2147483647": (2147483647, 0), "2147483648": "error", "-2147483648": (-2 ** 31, 0), "-2147483649": "error",
                   "200": (200, 1), "200.0": "error", "2e2": "error", "-0": (0, 0), "0200": "error"}


def test_mirror_totals():
    got = {}
    for t in E.TOTAL:
        try:
            got[t] = [P.predictions('{"responses":[%s]}' % x, [], False)[0].total for x in E.total_elements(t)]
        except ValueError:
            got[t] = "error"
    assert got == {str(2 ** 63 - 1): [2 ** 63 - 1] * 2, str(-(2 ** 63 - 1)): [-(2 ** 63 - 1)] * 2, str(2 ** 63): [-1, -1],
                   str(-2 ** 63): [-1, -1], "-0": [0, 0], "1.0": [-1, -1], "1e3": [-1, -1], "0": [0, 0], "00": "error"}


def test_mirror_index_page_integers():
    got = {}
    for f in E.SHARDS_FAILED:
        try:
            got[f] = um.index_page(E.shards_page(f))[1]
        except ValueError as e:
            got[f] = str(e).split(": ")[-1]
    assert got == {"0": 1, "-0": 1, "0.0": "_shards.failed is not 0", "1": "_shards.failed is not 0",
                   "-1": "_shards.failed is not 0", "00": "malformed JSON"}
    tot = {}
    for t in E.TOTAL:
        try:
            tot[t] = [um.index_page(x.encode())[3] for x in E.total_elements(t)]
        except ValueError as e:
            tot[t] = str(e).split(": ")[-1]
    assert tot == {str(2 ** 63 - 1): [2 ** 63 - 1] * 2, str(-(2 ** 63 - 1)): [-(2 ** 63 - 1)] * 2, str(2 ** 63): [-1, -1],
                   str(-2 ** 63): [-1, -1], "-0": [0, 0], "1.0": [-1, -1], "1e3": [-1, -1], "0": [0, 0], "00": "malformed JSON"}

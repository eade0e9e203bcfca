"""Directed JSON number texts for the _msearch reader's number path (cco_results.cuh sr_number, cco_api.cu sr_exact_value,
sr_java_text) and their exact reference.

The reader takes a number one of two ways: the device's fast path (Clinger: at most 15 significant digits, none lost past
the 19th, |e10| <= 22, one exact multiply or divide) or the host's exact path (strtod, and the shortest round-trip
digits).  Every directed text is labelled with the path it must take; route() restates the rule, including the
exponent literal's saturation, and the tests check the labels against it and the device's n_exact against both.

The reference of a text is its double from float() (None when it is out of the range of a double), with an integer
literal's -0 read as 0.0 (a JInt), and its Java text from ur_model.java_double."""
import math
import random
import struct
from decimal import Decimal
from fractions import Fraction

import numpy as np

from universal_recommender_b200.ur_model import java_double

FAST, EXACT = "fast", "exact"
SATURATE = 1 << 59   # the exponent literal saturates here (sr_number)
MAX = Fraction(2 ** 1024 - 2 ** 971)
OVERFLOW = Fraction(2 ** 1024 - 2 ** 970)   # the midpoint between DBL_MAX and 2^1024: this and above round to infinity


def parts(text: str):
    """a JSON number's text -> (negative, integer digits, fraction digits, exponent literal as an int, is an integer)"""
    neg = text.startswith("-")
    t = text[neg:]
    mant, e, exp = t.replace("E", "e").partition("e")
    ip, dot, fp = mant.partition(".")
    return neg, ip, fp, int(exp) if e else 0, not (dot or e)


def route(text: str) -> str:
    """the path sr_number sends a text down: the significant digits stripped of zeros, at most 15 of them (a lost
    non-zero digit past the 19th makes more than 15), and the power of ten they carry within +-22"""
    _, ip, fp, x, _ = parts(text)
    s = (ip + fp).lstrip("0")
    if not s:
        return FAST   # every zero is the fast path's
    t = s.rstrip("0")
    if abs(x) >= SATURATE:
        return EXACT
    e10 = x - len(fp) + len(s) - len(t)
    return FAST if len(t) <= 15 and -22 <= e10 <= 22 else EXACT


def value(text: str):
    """the double of a text, None out of range; an integer literal -0 is 0.0"""
    v = float(text)
    if math.isinf(v):
        return None
    return 0.0 if v == 0 and parts(text)[4] else v


def java(text: str):
    v = value(text)
    return None if v is None else java_double(v)


# ---- exact decimals ------------------------------------------------------------------------------------------------------
def decimal(q: Fraction) -> str:
    """the exact decimal text of a Fraction whose denominator divides a power of ten"""
    neg, q = q < 0, abs(q)
    d, a, b = q.denominator, 0, 0
    while d % 2 == 0:
        d, a = d // 2, a + 1
    while d % 5 == 0:
        d, b = d // 5, b + 1
    if d != 1:
        raise ValueError("not a terminating decimal")
    k = max(a, b)
    n = str((q * 10 ** k).numerator).rjust(k + 1, "0")
    s = n[:len(n) - k] + ("." + n[len(n) - k:] if k else "")
    return ("-" if neg else "") + s


def exact_fraction(text: str):
    """the exact value of a text as a Fraction; None when it lies beyond 10^+-400 (certainly out of range, or certainly
    rounding to zero), with the side as the second item"""
    _, ip, fp, x, _ = parts(text)
    s = (ip + fp).lstrip("0")
    if not s:
        return Fraction(0), 0
    lead = x - len(fp) + len(s)   # the value lies in [10^(lead - 1), 10^lead)
    if lead > 400:
        return None, 1
    if lead < -400:
        return None, -1
    return Fraction(Decimal(text)), 0   # Decimal: no limit on the digits of a string


def nextup(x: float) -> float:
    return math.nextafter(x, math.inf)


def nextdown(x: float) -> float:
    return math.nextafter(x, -math.inf)


def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# ---- directed sets ---------------------------------------------------------------------------------------------------------
def _both_signs(texts):
    return [t for x in texts for t in (x, "-" + x)]


def routing():
    out = []
    for t, p in [("123456789012345", FAST), ("1234567890123456", EXACT), ("123456789012345000000", FAST),
                 ("1234567890123456000000", EXACT), ("1.234567890123450000", FAST), ("1.2345678901234560000", EXACT),
                 ("12345678901234.5", FAST), ("1234567890123.456", EXACT), ("0.000123456789012345", FAST),
                 ("0.0000000123456789012345", FAST), ("0.00000000123456789012345", EXACT), ("999999999999999", FAST),
                 ("9999999999999999", EXACT),
                 ("123456789012345e22", FAST), ("123456789012345e23", EXACT), ("123456789012345e-22", FAST),
                 ("123456789012345e-23", EXACT), ("1.23456789012345e-8", FAST), ("1.23456789012345e-9", EXACT),
                 ("1234567890123456789", EXACT), ("12345678901234567890", EXACT), ("1000000000000000000", FAST),
                 ("10000000000000000000", FAST), ("1" + "0" * 22, FAST), ("1" + "0" * 23, EXACT),
                 ("1" + "0" * 18 + "1", EXACT), ("1" + "0" * 19 + "1", EXACT), ("1" + "0" * 30 + "1", EXACT),
                 ("1." + "0" * 18 + "1", EXACT), ("1." + "0" * 30, FAST), ("0.1" + "0" * 30, FAST),
                 ("1." + "0" * 30 + "1", EXACT), ("1" + "0" * 21 + ".000000", FAST), ("12" + "0" * 40 + "e-40", FAST),
                 ("12" + "0" * 40 + "e-62", FAST), ("12" + "0" * 40 + "e-63", EXACT), ("1" + "0" * 25 + "e-3", FAST),
                 ("1" + "0" * 25 + "e-2", EXACT), ("0.5e0", FAST), ("5E-1", FAST), ("1E+22", FAST), ("1E+23", EXACT)]:
        out.append((t, p))
    for e in range(-25, 26):
        p = FAST if abs(e) <= 22 else EXACT
        out += [(f"1e{e}", p), (f"123456789012345e{e}", p), (f"-9.87654321098765e{e + 14}", p), (f"7E{e:+d}", p)]
    for e in range(0, 26):
        out.append(("1" + "0" * e, FAST if e <= 22 else EXACT))
        out.append(("0." + "0" * e + "1", FAST if e + 1 <= 22 else EXACT))
        out.append(("0." + "0" * e + "123456789012345", FAST if e + 15 <= 22 else EXACT))
    for k in [21, 22, 23, 30, 100, 250, 322, 323, 324, 325, 330, 400]:   # leading fraction zeros
        out.append(("0." + "0" * k + "1", FAST if k + 1 <= 22 else EXACT))
        out.append(("0." + "0" * k + "5e" + str(k + 1), FAST))   # the offset cancels: 0.5
        out.append(("0." + "0" * k + "25e" + str(k + 20), FAST))
        out.append(("0." + "0" * k + "25e" + str(k + 25), EXACT))
        out.append(("-0." + "0" * k + "4940656458412465441765687928682213723651", EXACT))
    return out


def _pow2_values():
    vals = []
    for k in range(-1074, 1024):
        a = math.ldexp(1.0, k)
        vals += [x for x in (nextdown(a), a, nextup(a)) if x != 0 and not math.isinf(x)]
    return sorted(set(vals))


SAMPLE_K = sorted(set(range(-1074, 1024, 41)) | {-1074, -1073, -1022, -1017, -44, -24, 0, 52, 53, 89, 122, 1023})


def powers_of_two():
    out = []
    for x in _pow2_values():
        out += _both_signs([repr(x), "%.17e" % x])
    for k in SAMPLE_K:
        out += _both_signs([decimal(Fraction(2) ** k)])
    return [(t, route(t)) for t in out]


def _midpoints(x: float):
    """the exact midpoint between x and its upper neighbour, and that +- one unit 20 places past its last digit"""
    m = (Fraction(x) + Fraction(nextup(x))) / 2
    k = len(decimal(m).partition(".")[2])
    u = Fraction(1, 10 ** (k + 20))
    return [decimal(m), decimal(m + u), decimal(m - u)]


def ties():
    rng = random.Random(11)
    xs = [math.ldexp(1.0, k) for k in range(-1074, 1024, 7)]
    xs += [nextdown(math.ldexp(1.0, k)) for k in range(-1073, 1024, 7)]
    xs += [struct.unpack("<d", struct.pack("<Q", rng.getrandbits(63)))[0] for _ in range(150)]
    xs += [5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308, 1.0, 0.1, 9007199254740992.0, nextdown(float(MAX))]
    out = []
    for x in xs:
        if x == 0 or math.isinf(x) or math.isinf(nextup(x)):
            continue
        out += _midpoints(x)
    top = decimal(OVERFLOW)   # the overflow threshold itself: ties to even, to infinity
    out += [top, top + "." + "0" * 30 + "1", decimal(OVERFLOW - Fraction(1, 10 ** 30))]
    out += ["9007199254740993", "9007199254740993.000000000000000000000000001", "9007199254740992.999999999999999999999999",
            "2.2250738585072011e-308", "2.2250738585072012e-308", "2.4703282292062327e-324", "2.4703282292062328e-324",
            "4.9406564584124654e-324", "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308",
            "0.1000000000000000055511151231257827021181583404541015625", "0.1000000000000000055511151231257827021181583404541015624",
            "0.1000000000000000055511151231257827021181583404541015626"]
    return [(t, route(t)) for t in _both_signs(out)]


def zeros():
    return [("0", FAST), ("-0", FAST), ("0.0", FAST), ("-0.0", FAST), ("0e999999999", FAST), ("-0E-999999999", FAST),
            ("0.000", FAST), ("-0.000e+5", FAST), ("0e0", FAST), ("0." + "0" * 400, FAST), ("-0." + "0" * 400 + "e400", FAST),
            ("1e-400", EXACT), ("-1e-400", EXACT), ("2.4703282292062327e-324", EXACT), ("-2.4703282292062327e-324", EXACT),
            ("0." + "0" * 400 + "1", EXACT), ("-0." + "0" * 330 + "1", EXACT)]


def layout():
    vals = [1e-3, nextdown(1e-3), nextup(1e-3), 1e7, nextdown(1e7), nextup(1e7), 9999999.999999998, 0.001,
            0.00999, 0.0123, 1234567.0, 12345678.0, 1.5e10, 1.5e100, 1.5e-5, 1.5e-10, 1.5e-100, 1e8, 1e9, 1e10, 1e99,
            1e100, 1e-99, 1e-100, 1e300, 1e-300, 5e-324, float(MAX), 2.2250738585072014e-308, 100.0, 1.0, 0.5]
    out = ["9999999.999999998", "9999999.999999999", "0.0010", "0.00099999999999999999", "1.0E7", "1.0e-3"]
    for x in vals:
        out += [repr(x), "%.17e" % x, "%.16e" % x]
    return [(t, route(t)) for t in _both_signs(out)]


def saturation():
    out = []
    for x in ["99999", "100000", "100001", "1000000000000", "0000000000000000000022", "0000000000000000000023",
              "9" * 30, str(SATURATE - 1), str(SATURATE), str(SATURATE * 10)]:
        out += [f"1e{x}", f"1e-{x}", f"1.5E+{x}", f"2.5e-{x}"]
    z = "0" * 100000
    out += ["1" + z + "e-200000",   # 1e-100000: zero
            "0." + z + "1e200000",   # 1e99999: out of range
            "1" + z + "e-100000", "1" + z + "e-100022", "1" + z + "e-100023", "1" + z + "e-99978", "1" + z + "e-99977",
            "0." + z + "1e100001", "0." + z + "1e100000", "0." + z + "123e100023", "0." + z + "123e100024",
            "0." + z + "1e99979", "0." + z + "1e99978", "1" + z + ".5e-100001", "1" + z + "0" + "e-100001",
            "1" + z + "e-99700", "0." + z + "1e100300", "1" + z, "0." + z + "1"]
    return [(t, route(t)) for t in _both_signs(out)]


def integers():
    out = ["12345678901234567890", "99999999999999999999", "10000000000000000000", "18446744073709551615",
           "18446744073709551616", "1" + "0" * 308, "9" * 308, "9" * 309, "1" + "0" * 309, "1" * 309, "1" * 310,
           str(2 ** 1023), str(int(MAX)), str(int(OVERFLOW) - 1), str(int(OVERFLOW)), str(int(OVERFLOW) + 1),
           "17976931348623157" + "0" * 292, "17976931348623159" + "0" * 292,
           str(2 ** 53 - 1), str(2 ** 53), str(2 ** 53 + 1), str(2 ** 53 + 2), str(2 ** 53 + 3), str(2 ** 64 + 1),
           "1" * 400, "9" * 4301, "1" + "0" * 5000]
    return [(t, route(t)) for t in _both_signs(out)]


def float32():
    out = []
    for k in range(-149, 128):
        a = np.float32(2.0) ** np.float32(k) if k >= -126 else np.float32(math.ldexp(1.0, k))
        for x in (np.nextafter(a, np.float32(0)), a, np.nextafter(a, np.float32(np.inf))):
            if x != 0 and np.isfinite(x):
                out.append(str(x))
    return [(t, route(t)) for t in _both_signs(sorted(set(out)))]


def sets() -> dict:
    """name -> [(text, path)], each text once, in a fixed order"""
    s = {"routing": routing(), "powers_of_two": powers_of_two(), "ties": ties(), "zeros": zeros(), "layout": layout(),
         "saturation": saturation(), "integers": integers(), "float32": float32()}
    return {k: list(dict.fromkeys(v)) for k, v in s.items()}


def fuzz(n: int, seed: int = 1) -> list:
    """n number texts within the range of a double: repr, %.17g, %.16e and %.15g of random doubles, uniformly random bit
    patterns, and random digit strings with random exponents"""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        k = rng.randrange(6)
        if k < 4:
            x = rng.random() * 10.0 ** rng.randint(-300, 300) if rng.random() < 0.5 else rng.gauss(0, 1) * 2.0 ** rng.randint(-1070, 1020)
            t = [repr, lambda v: "%.17g" % v, lambda v: "%.16e" % v, lambda v: "%.15g" % v][k](x)
        elif k == 4:
            x = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
            if math.isnan(x) or math.isinf(x):
                continue
            t = repr(x)
        else:
            d = "".join(rng.choice("0123456789") for _ in range(rng.randint(1, 40)))
            d = d.lstrip("0") or "0"
            if rng.random() < 0.5 and len(d) > 1:
                c = rng.randrange(1, len(d))
                d = d[:c] + "." + d[c:]
            e = rng.randint(-360, 330) if rng.random() < 0.5 else rng.randint(-30, 30)
            t = ("-" if rng.random() < 0.3 else "") + d + (f"e{e}" if rng.random() < 0.8 else "")
        if "inf" in t or "nan" in t or value(t) is None:
            continue
        out.append(t)
    return out


# ---- integer fields of the two readers -------------------------------------------------------------------------------------
STATUS = ["2147483647", "2147483648", "-2147483648", "-2147483649", "200", "200.0", "2e2", "-0", "0200"]
TOTAL = [str(2 ** 63 - 1), str(-(2 ** 63 - 1)), str(2 ** 63), str(-2 ** 63), "-0", "1.0", "1e3", "0", "00"]
SHARDS_FAILED = ["0", "-0", "0.0", "1", "-1", "00"]


def status_element(s: str) -> str:
    return '{"status":%s,"hits":{"total":1,"hits":[{"_id":"a","_score":1.5}]}}' % s


def total_elements(t: str) -> list:
    """hits.total as the ES 6 scalar and as the ES 7 object"""
    return ['{"hits":{"total":%s,"hits":[]}}' % t, '{"hits":{"total":{"value":%s,"relation":"eq"},"hits":[]}}' % t]


def shards_page(f: str) -> bytes:
    return ('{"_shards":{"total":1,"successful":1,"failed":%s},"hits":{"hits":[{"_id":"a","_source":{}}]}}' % f).encode()

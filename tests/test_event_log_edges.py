"""eventTime spellings and export edges for the event-export reader, held to references that do not share its code: the
calendar and offset arithmetic of `datetime`, `json.loads` for strings.  The generators here also feed the device tests
(test_gpu_event_log_edges.py): exact times, accept/reject agreement, and the host/device differences the events.py
docstring lists."""
import datetime
import json
import random
import re

import pytest

from universal_recommender_b200 import encode_ids
from universal_recommender_b200 import events as E

UTC = datetime.timezone.utc
EPOCH = datetime.datetime(1970, 1, 1, tzinfo=UTC)
MS = datetime.timedelta(milliseconds=1)
DAY_MS = 86_400_000
Y400_MS = 146_097 * DAY_MS                     # 400 proleptic Gregorian years: the calendar repeats after them
YEAR0_MS = -62_167_219_200_000                 # 0000-01-01T00:00:00Z
YEAR1_MS = (datetime.datetime(1, 1, 1, tzinfo=UTC) - EPOCH) // MS
LOCAL_MAX_MS = (datetime.datetime(9999, 12, 31, 23, 59, 59, 999000, tzinfo=UTC) - EPOCH) // MS
OFF_MAX_MS = (23 * 60 + 59) * 60_000
T_MIN, T_MAX = YEAR0_MS - OFF_MAX_MS, LOCAL_MAX_MS + OFF_MAX_MS   # 0000-01-01T00:00:00+23:59, 9999-12-31T23:59:59.999-23:59


def datetime_ms(y, mo, d, h, mi, s, frac: str, off_min: int) -> int:
    """epoch ms (floor) of a local time by datetime arithmetic; year 0 goes through year 400, which has its calendar"""
    shift = 400 if y == 0 else 0
    us = int(frac[:6].ljust(6, "0")) if frac else 0
    dt = datetime.datetime(y + shift, mo, d, h, mi, s, us, tzinfo=datetime.timezone(datetime.timedelta(minutes=off_min)))
    return (dt - EPOCH) // MS - (Y400_MS if shift else 0)


_GRAMMAR = re.compile(r"([0-9]{4})-([0-9]{2})-([0-9]{2})T([0-9]{2}):([0-9]{2}):([0-9]{2})(?:\.([0-9]{1,9}))?"
                      r"(?:Z|([+-])([0-9]{2})(?::?([0-9]{2}))?)", re.ASCII)


def ref_time(text: str):
    """the reference reading of a decoded eventTime: epoch ms, or None when it is not a time (datetime validates the
    calendar, the clock and the offset hours)"""
    m = _GRAMMAR.fullmatch(text)
    if not m:
        return None
    y, mo, d, h, mi, s = (int(m.group(k)) for k in range(1, 7))
    off = 0
    if m.group(8):
        oh, om = int(m.group(9)), int(m.group(10) or 0)
        if om > 59:
            return None
        off = (oh * 60 + om) * (-1 if m.group(8) == "-" else 1)
    try:
        return datetime_ms(y, mo, d, h, mi, s, m.group(7) or "", off)
    except (ValueError, OverflowError):
        return None


def local_fields(local_ms: int):
    """(y, mo, d, h, mi, s, ms) of a local time in years 0000-9999"""
    shift = Y400_MS if local_ms < YEAR1_MS else 0
    dt = EPOCH + datetime.timedelta(milliseconds=local_ms + shift)
    return dt.year - (400 if shift else 0), dt.month, dt.day, dt.hour, dt.minute, dt.second, dt.microsecond // 1000


def json_escape(text: str, rng, p: float) -> str:
    """the inside of a JSON string literal of text, each character written as a \\u escape with probability p"""
    out = []
    for ch in text:
        if rng.random() < p:
            out.append(("\\u%04X" if rng.random() < 0.5 else "\\u%04x") % ord(ch))
        else:
            out.append(json.dumps(ch)[1:-1])
    return "".join(out)


def random_offset(rng):
    """(text, minutes) of Z, -00:00, +-23:59, +-hh:mm, +-hhmm or +-hh"""
    k = rng.randrange(8)
    if k == 0:
        return "Z", 0
    if k == 1:
        return "-00:00", 0
    sign = rng.choice("+-")
    sg = -1 if sign == "-" else 1
    if k == 2:
        return sign + "23:59", sg * 1439
    oh, om = rng.randint(0, 23), rng.choice([0, 30, 45, rng.randint(0, 59)])
    if k in (3, 4):
        return f"{sign}{oh:02d}:{om:02d}", sg * (oh * 60 + om)
    if k in (5, 6):
        return f"{sign}{oh:02d}{om:02d}", sg * (oh * 60 + om)
    return f"{sign}{oh:02d}", sg * oh * 60


def spell(t: int, rng, offset=None, p_escape: float = 0.0):
    """a random spelling of epoch ms t -> (JSON literal inside, decoded text), or None if the offset puts its local time
    outside years 0000-9999.  0-9 fraction digits where t allows them (digits past the third are noise: a floor)."""
    off_txt, off_min = offset or random_offset(rng)
    local = t + off_min * 60_000
    if not YEAR0_MS <= local <= LOCAL_MAX_MS:
        if offset or not YEAR0_MS <= t <= LOCAL_MAX_MS:
            return None
        off_txt, off_min, local = "Z", 0, t
    y, mo, d, h, mi, s, ms = local_fields(local)
    nd = rng.choice([k for k in range(10) if k >= 3 or ms % 10 ** (3 - k) == 0])
    frac = ("%03d" % ms + "".join(rng.choice("0123456789") for _ in range(6)))[:nd]
    text = "%04d-%02d-%02dT%02d:%02d:%02d" % (y, mo, d, h, mi, s) + ("." + frac if nd else "") + off_txt
    assert datetime_ms(y, mo, d, h, mi, s, frac, off_min) == t, text   # the generator spells what it meant to
    return json_escape(text, rng, p_escape), text


def _utc(*a) -> int:
    return (datetime.datetime(*a, tzinfo=UTC) - EPOCH) // MS


# instants the calendar is easy to get wrong around: year 0 and 9999, leap centuries, a non-leap century, month and year
# ends, the epoch; random offsets move their local dates across the day, month, year and Feb 29 boundaries
SPECIAL_INSTANTS = [YEAR0_MS, YEAR0_MS + DAY_MS + 1, YEAR0_MS + 59 * DAY_MS, YEAR0_MS + 60 * DAY_MS - 1,
                    _utc(1600, 2, 29), _utc(1600, 3, 1) - 1, _utc(1600, 3, 1), _utc(1900, 2, 28, 23, 59, 59, 999000), _utc(1900, 3, 1),
                    _utc(2000, 2, 29, 12), _utc(2000, 3, 1), _utc(2000, 2, 28, 23, 30), _utc(1969, 12, 31, 23, 59, 59, 999000), 0, 1, -1000,
                    _utc(1999, 12, 31, 23), _utc(2000, 1, 1, 0, 30), _utc(2024, 2, 29, 23, 45), _utc(2100, 3, 1, 0, 15),
                    _utc(1, 1, 1), _utc(1, 1, 1) - 1, _utc(9999, 12, 31), LOCAL_MAX_MS, T_MIN, T_MAX]
EXTREME_SPELLINGS = [("0000-01-01T00:00:00+23:59", T_MIN), ("9999-12-31T23:59:59.999-23:59", T_MAX),
                     ("0000-01-01T00:00:00Z", YEAR0_MS), ("0000-02-29T23:59:59.999999999Z", YEAR0_MS + 60 * DAY_MS - 1)]


def instants(seed: int = 11, n: int = 600) -> list:
    """n distinct epoch-ms instants at least 3 ms apart (the specials first), a third of the random ones whole seconds"""
    rng = random.Random(seed)
    out = list(dict.fromkeys(SPECIAL_INSTANTS))
    taken = set(out)
    while len(out) < n:
        t = rng.randint(YEAR0_MS + 2 * DAY_MS, LOCAL_MAX_MS - 2 * DAY_MS)
        if rng.random() < 0.33:
            t -= t % 1000
        if any(t + d in taken for d in range(-2, 3)):
            continue
        taken.add(t)
        out.append(t)
    return out


def time_spellings(seed: int = 11, n_instants: int = 600, per: int = 6):
    """[(instant index j, delta in {-1, 0, 1}, JSON literal inside, decoded text, epoch ms)]: per spellings of each m_j - 1,
    m_j and m_j + 1 that can be spelled, the extreme spellings, and some spellings written all in \\u escapes"""
    rng = random.Random(seed)
    ins = instants(seed, n_instants)
    out = []
    for j, m in enumerate(ins):
        for delta in (-1, 0, 1):
            for _ in range(per):
                s = spell(m + delta, rng, p_escape=rng.choice([0.0, 0.0, 0.0, 0.2, 1.0]))
                if s is not None:
                    out.append((j, delta, s[0], s[1], m + delta))
    for text, t in EXTREME_SPELLINGS:
        out.append((ins.index(t) if t in ins else -1, 0, text, text, t))
    return ins, out


# decoded eventTimes the reader must refuse: the host cases first, then the edges of the device's own parser
HOST_REJECTS = ["2017-05-01T12:34:56", "2017-05-01 12:34:56Z", "2017-5-01T12:34:56Z", "2017-02-29T00:00:00Z",
                "2017-05-01T24:00:00Z", "2017-05-01T12:60:00Z", "2017-05-01T12:34:60Z", "2017-05-01T12:34:56.Z",
                "2017-05-01T12:34:56.1234567890Z", "2017-05-01T12:34:56+24:00", "2017-05-01T12:34:56+05:3",
                "2017-05-01T12:34:56+5", "2017-05-01T12:34:56z", "2017-05-01T12:34:56Z ", "+2017-05-01T12:34:56Z",
                "２017-05-01T12:34:56Z", "2017-13-01T00:00:00Z", "2017-00-10T00:00:00Z", "1900-02-29T00:00:00Z"]
REJECT_LITERALS = [json.dumps(t, ensure_ascii=False)[1:-1] for t in HOST_REJECTS] + [
    "2017-05-01T12:34:56.0000000000Z", "1969-12-31T23:59:59.9999999999+01:00", "2017-05-01T12:34:56+05:60", "2017-05-01T12:34:56-24:00",
    "2017-05-01T12:34:56+0560", "2017-05-01T12:34:56-24", "2017-05-01T12:34:56.123456789+05:30000000", "2017-05-01T12:34:56.123456789+05:30\\u0000",
    "2017-05-01T12:34:56Z+05:00", "2017-05-01T12:34:56Z-00:00", "2017-05-01T12:34:56\\u0000Z", "\\u00002017-05-01T12:34:56Z",
    "2017-05-01T12:34:56+05:30:00", "2017-05-01T12:34:56+0530Z", "2017-05-01T12:34:56-", "2017-05-01T12:34:56+", "2017-05-01T12:34:56..1Z",
    "2017-05-01t12:34:56Z", "", "Z", "2017-05-01T12:34:56.1Z1", "12017-05-01T12:34:56Z", "-2017-05-01T12:34:56Z", "2017-05-01T1:34:56Z",
    "2100-02-29T00:00:00Z", "1700-02-29T00:00:00Z", "2000-02-30T00:00:00Z", "2017-04-31T00:00:00Z", "2017-05-00T00:00:00Z",
    "2017-05-01T12:34:56\\u00e9Z", "2017-05-01T12:34:56\\ud800Z", "2017-05-01T12:34:56\\u005a\\u005a", "2017-05-01T12:34:56\\u0020Z",
    "2017-05-01T12:34:56.\\u0030\\u0030\\u0030\\u0030\\u0030\\u0030\\u0030\\u0030\\u0030\\u0030Z", "2017-05-01T12:34:56+\\u00324:00",
    "2017-05-01T12:34:56.123+05:30" + " " * 13, "9999-12-31T23:59:59.999-23:59:00", "10000-01-01T00:00:00Z", "2017-05-01T12:34:56Z\\n"]
# spellings the reader must accept, with escapes where a careless decoder would stop
ACCEPT_LITERALS = ["2017-05-01\\u005412:34:56Z", "2017-05-01\\u005412:34:56.123456789\\u002B05\\u003a30", "\\u0032017-05-01T12:34:56Z",
                   "2017-05-01T12:34:56\\u005A", "2017-05-01T12:34:56.5\\u002b05:30",
                   json_escape("2017-05-01T12:34:56.123456789+05:30", random.Random(0), 1.0), "1900-03-01T00:00:00.000000001-00:00",
                   "2000-02-29T23:59:59.999+00", "1600-02-29T00:00:00+2359", "0000-12-31T23:59:59.9-0001"]


def decode_literal(lit: str) -> str:
    return json.loads('"' + lit + '"')


MUTATION_ALPHABET = "0123456789-:T.Z+ zt"


def time_mutants(seed: int = 5, n: int = 1500) -> list:
    """n distinct single-character edits (replace, delete, insert from MUTATION_ALPHABET) of valid decoded spellings"""
    rng = random.Random(seed)
    base = [text for _, _, _, text, _ in time_spellings(seed, 40, 2)[1]]
    out = {}
    while len(out) < n:
        t = rng.choice(base)
        i = rng.randrange(len(t) + 1)
        op = rng.randrange(3)
        c = rng.choice(MUTATION_ALPHABET)
        if op == 0 and i < len(t):
            m = t[:i] + c + t[i + 1:]
        elif op == 1 and i < len(t):
            m = t[:i] + t[i + 1:]
        else:
            m = t[:i] + c + t[i:]
        if m != t:
            out.setdefault(m, None)
    return list(out)


def mirror_time(text: str):
    try:
        return E.parse_event_time(text)
    except ValueError:
        return None


# ---- the mirror against datetime ----------------------------------------------------------------------------------------
def test_year_zero_anchor_and_extremes():
    assert datetime_ms(0, 1, 1, 0, 0, 0, "", 0) == YEAR0_MS
    assert datetime_ms(400, 1, 1, 0, 0, 0, "", 0) - Y400_MS == YEAR0_MS
    assert E.parse_event_time("0000-01-01T00:00:00Z") == YEAR0_MS
    for text, t in EXTREME_SPELLINGS:
        assert ref_time(text) == t and E.parse_event_time(text) == t, text
    assert E.days_from_civil(0, 3, 1) - E.days_from_civil(0, 2, 28) == 2   # year 0 is a leap year


def test_spellings_agree_with_datetime():
    ins, sp = time_spellings()
    assert len(ins) >= 500 and len(sp) >= 10_000
    assert sum(1 for s in sp if "\\u" in s[2]) > 1000
    for j, delta, lit, text, t in sp:
        assert decode_literal(lit) == text
        assert ref_time(text) == t, text
        assert E.parse_event_time(text) == t, text
    # every form is there: fraction lengths 0-9, each offset form, years 0000 and 9999, pre-1970
    texts = [s[3] for s in sp]
    assert {len(re.search(r"(?:\.([0-9]*))?(?:Z|[+-][0-9:]*)$", x).group(1) or "") for x in texts} == set(range(10))
    for pat in (r"Z$", r"-00:00$", r"[+-]23:59$", r"[+-][0-9]{2}:[0-9]{2}$", r"[+-][0-9]{4}$", r"[+-][0-9]{2}$", r"^0000-", r"^9999-", r"^1[0-8]"):
        assert any(re.search(pat, x) for x in texts), pat


@pytest.mark.parametrize("lit", REJECT_LITERALS)
def test_mirror_rejects(lit):
    text = decode_literal(lit)
    assert ref_time(text) is None
    with pytest.raises(ValueError):
        E.parse_event_time(text)


@pytest.mark.parametrize("lit", ACCEPT_LITERALS)
def test_mirror_accepts(lit):
    text = decode_literal(lit)
    assert ref_time(text) is not None
    assert E.parse_event_time(text) == ref_time(text)


def test_mutation_fuzz_mirror_agrees_with_datetime():
    mut = time_mutants()
    assert len(mut) == 1500
    n_acc = 0
    for text in mut:
        assert mirror_time(text) == ref_time(text), text
        n_acc += ref_time(text) is not None
    assert 100 < n_acc < 1400   # both verdicts are exercised


# ---- the mirror's line decoding ---------------------------------------------------------------------------------------------
GOOD = b'{"event":"v","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z"}'
BOM = b"\xef\xbb\xbf"


@pytest.mark.parametrize("at", [0, 1, 2])
def test_a_byte_order_mark_is_not_whitespace(at):
    lines = [GOOD, GOOD, GOOD]
    lines[at] = BOM + lines[at]
    with pytest.raises(ValueError, match=f"line {at}"):
        E.read_export(b"\n".join(lines))
    # inside a string it is an ordinary character
    got = E.read_export(GOOD.replace(b'"u"', b'"u' + BOM + b'"'))
    assert got.ranking_events == {"v": []} and E.parse_line(0, GOOD.replace(b'"u"', b'"u' + BOM + b'"')).entity_id == "u\ufeff"


@pytest.mark.parametrize("bad", [b"\xff", b"\xc3", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\xc0\xaf"])
def test_invalid_utf8_raises_naming_the_line(bad):
    with pytest.raises(ValueError, match="line 1"):
        E.read_export(GOOD + b"\n" + GOOD.replace(b'"u"', b'"u' + bad + b'"') + b"\n")


def test_lone_surrogate_escapes_cannot_be_encoded():
    line = (b'{"event":"buy","entityType":"user","entityId":"\\ud800","targetEntityType":"item","targetEntityId":"\\udc00x",'
            b'"eventTime":"2020-01-01T00:00:00Z"}')
    got = E.read_export(line)
    assert got.events == [("\ud800", "buy", "\udc00x", 1577836800000)]
    with pytest.raises(UnicodeEncodeError):
        encode_ids([got.events[0][0]])


def test_mismatched_brackets_in_a_nested_value_raise():
    line = b'{"event":"$set","entityType":"item","entityId":"i","eventTime":"2020-01-01T00:00:00Z","properties":{"p":{"a":{]}}}'
    with pytest.raises(ValueError, match="line 0"):
        E.read_export(line)

"""CPU tests of REGEXP_LIKE and LIKE: the pattern compiler and matcher (pinot_b200/csrc/pb200_pattern.h, the code the
device kernel runs) compiled with g++ through tests/pattern_probe and held to the independent reference
tests/pattern_ref.py; the LIKE rewrite against a wildcard matcher; the SQL front end's forms and refusals."""
import ctypes as C
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import pattern_ref as R
from pinot_b200 import sql
from pinot_b200.query import Filter, Predicate, optimize_filter

HERE = os.path.dirname(os.path.abspath(__file__))
OK, UNSUPPORTED, INVALID = 0, 1, 2


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = tmp_path_factory.mktemp("pattern_probe") / "libpattern_probe.so"
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-Wall", "-Werror", "-o", str(out),
                    os.path.join(HERE, "pattern_probe", "pattern_probe.cpp")], check=True)
    lib = C.CDLL(str(out))
    lib.probe_pattern_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_int32]
    lib.probe_pattern_match.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def compile_status(probe, pattern):
    why = C.create_string_buffer(256)
    p = pattern if isinstance(pattern, bytes) else pattern.encode("utf-8")
    return probe.probe_pattern_compile(p, why, 256), why.value.decode()


def match(probe, pattern, entries):
    data = b"".join(entries)
    offsets = np.zeros(len(entries) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(e) for e in entries])
    buf = np.frombuffer(data + b"\0", dtype=np.uint8)
    out = np.zeros(max(1, len(entries)), dtype=np.uint8)
    rc = probe.probe_pattern_match(pattern.encode("utf-8"), buf.ctypes.data, offsets.ctypes.data, len(entries), out.ctypes.data)
    assert rc == OK, pattern
    return [bool(x) for x in out[:len(entries)]]


# --------------------------------------------------------------------------------------------------- accepted / refused
ACCEPTED = [
    "", "a", "abc", "^abc", "abc$", "^$", "^", "$", ".", "a.c", "a*", "a+", "a?", "a{3}", "a{2,}", "a{2,4}", "a{0}",
    "a{0,1}", "a*?", "a+?", "a??", "a{2,3}?", "(ab)+", "(?:ab)*c", "a|b", "a||b", "|a", "(|a)", "()", "(a|)*",
    "[abc]", "[^abc]", "[a-z0-9_]", "[^\\n]", "[\\d\\s]", "[\\x41-\\x5A]", "[\\u00e0-\\u00ff]", "[é-ü]", "[a^]", "[a$]",
    "\\d+", "\\D", "\\w\\W", "\\s\\S", "\\t\\n\\r\\f\\a\\e", "\\x41", "\\u00e9", "\\.", "\\*", "\\\\", "\\$", "a\\$",
    "\\[", "\\]", "\\{", "\\}", "\\(", "\\)", "\\|", "\\-", "\\/", "/api/v[0-9]+/users", "^https?://[^/]+/", "日本",
    "😀+", "[😀-😂]", ".{64}", "(a|b){32}", "a{0,63}b", "^(?:a|b)$", "\\^", "a\\\\$",
]

REFUSED = [
    "(a)\\1", "(?=a)", "(?!a)", "(?<=a)", "(?<!a)", "\\b", "\\B", "\\A", "\\z", "\\Z", "\\G", "\\p{L}", "\\P{L}",
    "\\Qa\\E", "\\0", "\\01", "(?i)a", "(?i:a)", "a*+", "a++", "a?+", "a{2}+", "[a&&b]", "[a[b]]", "[]a]", "[^]a]",
    "[a-]", "[-a]", "[a-c-e]", "[\\d-z]", "[z-a]", "a]", "]", "a{", "a{x}", "a{,3}", "}", "a}", "a^", "^^a", "a$b",
    "$a", "a$$", "\\y", "\\h", "\\v", "\\R", "\\X", "\\N", "\\c", "\\x4", "\\x{41}", "\\u12", "\\ud800", "*a", "+",
    "?", "{2}", "a**", "a*{2}", "(*)", "(|*)", "a{3,2}", "(", ")", "(a", "a)", "[abc", "\\", "^a|b", "a|b$", "(?<n>a)",
    "(?>a)", "a{65}", ".{65}", "(a|b){33}", "(.{8}){9}", "a{0,64}b", "a{100000000}", "[abc", "\\é",
    "[" + "".join(chr(0x100 + 2 * k) for k in range(70)) + "]",
]


@pytest.mark.parametrize("pattern", ACCEPTED)
def test_accepted_patterns_compile(probe, pattern):
    rc, why = compile_status(probe, pattern)
    assert rc == OK, (pattern, why)


@pytest.mark.parametrize("pattern", REFUSED)
def test_refused_patterns(probe, pattern):
    rc, why = compile_status(probe, pattern)
    assert rc == UNSUPPORTED and why, (pattern, rc)


def test_pattern_that_is_not_utf8_is_invalid(probe):
    for bad in (b"a\xff", b"\xc3", b"\xed\xa0\x80", b"\xc0\xaf", b"\xf4\x90\x80\x80"):
        assert compile_status(probe, bad)[0] == INVALID, bad


# ---------------------------------------------------------------------------------------------------- the matcher
EDGE_ENTRIES = [
    b"", b"a", b"ab", b"abc", b"xabcx", b"\n", b"\r", b"\r\n", b"a\n", b"a\r", b"a\r\n", b"a\n\n", b"a\r\r", b"\na",
    b"a\nb", "a\u0085".encode(), "a ".encode(), "a ".encode(), "\u0085".encode(), "a b".encode(),
    "é".encode(), "aé".encode(), "日本語".encode(), "x😀y".encode(), "😀😀".encode(), b"\xff", b"a\xffb", b"\xe2\x82",
    b"\xe2\x82a", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf0\x9f\x98", "�".encode(), b"abc\0\0\0", b"ab\0c",
    b"aaaa", b"aaaaaaaa", b"ababab", b"123", b"a1_ b", b"\t\x0b\x0c", b"\x1b\x07", b"/api/v2/users/17",
    b"https://example.com/x", b"HTTP://EXAMPLE.COM/", bytes(range(1, 128)), bytes(range(128, 256)),
]


def test_matcher_against_the_reference_on_edge_entries(probe):
    for pattern in ACCEPTED:
        got = match(probe, pattern, EDGE_ENTRIES)
        want = [R.matches(pattern, e) for e in EDGE_ENTRIES]
        bad = [(e, g, w) for e, g, w in zip(EDGE_ENTRIES, got, want) if g != w]
        assert not bad, (pattern, bad[:5])


def test_full_width_entries_without_nul(probe):
    """An entry that fills its padded width has no NUL: its last byte belongs to the value."""
    entries = [b"abcd", b"abc\0", b"ab\0\0"]
    assert match(probe, "d$", entries) == [True, False, False]
    assert match(probe, "^abc$", entries) == [False, True, False]


def _random_pattern(rng):
    atoms = ["a", "b", ".", "[ab]", "[^a]", "\\d", "\\w", "\\s", "é", "\\n", "(a|b)", "(?:ab|)", "[a-c]", "😀", "\\W"]
    quants = ["", "", "*", "+", "?", "{2}", "{1,3}", "{0,2}", "{2,}", "*?"]
    body = "".join(rng.choice(atoms) + rng.choice(quants) for _ in range(rng.randint(0, 5)))
    if rng.random() < 0.3:
        body = rng.choice(["a", "b|c", ""]) + "|" + body
        return body   # no anchors next to a top-level |
    return ("^" if rng.random() < 0.3 else "") + body + ("$" if rng.random() < 0.3 else "")


def _random_entry(rng):
    pool = ["a", "b", "c", "1", "_", " ", "\n", "\r", "é", "😀", " ", "\u0085", "x"]
    s = "".join(rng.choice(pool) for _ in range(rng.randint(0, 8))).encode()
    if rng.random() < 0.1:
        s += rng.choice([b"\xff", b"\xe2\x82", b"\xc0"])
    return s


def test_matcher_against_the_reference_on_random_patterns(probe):
    rng = random.Random(7)
    entries = [_random_entry(rng) for _ in range(300)] + EDGE_ENTRIES
    checked = 0
    for _ in range(400):
        pattern = _random_pattern(rng)
        rc, why = compile_status(probe, pattern)
        if rc != OK:
            assert "64" in why, (pattern, why)   # the generator only writes accepted syntax
            continue
        got = match(probe, pattern, entries)
        want = [R.matches(pattern, e) for e in entries]
        bad = [(e, g, w) for e, g, w in zip(entries, got, want) if g != w]
        assert not bad, (pattern, bad[:5])
        checked += 1
    assert checked > 300


def test_64_positions(probe):
    assert match(probe, "a{64}", [b"a" * 63, b"a" * 64, b"b" + b"a" * 64]) == [False, True, True]
    assert match(probe, "^(?:ab){32}$", [b"ab" * 32, b"ab" * 31, b"ab" * 33]) == [True, False, False]


# ----------------------------------------------------------------------------------------------------- LIKE
LIKES = ["", "%", "%%", "a", "a%", "%a", "%a%", "a_c", "_", "__", "%_%", "a%c", "%a%c%", "a.c", "a*", "(a)", "[a]",
         "a$", "^a", "a|b", "a+b", "a?", "{a}", "é_", "%😀%", "100%", "_%_", "%%a%%"]
VALUES = ["", "a", "ab", "abc", "ac", "a.c", "axc", "a\nc", "\na", "a\n", "a\r\n", "ba", "bab", "a*", "(a)", "[a]", "a$",
          "^a", "a|b", "a+b", "a?", "{a}", "éx", "é\n", "x😀y", "100%", "1000", "aa", "a c", " a "]


def test_like_rewrite_against_a_wildcard_matcher(probe):
    for like in LIKES:
        regex = sql.like_to_regexp(like)
        assert compile_status(probe, regex)[0] == OK, (like, regex)
        got = match(probe, regex, [v.encode() for v in VALUES])
        want = [R.like_matches(like, v) for v in VALUES]
        assert got == want, (like, regex, [(v, g, w) for v, g, w in zip(VALUES, got, want) if g != w])


def test_like_rewrite_rules():
    assert sql.like_to_regexp("") == "^$"
    assert sql.like_to_regexp("%") == sql.like_to_regexp("%%%") == ""
    assert sql.like_to_regexp("a%") == "^a"
    assert sql.like_to_regexp("%a") == "a$"
    assert sql.like_to_regexp("%%a%%") == "a"
    assert sql.like_to_regexp("a_b%c") == "^a.b.*c$"
    assert sql.like_to_regexp("a.b(c)") == "^a\\.b\\(c\\)$"
    with pytest.raises(sql.SqlError):
        sql.like_to_regexp("a\\%")


# ----------------------------------------------------------------------------------------------------- SQL forms
def _leaf(f):
    return f.children[0] if isinstance(f, Filter) and f.type == "NOT" else f


def test_sql_forms():
    q = sql.parse("SELECT COUNT(*) FROM t WHERE u LIKE 'a%'")
    assert q.filter == Predicate("REGEXP_LIKE", "u", ["^a"])
    q = sql.parse("SELECT COUNT(*) FROM t WHERE u NOT LIKE '%b'")
    assert q.filter == Filter("NOT", [Predicate("REGEXP_LIKE", "u", ["b$"])])
    q = sql.parse("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, '^x[0-9]+$')")
    assert q.filter == Predicate("REGEXP_LIKE", "u", ["^x[0-9]+$"])
    q = sql.parse("SELECT COUNT(*) FROM t WHERE NOT regexp_like(u, 'x')")
    assert q.filter == Filter("NOT", [Predicate("REGEXP_LIKE", "u", ["x"])])
    q = sql.parse("SELECT COUNT(*) FILTER (WHERE u LIKE '%x%'), SUM(m) FROM t WHERE k = 1 GROUP BY k")
    assert q.aggregations[0].filter == Predicate("REGEXP_LIKE", "u", ["x"])
    s = sql.parse_selection("SELECT u FROM t WHERE u LIKE 'a%' OR REGEXP_LIKE(v, 'b') LIMIT 5")
    assert s.filter.type == "OR" and [c.type for c in s.filter.children] == ["REGEXP_LIKE", "REGEXP_LIKE"]
    d = sql.parse_distinct("SELECT DISTINCT u FROM t WHERE u NOT LIKE 'a%'")
    assert _leaf(d.filter) == Predicate("REGEXP_LIKE", "u", ["^a"])


@pytest.mark.parametrize("text", [
    "SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 'a', 'i')",
    "SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 3)",
    "SELECT COUNT(*) FROM t WHERE u LIKE 3",
    "SELECT COUNT(*) FROM t WHERE u LIKE 'a\\%'",
    "SELECT COUNT(*) FROM t WHERE u NOT = 'a'",
    "SELECT k, COUNT(*) FROM t GROUP BY k HAVING REGEXP_LIKE(k, 'a')",
    "SELECT k, COUNT(*) FROM t GROUP BY k HAVING COUNT(*) LIKE 'a'",
])
def test_sql_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


def test_pattern_leaves_are_never_merged():
    """flatten / optimize_filter merge EQ and IN leaves of an OR and RANGE leaves of an AND, never a pattern leaf."""
    a, b = Predicate("REGEXP_LIKE", "u", ["a"]), Predicate("REGEXP_LIKE", "u", ["b"])
    f = optimize_filter(Filter("OR", [a, Filter("OR", [b, Predicate("EQ", "u", ["c"])])]))
    assert f.type == "OR" and sorted(str(c.values) for c in f.children) == ["['a']", "['b']", "['c']"]
    f = optimize_filter(Filter("AND", [a, b]))
    assert f == Filter("AND", [a, b])
    q = sql.parse("SELECT COUNT(*) FROM t WHERE u LIKE 'a%' OR u = 'x' OR u = 'y'")
    assert sorted(c.type for c in q.filter.children) == ["IN", "REGEXP_LIKE"]


def test_reference_decoder():
    assert R.decode(b"\xe2\x82a") == "��a"
    assert R.decode("😀é".encode()) == "😀é"
    assert R.decode(b"\xed\xa0\x80") == "�" * 3
    assert list(itertools.islice(R.decode(b"\xff\xfe"), 5)) == ["�", "�"]

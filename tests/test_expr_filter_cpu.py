"""Predicates on expressions over two or more columns without a GPU (DESIGN.md section 3.16): the parser's comparison
rewrites (the reference's PredicateComparisonRewriter) and refusals, the comparison the doc-mask pass runs
(pb200::expr_matches through a g++ probe) against tests/float_edges_ref.raw_matches at NaN, +-0.0, +-inf, subnormals, every
bound kind, IN with duplicates and both zeros and literals beyond 2^53, which filter leaves are evaluated per row, and the
pb200h_explain text of trees that mix expression leaves with folded, sorted and inverted leaves."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from float_edges_ref import raw_matches
from oracle import segment_builder as sb
from pinot_b200 import _lib, sql
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED
from pinot_b200.plan_maker import _marshal_query
from pinot_b200.query import Filter, Predicate

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "expr_filter_probe", "expr_filter_probe.cpp")
    out = os.path.join(HERE, "expr_filter_probe", "libexpr_filter_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    deps = [src, _lib.LIB_PATH, os.path.join(ROOT, "pinot_b200", "csrc", "pb200_expr.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.efp_matches.argtypes = [C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.efp_is_expression_filter.argtypes = [C.c_char_p]
    lib.efp_explain.restype = C.c_int32
    lib.efp_explain.argtypes = [C.POINTER(_lib.HColumn), C.c_int32, C.c_int32, C.POINTER(_lib.HQuery), C.c_char_p, C.c_int32]
    return lib


def _where(text):
    return sql.parse(f"SELECT COUNT(*) FROM t WHERE {text}").filter


# ---- the parser ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("text,want", [
    ("a > b", Predicate("RANGE", "minus(a,b)", [], 0, None, False, True)),
    ("a >= b", Predicate("RANGE", "minus(a,b)", [], 0, None, True, True)),
    ("a < b", Predicate("RANGE", "minus(a,b)", [], None, 0, True, False)),
    ("a = b", Predicate("EQ", "minus(a,b)", [0])),
    ("a <> b", Predicate("NEQ", "minus(a,b)", [0])),
    ("a != b * 2", Predicate("NEQ", "minus(a,times(b,'2'))", [0])),
    ("5 < a", Predicate("RANGE", "a", [], 5, None, False, True)),
    ("5 >= a * b", Predicate("RANGE", "times(a,b)", [], None, 5, True, True)),
    ("2.5 = a - b", Predicate("EQ", "minus(a,b)", [2.5])),
    ("a + b IN (1, 2)", Predicate("IN", "plus(a,b)", [1, 2])),
    ("a + b NOT IN (1, 2, 2)", Predicate("NOT_IN", "plus(a,b)", [1, 2, 2])),
    ("a * b BETWEEN 1 AND 10", Predicate("RANGE", "times(a,b)", [], 1, 10, True, True)),
    ("end_ts - start_ts > 60000", Predicate("RANGE", "minus(end_ts,start_ts)", [], 60000, None, False, True)),
    ("NOT a > b", Filter("NOT", [Predicate("RANGE", "minus(a,b)", [], 0, None, False, True)])),
])
def test_parser_rewrites(text, want):
    assert _where(text) == want


def test_parser_rewrites_inside_trees():
    got = _where("a > b AND (c = 3 OR price * qty > 1000)")
    assert got == Filter("AND", [Predicate("RANGE", "minus(a,b)", [], 0, None, False, True),
                                 Filter("OR", [Predicate("EQ", "c", [3]),
                                               Predicate("RANGE", "times(price,qty)", [], 1000, None, False, True)])])
    assert sql.parse_selection("SELECT a FROM t WHERE bytes_out > bytes_in LIMIT 3").filter == \
        Predicate("RANGE", "minus(bytes_out,bytes_in)", [], 0, None, False, True)
    # a FILTER clause takes the same rewrite
    q = sql.parse("SELECT SUM(a * b) FILTER (WHERE a * b > 0), COUNT(*) FROM t")
    assert q.aggregations[0].filter == Predicate("RANGE", "times(a,b)", [], 0, None, False, True)
    # HAVING is unchanged: aggregations against literals
    assert sql.parse("SELECT g, COUNT(*) FROM t GROUP BY g HAVING COUNT(*) > 3").having is not None


@pytest.mark.parametrize("text", ["a BETWEEN b AND 3", "a BETWEEN 1 AND b", "a * b BETWEEN c AND 10", "a IN (1, b)", "a NOT IN (b)",
                                  "1 < 2", "5 BETWEEN a AND b", "5 IN (a)"])
def test_parser_refusals(text):
    with pytest.raises(sql.SqlError):
        _where(text)


# ---- the comparison (pb200_expr.h expr_matches) against raw_matches -------------------------------------------------------
EQ, NEQ, IN, NOT_IN, RANGE = (_lib.EXPR_OPS[k] for k in ("EQ", "NEQ", "IN", "NOT_IN", "RANGE"))
EDGES = [math.nan, -math.nan, 0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 1.0, -1.0, 2.5, 3.0,
         1e300, -1e300, float(2 ** 53), float(2 ** 53 + 2), float(-(2 ** 53)), 0.1, 1.7976931348623157e308]
LITERALS = [0, 0.0, -0.0, 1, -1, 2.5, 3, 2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 63 + 5, 1e300, 5e-324, math.inf, -math.inf]


def _probe_matches(probe, p: Predicate, xs):
    if p.type == "RANGE":
        flags = (1 if p.lower is None else 0) | (2 if p.upper is None else 0) | (0 if p.lower_inclusive else 4) | (0 if p.upper_inclusive else 8)
        lo = 0.0 if p.lower is None else float(p.lower)
        hi = 0.0 if p.upper is None else float(p.upper)
        vals = np.zeros(1)
        nv, op = 0, RANGE
    else:
        vals = np.array([float(v) for v in p.values], dtype=np.float64)
        nv, op, flags, lo, hi = len(vals), _lib.EXPR_OPS[p.type], 0, 0.0, 0.0
    x = np.array(xs, dtype=np.float64)
    out = np.zeros(len(x), dtype=np.uint8)
    probe.efp_matches(op, flags, lo, hi, vals.ctypes.data, nv, x.ctypes.data, len(x), out.ctypes.data)
    return [bool(v) for v in out]


def _predicates():
    out = []
    for a in LITERALS:
        out += [Predicate("EQ", "e", [a]), Predicate("NEQ", "e", [a])]
        for inc in (True, False):
            out += [Predicate("RANGE", "e", [], a, None, inc, True), Predicate("RANGE", "e", [], None, a, True, inc)]
        for b in LITERALS[::3]:
            for li in (True, False):
                for ui in (True, False):
                    out.append(Predicate("RANGE", "e", [], a, b, li, ui))
    out += [Predicate("RANGE", "e", [], None, None, True, True)]   # both sides unbounded: every value but NaN
    for vals in ([1, 1, 2.5], [0.0, -0.0], [-0.0], [2 ** 53 + 1, 2 ** 53], [math.inf, -math.inf, 0], [5e-324, 3, 3]):
        out += [Predicate("IN", "e", vals), Predicate("NOT_IN", "e", vals)]
    return out


def test_comparison_matches_the_reference_rule(probe):
    rng = np.random.default_rng(16)
    xs = EDGES + list(rng.normal(scale=5, size=40)) + list(rng.integers(-4, 5, size=20).astype(float))
    n = 0
    for p in _predicates():
        got = _probe_matches(probe, p, xs)
        want = [raw_matches(x, p, sb.DOUBLE) for x in xs]
        assert got == want, p
        n += 1
    assert n > 300


def test_comparison_edges_spelled_out(probe):
    nan = math.nan
    assert _probe_matches(probe, Predicate("NEQ", "e", [1]), [nan]) == [True]
    assert _probe_matches(probe, Predicate("NOT_IN", "e", [1, 2]), [nan]) == [True]
    assert _probe_matches(probe, Predicate("EQ", "e", [0]), [0.0, -0.0, nan]) == [True, True, False]
    assert _probe_matches(probe, Predicate("RANGE", "e", [], None, None, True, True), [nan, -math.inf, math.inf]) == [False, True, True]
    assert _probe_matches(probe, Predicate("RANGE", "e", [], 0, None, False, True), [-0.0, 0.0, 5e-324]) == [False, False, True]
    # a literal beyond 2^53 is compared as the double it rounds to
    assert _probe_matches(probe, Predicate("EQ", "e", [2 ** 53 + 1]), [float(2 ** 53)]) == [True]


# ---- which leaves are evaluated per row ------------------------------------------------------------------------------
@pytest.mark.parametrize("text,want", [("minus(a,b)", 1), ("times(price,qty)", 1), ("plus(times(a,'2'),b)", 1), ("a", 0),
                                       ("times(a,'2')", 0), ("minus(a,a)", 0), ("plus(a,plus(a,'1'))", 0),
                                       ("datetrunc('DAY',ts)", 0), ("plus(datetrunc('DAY',ts),b)", 1)])
def test_expression_filter_leaves(probe, text, want):
    assert probe.efp_is_expression_filter(text.encode()) == want


# ---- pb200h_explain ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_segment(oracle):
    rng = np.random.default_rng(3)
    n = 2000
    seg = oracle.build_segment("ef", {"a": rng.integers(0, 50, size=n).astype(np.int32),
                                      "b": rng.integers(0, 10, size=n).astype(np.int32),
                                      "s": np.sort(rng.integers(0, 8, size=n)).astype(np.int32),
                                      "d": rng.normal(size=n),
                                      "name": np.array([b"x", b"y"])[rng.integers(0, 2, size=n)]}, inverted=["b"])
    arr = (_lib.HColumn * len(seg.columns))()
    keep = []
    for i, c in enumerate(seg.columns):
        nm = c.name.encode()
        keep.append(nm)
        has_inv = c.inv is not None and not c.is_sorted
        arr[i] = _lib.HColumn(nm, c.data_type, 1, c.bits, c.cardinality, int(c.is_sorted), c.dict_entry_bytes, c.fwd.ctypes.data,
                              len(c.fwd), c.dict.ctypes.data, len(c.dict), c.inv.ctypes.data if has_inv else None,
                              len(c.inv) if has_inv else 0)
    return seg, arr, keep


def _explain(probe, host_segment, text):
    seg, arr, _ = host_segment
    hq, keep = _marshal_query(sql.parse(text), False)
    buf = C.create_string_buffer(8192)
    m = probe.efp_explain(arr, len(seg.columns), seg.num_docs, C.byref(hq), buf, 8192)
    return m, buf.value.decode()


def test_explain_trees(probe, host_segment):
    ex = lambda t: _explain(probe, host_segment, t)[1]
    assert ex("SELECT SUM(a) FROM t WHERE a > b") == "AGGREGATE(FILTER_EXPRESSION(RANGE,minus(a,b)))"
    assert ex("SELECT SUM(a) FROM t WHERE a * d IN (1, 2)") == "AGGREGATE(FILTER_EXPRESSION(IN,times(a,d)))"
    assert ex("SELECT SUM(a) FROM t WHERE a - d <> 3") == "AGGREGATE(FILTER_EXPRESSION(NOT_EQ,minus(a,d)))"
    # never folded: an expression leaf is no constant, next to leaves that are
    assert ex("SELECT SUM(a) FROM t WHERE a > b AND a >= 0") == \
        "AGGREGATE(FILTER_AND(FILTER_EXPRESSION(RANGE,minus(a,b)),FILTER_MATCH_ENTIRE_SEGMENT))"
    assert ex("SELECT SUM(a) FROM t WHERE a > b AND a > 1000") == "EMPTY(FILTER_EMPTY)"
    assert ex("SELECT MAX(a) FROM t WHERE a > b OR a >= 0") == "AGGREGATE_NO_SCAN(FILTER_MATCH_ENTIRE_SEGMENT)"
    assert ex("SELECT SUM(a) FROM t WHERE NOT (a + b BETWEEN 3 AND 9)") == "AGGREGATE(FILTER_NOT(FILTER_EXPRESSION(RANGE,plus(a,b))))"
    g = ex("SELECT SUM(a) FROM t WHERE s = 2 AND b = 3 AND a * b > d GROUP BY b")
    assert g == ("GROUP_BY(FILTER_AND(FILTER_SORTED_INDEX(EQ,s),FILTER_INVERTED_INDEX(EQ,b),"
                 "FILTER_EXPRESSION(RANGE,minus(times(a,b),d))))")
    two = ex("SELECT COUNT(*) FROM t WHERE a > b OR a * d < 0")
    assert two == "AGGREGATE(FILTER_OR(FILTER_EXPRESSION(RANGE,minus(a,b)),FILTER_EXPRESSION(RANGE,times(a,d))))"


def test_explain_refusals(probe, host_segment):
    for text, code in (("SELECT SUM(a) FROM t WHERE a - name > 0", E_UNSUPPORTED),          # a STRING leaf
                       ("SELECT SUM(a) FROM t WHERE REGEXP_LIKE(a * b, 'x')", E_UNSUPPORTED),
                       ("SELECT SUM(a) FROM t WHERE a + b LIKE 'x%'", E_UNSUPPORTED),
                       ("SELECT SUM(a) FROM t WHERE plus(datetrunc('DAY', a), b) > 0", E_UNSUPPORTED),
                       ("SELECT SUM(a) FROM t WHERE " + "plus(" * 8 + "a" + ",b)" * 8 + " > 0", E_UNSUPPORTED),
                       ("SELECT SUM(a) FROM t WHERE a * b = 'x'", E_UNSUPPORTED),
                       ("SELECT SUM(a) FROM t WHERE a * nosuch > 0", E_INVALID)):
        m, _ = _explain(probe, host_segment, text)
        assert m == code, text

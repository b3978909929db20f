"""CASE WHEN aggregations without a GPU (DESIGN.md section 3.19): the SQL parser's canonical text and refusals, the host
compiler, the program check on malformed CASE programs, the evaluator of pb200_expr.h through a g++ probe against the
independent reference tests/case_ref.py, and the host's condition resolution against the values it stands for."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import case_ref
from pinot_b200 import _lib, sql
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED
from pinot_b200.query import is_multi_column_expression

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
T_COLUMN, T_LONG, T_PLUS = 0, 1, 3
INT, LONG, FLOAT, DOUBLE, STRING = 0, 1, 2, 3, 4


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "case_probe", "case_probe.cpp")
    out = os.path.join(HERE, "case_probe", "libcase_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    deps = [src, _lib.LIB_PATH, os.path.join(ROOT, "pinot_b200", "csrc", "pb200_expr.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.cp_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.cp_compile_plain.argtypes = [C.c_char_p]
    lib.cp_is_multi.argtypes = [C.c_char_p]
    lib.cp_is_filter.argtypes = [C.c_char_p]
    lib.cp_eval.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double),
                            C.POINTER(C.c_uint32), C.POINTER(C.c_double)]
    lib.cp_check.argtypes = [C.POINTER(_lib.TransformOp), C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    lib.cp_ids.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_char_p),
                           C.c_int32, C.POINTER(C.c_int32)]
    lib.cp_like.argtypes = [C.c_char_p, C.c_char_p, C.c_int32]
    return lib


def arg(text):
    return sql.parse(f"SELECT SUM({text}) FROM t").aggregations[0].column


# ---- parser ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("text,canonical", [
    ("CASE WHEN status = 'error' THEN bytes ELSE 0 END", "case(equals(status,'error'),bytes,'0')"),
    ("case when dir='in' then bytes else -bytes end", "case(equals(dir,'in'),bytes,times('-1',bytes))"),
    ("CASE WHEN a > 5 THEN a * b WHEN a <= -2.5 THEN 1.5 ELSE c END",
     "case(greater_than(a,'5'),times(a,b),less_than_or_equal(a,'-2.5'),'1.5',c)"),
    ("CASE WHEN 5 < a THEN 1 ELSE 0 END", "case(greater_than(a,'5'),'1','0')"),
    ("CASE WHEN a <> 1 AND (b BETWEEN 1 AND 3 OR NOT c >= 2.0) THEN 1 ELSE 0 END",
     "case(and(not_equals(a,'1'),or(between(b,'1','3'),not(greater_than_or_equal(c,'2')))),'1','0')"),
    ("CASE WHEN s IN ('x', 'it''s') AND t NOT IN (1, 2) THEN 1 ELSE 0 END", "case(and(in(s,'x','it''s'),not_in(t,'1','2')),'1','0')"),
    ("CASE WHEN s NOT LIKE 'a%' OR REGEXP_LIKE(s, '^b') THEN x ELSE 0 END", "case(or(not(like(s,'a%')),regexp_like(s,'^b')),x,'0')"),
    ("CASE WHEN l > 9007199254740993.5 THEN 1 ELSE 0 END", "case(greater_than(l,'9007199254740994.0'),'1','0')"),
])
def test_canonical_text(text, canonical):
    assert arg(text) == canonical


def test_equal_spellings_are_one_aggregation():
    a = arg("CASE WHEN (a = 1) THEN b ELSE 0 END")
    b = arg("case   when a=1.0 then (b) else 0.0 end")
    assert a == b
    q = sql.parse(f"SELECT SUM(CASE WHEN a = 1 THEN b ELSE 0 END), COUNT(CASE WHEN a = 1 THEN b ELSE 0 END) FROM t")
    assert [(g.function, g.column) for g in q.aggregations] == [("SUM", a), ("COUNT", None)]


@pytest.mark.parametrize("text", [
    "SELECT SUM(CASE WHEN a = 1 THEN 1 END) FROM t",                                        # no ELSE
    "SELECT SUM(CASE WHEN a = 1 THEN CASE WHEN b = 1 THEN 1 ELSE 0 END ELSE 0 END) FROM t",  # nested
    "SELECT SUM(CASE a WHEN 1 THEN 1 ELSE 0 END) FROM t",                                   # simple CASE
    "SELECT SUM(CASE WHEN a = b THEN 1 ELSE 0 END) FROM t",                                 # column against column
    "SELECT SUM(CASE WHEN a + 1 > 2 THEN 1 ELSE 0 END) FROM t",                             # expression operand
    "SELECT SUM(CASE WHEN ABS(a) > 2 THEN 1 ELSE 0 END) FROM t",
    "SELECT SUM(CASE WHEN a > 1 THEN 'x' ELSE 0 END) FROM t",                               # string value
    "SELECT DISTINCTCOUNT(CASE WHEN a > 1 THEN 1 ELSE 0 END) FROM t",                       # other functions
    "SELECT SUM(x) FROM t GROUP BY CASE WHEN a = 1 THEN 1 ELSE 0 END",                      # group-by key
    "SELECT SUM(x) FROM t WHERE CASE WHEN a = 1 THEN 1 ELSE 0 END > 0",                     # WHERE operand
    "SELECT COUNT(*) FROM t GROUP BY g HAVING CASE WHEN a = 1 THEN 1 ELSE 0 END > 0",      # HAVING operand
    "SELECT CASE WHEN a = 1 THEN 1 ELSE 0 END FROM t",                                      # selection
    "SELECT DISTINCT CASE WHEN a = 1 THEN 1 ELSE 0 END FROM t",                             # DISTINCT
    "SELECT SUM(x) FROM t GROUP BY g ORDER BY CASE WHEN a = 1 THEN 1 ELSE 0 END",          # order item
    "SELECT SUM(CASE WHEN a = 1 THEN 1 ELSE 0 END * 2) FROM t",                             # not the whole argument
    "SELECT SUM(CASE WHEN s LIKE 'a\\b' THEN 1 ELSE 0 END) FROM t",                         # LIKE escape
])
def test_parser_refusals(text):
    with pytest.raises(sql.SqlError):
        if text.startswith("SELECT DISTINCT"):
            sql.parse_distinct(text)
        elif "GROUP BY" not in text and "SUM(" not in text and "COUNT(" not in text:
            sql.parse_selection(text)
        else:
            sql.parse(text)


def test_case_takes_the_per_row_route(probe):
    one = arg("CASE WHEN a = 1 THEN a ELSE 0 END")
    assert is_multi_column_expression("SUM", one) and is_multi_column_expression("MAX", one)
    assert not is_multi_column_expression("COUNT", one)
    assert probe.cp_is_multi(one.encode()) == 1
    assert probe.cp_is_filter(one.encode()) == 0   # as a filter leaf it would be derived, which refuses it
    assert probe.cp_compile_plain(one.encode()) == E_UNSUPPORTED


# ---- host compiler --------------------------------------------------------------------------------------------------
def compile_case(probe, text):
    buf = C.create_string_buffer(2048)
    nl, nc = C.c_int32(), C.c_int32()
    n = probe.cp_compile(text.encode(), buf, 2048, C.byref(nl), C.byref(nc))
    return n, buf.value.decode(), nl.value, nc.value


def test_host_canonical_text_matches_the_parser(probe):
    for text in ["CASE WHEN a > 5 AND NOT (s IN ('x', 'y') OR s LIKE '%z') THEN a * b WHEN c BETWEEN 1 AND 2 THEN -c ELSE 0.5 END",
                 "CASE WHEN s = 'it''s' THEN 1 ELSE 0 END"]:
        canonical = arg(text)
        n, text2, _, _ = compile_case(probe, canonical)
        assert n > 0 and text2 == canonical
        assert compile_case(probe, canonical.replace(",", " , ").replace("greater_than", "GREATER_THAN"))[1] == canonical


@pytest.mark.parametrize("text,rc", [
    ("case(equals(a,'1'),'1')", E_UNSUPPORTED),                                  # no ELSE
    ("case(equals(a,'1'),case(equals(b,'1'),'1','0'),'0')", E_UNSUPPORTED),      # nested
    ("case(equals(a,b),'1','0')", E_UNSUPPORTED),                                # column against column
    ("case(equals(plus(a,'1'),'2'),'1','0')", E_UNSUPPORTED),                     # expression operand
    ("case(a,'1','0')", E_UNSUPPORTED),                                          # no condition
    ("case(equals(a,'1'),'x','0')", E_UNSUPPORTED),                              # string value
    ("case(equals(a,'1'),year(t),'0')", E_UNSUPPORTED),                          # time function
    ("case(equals(a,'1'),equals(b,'1'),'0')", E_UNSUPPORTED),                    # condition as a value
    ("case(between(a,'1'),'1','0')", E_UNSUPPORTED),
    ("case(and(equals(a,'1')),'1','0')", E_UNSUPPORTED),
    ("case(" + ",".join(f"equals(c{k},'1'),'{k}'" for k in range(8)) + ",x)", E_UNSUPPORTED),   # 9 column leaves
])
def test_host_refusals(probe, text, rc):
    assert compile_case(probe, text)[0] == rc


def test_leaf_counts(probe):
    n, _, nl, nc = compile_case(probe, "case(equals(a,'1'),a,'0')")
    assert (nl, nc) == (1, 1) and n == 4
    assert compile_case(probe, "case(" + ",".join(f"equals(c{k},'1'),'{k}'" for k in range(7)) + ",x)")[2:] == (1, 7)


# ---- the program check on malformed CASE programs -------------------------------------------------------------------
def ops(*items):
    arr = (_lib.TransformOp * len(items))()
    for k, (op, i) in enumerate(items):
        arr[k].op, arr[k].i = op, i
    return arr, len(items)


def test_program_check(probe):
    leaves = C.c_int32()
    T_COND, T_AND, T_OR, T_NOT, T_CASE = _lib.T_COND, _lib.T_AND, _lib.T_OR, _lib.T_NOT, _lib.T_CASE
    good = ops((T_COND, 0), (T_COLUMN, 0), (T_LONG, 0), (T_CASE, 0))
    assert probe.cp_check(*good, 1, C.byref(leaves)) == 0 and leaves.value == 2
    assert probe.cp_check(*good, 0, C.byref(leaves)) == E_INVALID                              # index out of range
    assert probe.cp_check(*ops((T_COND, 1), (T_COLUMN, 0), (T_LONG, 0), (T_CASE, 0)), 1, C.byref(leaves)) == E_INVALID
    assert probe.cp_check(*ops((T_COND, -1), (T_COLUMN, 0), (T_LONG, 0), (T_CASE, 0)), 1, C.byref(leaves)) == E_INVALID
    assert probe.cp_check(*ops((T_COND, 0), (T_COLUMN, 0), (T_CASE, 0)), 1, C.byref(leaves)) == E_INVALID   # underflow
    assert probe.cp_check(*ops((T_COND, 0), (T_AND, 0)), 1, C.byref(leaves)) == E_INVALID                  # underflow
    assert probe.cp_check(*ops((T_COLUMN, 0), (T_COND, 0), (T_LONG, 0), (T_CASE, 0)), 1, C.byref(leaves)) == E_INVALID  # arity order
    assert probe.cp_check(*ops((T_COND, 0), (T_COND, 0), (T_LONG, 0), (T_CASE, 0)), 1, C.byref(leaves)) == E_INVALID    # value is a condition
    assert probe.cp_check(*ops((T_COND, 0), (T_COLUMN, 0), (T_AND, 0)), 1, C.byref(leaves)) == E_INVALID    # AND over a value
    assert probe.cp_check(*ops((T_COND, 0), (T_NOT, 0)), 1, C.byref(leaves)) == E_INVALID                  # a condition result
    assert probe.cp_check(*ops((T_COND, 0), (T_LONG, 1), (T_PLUS, 0)), 1, C.byref(leaves)) == E_INVALID    # arithmetic on a condition
    nested = ops((T_COND, 0), (T_COND, 1), (T_NOT, 0), (T_OR, 0), (T_COLUMN, 0), (T_COND, 2), (T_COLUMN, 1), (T_LONG, 3),
                 (T_CASE, 0), (T_CASE, 0))
    assert probe.cp_check(*nested, 3, C.byref(leaves)) == 0 and leaves.value == 5
    assert probe.cp_check(*ops((99, 0), (T_LONG, 1)), 1, C.byref(leaves)) == E_INVALID


# ---- the evaluator against tests/case_ref.py ------------------------------------------------------------------------
def run_eval(probe, text, rows, cond_words):
    """rows: per row the value leaves in leaf order (ints stay ints: converted by the probe as the device does)."""
    n = len(rows)
    nl = len(rows[0])
    integral = (C.c_int32 * nl)(*[isinstance(v, int) for v in rows[0]])
    ints = (C.c_int64 * (n * nl))(*[v if isinstance(v, int) else 0 for r in rows for v in r])
    dbls = (C.c_double * (n * nl))(*[0.0 if isinstance(v, int) else v for r in rows for v in r])
    cw = (C.c_uint32 * n)(*cond_words)
    out = (C.c_double * n)()
    assert probe.cp_eval(text.encode(), n, nl, integral, ints, dbls, cw, out) == 0
    return list(out)


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))


def leaf_order(text):
    """The value leaves of a CASE text in program order (the order the host compiler numbers them)."""
    tree = case_ref.parse(text)
    out = []

    def walk(t, cond):
        if t[0] == "col":
            if not cond:
                out.append(t[1])
            return
        if t[0] == "lit":
            return
        for k, a in enumerate(t[1]):
            walk(a, cond or (t[0] == "case" and k % 2 == 0 and k + 1 < len(t[1])))
    walk(tree, False)
    return out


def conditions(text):
    tree = case_ref.parse(text)
    out = []

    def walk(t):
        if t[0] in ("and", "or", "not"):
            for a in t[1]:
                walk(a)
        else:
            out.append(t)
    for k in range(0, len(tree[1]) - 1, 2):
        walk(tree[1][k])
    return out


EDGE_LONGS = [INT64_MIN, INT64_MAX, (1 << 53) + 1, -(1 << 53) - 1, 0, 7]
EDGE_DOUBLES = [math.nan, math.inf, -math.inf, -0.0, 0.0, 2.5, 1e308]


@pytest.mark.parametrize("text", [
    "case(greater_than(i,'5'),l,d)",
    "case(equals(s,'x'),times(l,d),less_than(i,'0'),divide(d,i),minus(i,l))",
    "case(and(greater_than(i,'0'),not(equals(s,'y'))),plus(d,'1'),or(less_than(i,'-3'),equals(s,'x')),times('-1',d),'0')",
    "case(greater_than(i,'100'),d,greater_than(i,'0'),l,'-0.5')",   # first WHEN wins when both hold
])
def test_eval_against_reference(probe, text):
    rng = np.random.default_rng(7)
    canonical = compile_case(probe, text)[1]
    names = leaf_order(canonical)
    conds = conditions(canonical)
    rows, words, want = [], [], []
    for r in range(400):
        row = {"i": np.int32(rng.choice([INT_MIN, INT_MAX, -4, 0, 5, 101, 3])), "l": np.int64(rng.choice(EDGE_LONGS)),
               "d": float(rng.choice(EDGE_DOUBLES)), "s": [b"x", b"y", b"z"][r % 3]}
        if r % 5 == 0:
            row["d"] = float(rng.integers(-100, 100)) / 4
        w = 0
        for k, c in enumerate(conds):
            w |= case_ref.holds(c, row) << k
        rows.append([int(row[n]) if n in ("i", "l") else row[n] for n in names])
        words.append(w)
        want.append(case_ref.evaluate(case_ref.parse(canonical), row))
    got = run_eval(probe, canonical, rows, words)
    for k, (g, w) in enumerate(zip(got, want)):
        assert same(g, w), f"row {k}: {g!r} != {w!r} ({rows[k]}, conditions {words[k]:b})"


def test_first_when_wins(probe):
    # both conditions hold: the first value; neither: ELSE; only the second: its value
    got = run_eval(probe, "case(greater_than(a,'0'),'1',greater_than(a,'-5'),'2',a)", [[3], [3], [3], [3]], [0b11, 0b00, 0b10, 0b01])
    assert got == [1.0, 3.0, 2.0, 1.0]


def test_branches_keep_nan_inf_and_negative_zero(probe):
    rows = [[math.nan, -0.0], [math.inf, -0.0], [-math.inf, math.nan]]
    got = run_eval(probe, "case(equals(s,'x'),a,b)", rows, [1, 0, 1])
    assert math.isnan(got[0]) and same(got[1], -0.0) and got[2] == -math.inf


# ---- condition resolution against values ----------------------------------------------------------------------------
def ids(probe, text, typ, values, flags=0):
    card = len(values)
    ints = (C.c_int64 * max(card, 1))(*[int(v) if typ in (INT, LONG) else 0 for v in values])
    dbls = (C.c_double * max(card, 1))(*[float(v) if typ in (FLOAT, DOUBLE) else 0.0 for v in values])
    strs = (C.c_char_p * max(card, 1))(*[v.encode() if typ == STRING else b"" for v in values])
    out = (C.c_int32 * max(card, 1))()
    n = probe.cp_ids(text.encode(), typ, card, ints, dbls, strs, flags, out)
    return n if n < 0 else list(out[:n])


def by_value(text, typ, values):
    """The dictIds whose value satisfies the first condition of `text`, by tests/case_ref.py."""
    cond = conditions(text)[0]
    cast = {INT: np.int32, LONG: np.int64, FLOAT: np.float32, DOUBLE: float, STRING: lambda v: v.encode()}[typ]
    return [k for k, v in enumerate(values) if case_ref.holds(cond, {cond[1][0][1]: cast(v)})]


INTS = [INT_MIN, -7, -3, 0, 2, 3, 10, INT_MAX]
LONGS = [INT64_MIN, -(1 << 53) - 1, -5, 0, 5, (1 << 53), (1 << 53) + 1, INT64_MAX]


@pytest.mark.parametrize("cond", [
    "equals(x,'3')", "equals(x,'2.5')", "not_equals(x,'2.5')", "greater_than(x,'2.5')", "greater_than_or_equal(x,'-3')",
    "less_than(x,'-2.5')", "less_than_or_equal(x,'1e10')", "greater_than(x,'-1e10')", "between(x,'-3.5','3')",
    "in(x,'3','3','2','99')", "not_in(x,'3','-7','0.5')", "greater_than(x,'99999999999999999999')",
])
@pytest.mark.parametrize("typ,values", [(INT, INTS), (LONG, LONGS)])
def test_integral_conditions_resolve_by_exact_value(probe, cond, typ, values):
    text = f"case({cond},'1','0')"
    assert ids(probe, text, typ, values) == by_value(text, typ, values)


def test_long_conditions_at_2_pow_53(probe):
    for cond in ["equals(x,'9007199254740993')", "greater_than(x,'9007199254740992')", "less_than(x,'-9007199254740993')"]:
        text = f"case({cond},'1','0')"
        assert ids(probe, text, LONG, LONGS) == by_value(text, LONG, LONGS)
    assert ids(probe, "case(greater_than(x,'9007199254740994.0'),'1','0')", LONG, LONGS) == E_UNSUPPORTED
    assert ids(probe, "case(greater_than(x,'9007199254740994.0'),'1','0')", DOUBLE, [0.0, 1e16, 2e16]) == [1, 2]


@pytest.mark.parametrize("cond", ["equals(x,'b')", "equals(x,'absent')", "not_equals(x,'absent')", "in(x,'c','a','c','zz')",
                                  "not_in(x,'b','b')", "equals(x,'it''s')"])
def test_string_conditions(probe, cond):
    values = ["a", "b", "c", "it's"]
    text = f"case({cond},'1','0')"
    assert ids(probe, text, STRING, values) == by_value(text, STRING, values)


def test_floating_conditions(probe):
    for typ in (FLOAT, DOUBLE):
        values = [-2.5, 0.0, 0.1, 1.5, 3.0]
        for cond in ["equals(x,'0.1')", "greater_than(x,'0.1')", "between(x,'0','1.5')", "not_in(x,'3','0')"]:
            text = f"case({cond},'1','0')"
            assert ids(probe, text, typ, values) == by_value(text, typ, values)


def test_condition_refusals(probe):
    assert ids(probe, "case(greater_than(x,'1'),'1','0')", DOUBLE, [-1.0, math.nan]) == E_UNSUPPORTED     # NaN
    assert ids(probe, "case(greater_than(x,'1'),'1','0')", FLOAT, [-0.0, 1.0]) == E_UNSUPPORTED           # -0.0
    assert ids(probe, "case(greater_than(x,'b'),'1','0')", STRING, ["a", "c"]) == E_UNSUPPORTED           # STRING range
    assert ids(probe, "case(between(x,'a','b'),'1','0')", STRING, ["a", "c"]) == E_UNSUPPORTED
    assert ids(probe, "case(like(x,'a%'),'1','0')", INT, [1, 2]) == E_UNSUPPORTED                          # pattern on INT
    assert ids(probe, "case(equals(x,'1'),'1','0')", INT, [1, 2], flags=2) == E_UNSUPPORTED                # no dictIds
    assert ids(probe, "case(equals(x,'abc'),'1','0')", INT, [1, 2]) == E_UNSUPPORTED                       # not a number
    assert ids(probe, "case(equals(x,'1'),'1','0')", INT, [1, 2], flags=1) == [0]                          # synthesised


@pytest.mark.parametrize("like", ["a%", "%b", "%c%", "a_c", "%", "", "a.b%", "(x)"])
def test_like_patterns_match_the_sql_front_end(probe, like):
    buf = C.create_string_buffer(256)
    assert probe.cp_like(like.encode(), buf, 256) == 0
    assert buf.value.decode() == sql.like_to_regexp(like)
    assert probe.cp_like(b"a\\b", buf, 256) == -1


def test_result_type_refusal_reaches_no_library_call():
    # the rule needs column types, so the host refuses it; the parser accepts the text
    assert arg("CASE WHEN s = 'x' THEN f ELSE i END") == "case(equals(s,'x'),f,i)"


def test_group_by_refused_across_gpus_before_any_collective():
    from pinot_b200._lib import UnsupportedQueryError
    from pinot_b200.distributed import execute_and_combine

    class NoCollective:
        def __getattr__(self, name):
            raise AssertionError(f"collective {name} issued")
    q = sql.parse("SELECT g, SUM(CASE WHEN a = 1 THEN b ELSE 0 END) FROM t GROUP BY g")
    with pytest.raises(UnsupportedQueryError):
        execute_and_combine(object(), [], q, NoCollective())

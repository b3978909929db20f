"""CPU tests of ORDER BY / SELECT arithmetic over aggregations (post-aggregation expressions): the SQL front end (grammar,
hidden operands, ORDER BY matching, refusals), the library's evaluator (pinot_b200/csrc/pb200_postagg.h, shared by the
device order pass and the host order) compiled with g++ through tests/postagg_probe and held bit for bit to Python floats,
its validation, the marshalled programs, and the expression columns of pinot_b200.cli.final_rows."""
import ctypes as C
import math
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import order_spec, post_spec
from pinot_b200.query import java_divide, post_eval

HERE = os.path.dirname(os.path.abspath(__file__))
INF, NAN = float("inf"), float("nan")


def _q(text, **kw):
    return sql.parse(text, **kw)


# ------------------------------------------------------------------------------------------------ SQL front end
def test_ratio_query_of_the_dashboard_shape():
    q = _q("SELECT campaign, SUM(clicks) / SUM(views) FROM t WHERE day > 3 GROUP BY campaign "
           "ORDER BY SUM(clicks) / SUM(views) DESC LIMIT 10")
    assert [(a.function, a.column, a.hidden) for a in q.aggregations] == [("SUM", "clicks", True), ("SUM", "views", True)]
    assert [(p.text, p.program) for p in q.post_aggregations] == [
        ("divide(sum(clicks),sum(views))", [("AGG", 0), ("AGG", 1), ("DIV",)])]
    assert q.select == [("COLUMN", "campaign"), ("POST", 0)]
    assert sql.resolve_order_by(q) == [("POST", 0, False)]


@pytest.mark.parametrize("expr, program", [
    ("SUM(a) + SUM(b) * 2", [("AGG", 0), ("AGG", 1), ("LIT", 2.0), ("MUL",), ("ADD",)]),
    ("(SUM(a) + SUM(b)) * 2", [("AGG", 0), ("AGG", 1), ("ADD",), ("LIT", 2.0), ("MUL",)]),
    ("SUM(a) - SUM(b) - 1", [("AGG", 0), ("AGG", 1), ("SUB",), ("LIT", 1.0), ("SUB",)]),           # left associative
    ("SUM(a) / SUM(b) / 4", [("AGG", 0), ("AGG", 1), ("DIV",), ("LIT", 4.0), ("DIV",)]),
    ("SUM(a) -1", [("AGG", 0), ("LIT", 1.0), ("SUB",)]),                                            # `-1` is one token
    ("-SUM(a) * SUM(b)", [("AGG", 0), ("NEG",), ("AGG", 1), ("MUL",)]),
    ("- -SUM(a)", [("AGG", 0), ("NEG",), ("NEG",)]),
    ("SUM(a) * -1.5", [("AGG", 0), ("LIT", -1.5), ("MUL",)]),
    ("COUNT(*) * 100.0 / SUM(b)", [("AGG", 2), ("LIT", 100.0), ("MUL",), ("AGG", 1), ("DIV",)]),
    ("((SUM(a)))", [("AGG", 0)]),
])
def test_precedence_and_unary_minus(expr, program):
    q = _q(f"SELECT k, SUM(a), SUM(b), COUNT(*), {expr} FROM t GROUP BY k")
    assert q.post_aggregations[0].program == program
    assert [a.hidden for a in q.aggregations] == [False, False, False]


def test_hidden_operands_are_deduplicated():
    q = _q("SELECT k, SUM(m), SUM(m) / COUNT(*), count(*) * 2 + avg(x), AVG(x) - COUNT(*) FROM t GROUP BY k "
           "HAVING MAX(m) > 1")
    assert [(a.function, a.column, a.hidden) for a in q.aggregations] == [
        ("SUM", "m", False), ("MAX", "m", True), ("COUNT", None, True), ("AVG", "x", True)]
    assert [p.program for p in q.post_aggregations] == [
        [("AGG", 0), ("AGG", 2), ("DIV",)],
        [("AGG", 2), ("LIT", 2.0), ("MUL",), ("AGG", 3), ("ADD",)],
        [("AGG", 3), ("AGG", 2), ("SUB",)]]
    # an operand that a later SELECT item names is that item, not a hidden copy
    q = _q("SELECT k, SUM(a) / SUM(b), SUM(b) FROM t GROUP BY k")
    assert [(a.column, a.hidden) for a in q.aggregations] == [("b", False), ("a", True)]
    assert q.post_aggregations[0].program == [("AGG", 1), ("AGG", 0), ("DIV",)]
    assert q.select == [("COLUMN", "k"), ("POST", 0), ("AGG", 0)]


def test_a_filter_clause_operand_is_its_own_aggregation():
    q = _q("SELECT k, SUM(m) FILTER (WHERE d > 3) / COUNT(*), SUM(m) FROM t GROUP BY k "
           "ORDER BY SUM(m) FILTER (WHERE d > 3) / count(*) DESC")
    assert [(a.function, a.filter is None, a.hidden) for a in q.aggregations] == [
        ("SUM", True, False), ("SUM", False, True), ("COUNT", True, True)]
    assert q.post_aggregations[0].program == [("AGG", 1), ("AGG", 2), ("DIV",)]
    assert sql.resolve_order_by(q) == [("POST", 0, False)]


@pytest.mark.parametrize("order", [
    "sum(A)/Count(*)", "SUM(A) / COUNT( * )", "(SUM(A)) / (COUNT(*))", "((sum(A) / count(*)))",
])
def test_order_by_matches_the_select_item_after_normalisation(order):
    q = _q(f"SELECT k, SUM(A) / COUNT(*) FROM t GROUP BY k ORDER BY {order} DESC, k")
    assert sql.resolve_order_by(q) == [("POST", 0, False), ("GROUP_BY", 0, True)]


def test_expression_items_among_plain_order_items():
    q = _q("SELECT k, SUM(a), SUM(a) * 2, MAX(b) - MIN(b) FROM t GROUP BY k ORDER BY MAX(b) - MIN(b), SUM(a), SUM(a) * 2 DESC")
    assert sql.resolve_order_by(q) == [("POST", 1, True), ("AGG", 0, True), ("POST", 0, False)]
    spec, post = order_spec(q, merge=True), post_spec(q)
    assert [(it.kind, it.index, it.descending) for it in spec.items[:spec.num_items]] == [
        (_lib.ORDER_POST, 0, 0), (_lib.ORDER_AGG, 0, 0), (_lib.ORDER_POST, 1, 1)]
    # only programs named by ORDER BY travel, in the order of their items
    assert post.num_programs == 2
    assert [(n.op, n.agg) for n in post.programs[0].nodes[:post.programs[0].num_nodes]] == [
        (_lib.POST_CODES["AGG"], 1), (_lib.POST_CODES["AGG"], 2), (_lib.POST_CODES["SUB"], 0)]
    assert [(n.op, n.value) for n in post.programs[1].nodes[:post.programs[1].num_nodes]] == [
        (_lib.POST_CODES["AGG"], 0.0), (_lib.POST_CODES["LIT"], 2.0), (_lib.POST_CODES["MUL"], 0.0)]


def test_queries_without_ordered_expressions_send_no_programs():
    assert post_spec(_q("SELECT k, SUM(a) / SUM(b) FROM t GROUP BY k ORDER BY k")) is None
    assert post_spec(_q("SELECT k, SUM(a) FROM t GROUP BY k ORDER BY SUM(a)")) is None
    q = _q("SELECT SUM(a) / COUNT(*) FROM t")   # aggregation only: one row, computed by the caller
    assert post_spec(q) is None and q.select == [("POST", 0)]


def test_sixteen_nodes_are_accepted():
    expr = "-" + " + ".join(["SUM(a)"] * 8)   # 8 operands, NEG, 7 operators
    q = _q(f"SELECT k, {expr} FROM t GROUP BY k ORDER BY {expr}")
    assert len(q.post_aggregations[0].program) == 16
    assert post_spec(q).programs[0].num_nodes == 16
    with pytest.raises(sql.SqlError):
        _q(f"SELECT k, {expr} + 1 FROM t GROUP BY k")


@pytest.mark.parametrize("text", [
    "SELECT k, 1 + 2 FROM t GROUP BY k",                                          # no aggregation
    "SELECT k, SUM(a) FROM t GROUP BY k ORDER BY 2 * 3",
    "SELECT k, SUM(a) / k FROM t GROUP BY k",                                     # a GROUP BY column as an operand
    "SELECT k, SUM(a) + m FROM t GROUP BY k",                                     # a plain column
    "SELECT k, SUM(a) * plus(m, 1) FROM t GROUP BY k",                            # a column expression
    "SELECT k, ABS(SUM(a)) FROM t GROUP BY k",                                    # a function that is not an aggregation
    "SELECT k, ROUND(SUM(a) / COUNT(*), 2) FROM t GROUP BY k",
    "SELECT k, SUM(a) / 'x' FROM t GROUP BY k",                                   # string literal
    "SELECT k, SUM(a) * 1.0e999 FROM t GROUP BY k",                               # non-finite literals
    "SELECT k, SUM(a) * " + "9" * 400 + " FROM t GROUP BY k",
    "SELECT k, SUM(a) / NaN FROM t GROUP BY k",
    "SELECT k, SUM(a) % 2 FROM t GROUP BY k",
    "SELECT k, SUM(a) / COUNT(*) FROM t GROUP BY k ORDER BY SUM(a) * COUNT(*)",  # ORDER BY outside the SELECT list
    "SELECT k, SUM(a) FROM t GROUP BY k ORDER BY SUM(a) / COUNT(*)",
    "SELECT k, LASTWITHTIME(s, ts, 'STRING') + 1 FROM t GROUP BY k",             # a STRING FIRST/LASTWITHTIME operand
    "SELECT k, SUM(a) / COUNT(*) FROM t GROUP BY k HAVING SUM(a) / COUNT(*) > 3",  # HAVING over an expression
])
def test_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


def test_queries_without_expressions_are_unchanged():
    q = _q("SELECT SUM(m), k FROM t GROUP BY k HAVING COUNT(*) > 1 ORDER BY SUM(m) DESC, k LIMIT 5")
    assert q.post_aggregations == [] and post_spec(q) is None
    assert sql.resolve_order_by(q) == [("AGG", 0, False), ("GROUP_BY", 0, True)]
    assert cli.output_columns(q) == [("k", 0), ("sum(m)", 1)]   # keys first, as before


# ------------------------------------------------------------------------------------------------ the evaluator, g++
@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = tmp_path_factory.mktemp("postagg_probe") / "libpostagg_probe.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-o", str(out),
                    os.path.join(HERE, "postagg_probe", "postagg_probe.cpp")], check=True)
    lib = C.CDLL(str(out))
    lib.probe_postagg_validate.argtypes = [C.POINTER(_lib.PostProgram), C.c_int32]
    lib.probe_postagg_eval.argtypes = [C.POINTER(_lib.PostProgram), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int64, C.c_void_p]
    return lib


def _eval(probe, prog, fns, dv, lv, rows):
    """The probe's values of `prog` over `rows` rows (the arrays stay referenced for the call)."""
    fns = np.ascontiguousarray(fns, dtype=np.int32)
    dv = np.ascontiguousarray(dv, dtype=np.float64)
    lv = np.ascontiguousarray(lv, dtype=np.int64)
    out = np.empty(rows, dtype=np.float64)
    probe.probe_postagg_eval(C.byref(prog), len(fns), fns.ctypes.data, dv.ctypes.data, lv.ctypes.data, rows, out.ctypes.data)
    return out


def _program(nodes):
    p = _lib.PostProgram(len(nodes), 0)
    for i, n in enumerate(nodes):
        p.nodes[i] = _lib.PostNode(_lib.POST_CODES[n[0]], n[1] if n[0] == "AGG" else 0, n[1] if n[0] == "LIT" else 0.0)
    return p


def _bits(v):
    return "nan" if math.isnan(v) else struct.pack("<d", v)


FNS = ["COUNT", "SUM", "AVG", "DISTINCTCOUNT", "MIN", "MAX", "VARPOP"]
EDGE = [NAN, -INF, -1e308, -2.5, -0.0, 0.0, 5e-324, 1.0, 3.0, 0.1, 1e308, INF]
COUNTS = [0, 1, 3, 7, (1 << 53) + 1]
LITERALS = [0.0, -0.0, 1.0, -1.0, 2.0, 100.0, 0.1, 1e-300, 1e300, 3.0]


def _final(fn, dv, lv):
    """having_value in Python: COUNT / DISTINCTCOUNT the count, AVG sum / count (-inf at count 0), else the double."""
    if fn in ("COUNT", "DISTINCTCOUNT"):
        return float(lv)
    if fn == "AVG":
        return dv / lv if lv else -INF
    return dv


def _tree(rng, leaves, nagg):
    """Postfix nodes of a random binary tree over `leaves` operands and literals."""
    if leaves == 1:
        return [("AGG", rng.randrange(nagg)) if rng.random() < 0.7 else ("LIT", rng.choice(LITERALS))]
    k = rng.randint(1, leaves - 1)
    return _tree(rng, k, nagg) + _tree(rng, leaves - k, nagg) + [(rng.choice(["ADD", "SUB", "MUL", "DIV"]),)]


def _random_program(rng, nagg):
    """A random well-formed program of at most 16 nodes: up to 8 leaves, their operators and one NEG at a random place
    (after any node there is a value to negate)."""
    nodes = _tree(rng, rng.randint(1, 8), nagg)
    if rng.random() < 0.5:
        nodes.insert(rng.randrange(len(nodes)) + 1, ("NEG",))
    return nodes


def test_evaluator_matches_python_floats_bit_for_bit(probe):
    rng = random.Random(7)
    nagg = len(FNS)
    rows = 400
    fns = np.array([_lib.AGG_CODES[f] for f in FNS], dtype=np.int32)
    dv = np.array([[rng.choice(EDGE) for _ in FNS] for _ in range(rows)], dtype=np.float64)
    lv = np.array([[rng.choice(COUNTS) for _ in FNS] for _ in range(rows)], dtype=np.int64)
    dv[0, :], lv[0, :] = 0.0, 0                 # 0 / 0, AVG of an empty group
    dv[1, :], lv[1, :] = -0.0, 1
    for _ in range(300):
        nodes = _random_program(rng, nagg)
        prog = _program(nodes)
        assert probe.probe_postagg_validate(C.byref(prog), nagg) == 0, nodes
        out = _eval(probe, prog, fns, dv, lv, rows)
        for r in range(rows):
            want = post_eval(nodes, lambda a: _final(FNS[a], float(dv[r, a]), int(lv[r, a])))
            assert _bits(float(out[r])) == _bits(want), (nodes, r)


@pytest.mark.parametrize("x, y, want", [
    (1.0, 0.0, INF), (-1.0, 0.0, -INF), (1.0, -0.0, -INF), (-1.0, -0.0, INF), (0.0, 0.0, NAN), (-0.0, 0.0, NAN),
    (NAN, 0.0, NAN), (INF, 0.0, INF), (INF, -0.0, -INF), (INF, INF, NAN), (1e308, 1e-308, INF), (3.0, 2.0, 1.5),
    (-0.0, 5.0, -0.0), (0.0, -5.0, -0.0), (1.0, INF, 0.0), (-1.0, INF, -0.0),
])
def test_division_is_javas(probe, x, y, want):
    assert _bits(java_divide(x, y)) == _bits(want)
    prog = _program([("AGG", 0), ("AGG", 1), ("DIV",)])
    out = _eval(probe, prog, [_lib.AGG_CODES["SUM"]] * 2, [x, y], [0, 0], 1)
    assert _bits(float(out[0])) == _bits(want)


def test_operators_are_not_contracted(probe):
    """a * b + c rounds the product first: an FMA would give the exactly rounded 2^-104 here, the IEEE steps give 0."""
    a = 1.0 + 2.0 ** -52
    prog = _program([("AGG", 0), ("AGG", 0), ("MUL",), ("LIT", -(1.0 + 2.0 ** -51)), ("ADD",)])
    out = _eval(probe, prog, [_lib.AGG_CODES["SUM"]], [a], [0], 1)
    assert out[0] == a * a - (1.0 + 2.0 ** -51) == 0.0


@pytest.mark.parametrize("nodes, nagg", [
    ([], 2),                                                          # no node
    ([("AGG", 2)], 2),                                                # aggregation out of range
    ([("AGG", -1)], 2),
    ([("LIT", INF)], 2),                                              # non-finite literals
    ([("LIT", -INF)], 2),
    ([("LIT", NAN)], 2),
    ([("AGG", 0), ("AGG", 1)], 2),                                    # two values left
    ([("AGG", 0), ("ADD",)], 2),                                      # operator without its operands
    ([("NEG",), ("AGG", 0)], 2),
    ([("AGG", 0), ("AGG", 1), ("DIV",), ("MUL",)], 2),
    ([("ADD",)], 2),
])
def test_malformed_programs_are_refused(probe, nodes, nagg):
    prog = _program(nodes)
    assert probe.probe_postagg_validate(C.byref(prog), nagg) == 1


def test_node_count_outside_1_to_16_is_refused(probe):
    prog = _program([("AGG", 0)] * 8 + [("ADD",)] * 7 + [("NEG",)])
    assert probe.probe_postagg_validate(C.byref(prog), 1) == 0
    for n in (17, 0, -1):
        prog.num_nodes = n
        assert probe.probe_postagg_validate(C.byref(prog), 1) == 1


def test_unknown_op_is_refused(probe):
    prog = _program([("AGG", 0)])
    prog.nodes[0].op = 7
    assert probe.probe_postagg_validate(C.byref(prog), 1) == 1
    prog.nodes[0].op = -1
    assert probe.probe_postagg_validate(C.byref(prog), 1) == 1


def test_sixteen_node_program_is_valid(probe):
    prog = _program([("AGG", 0)] * 8 + [("MUL",)] * 7 + [("NEG",)])
    assert probe.probe_postagg_validate(C.byref(prog), 1) == 0
    out = _eval(probe, prog, [_lib.AGG_CODES["COUNT"]], [0.0], [3], 1)
    assert out[0] == -(3.0 ** 8)


# ------------------------------------------------------------------------------------------------ cli.final_rows
TABLE = {  # key values: [COUNT, SUM(m), AVG(m) (sum, count), SUM(n)]
    ("a", 1): [4, 10.0, (10.0, 4), 2.0],
    ("b", 1): [3, -6.0, (-6.0, 3), 0.0],
    ("a", 2): [1, 0.0, (0.0, 1), 0.0],
    ("c", 0): [2, -0.0, (-0.0, 2), 5.0],
    ("b", 0): [5, NAN, (NAN, 5), 1.0],
    ("d", 3): [6, 12.0, (12.0, 6), -0.0],
}


def test_final_rows_print_select_order_with_expression_columns():
    q = _q("SELECT SUM(m) / SUM(n), k, COUNT(*) * 100.0 / SUM(n), s FROM t GROUP BY s, k "
           "ORDER BY SUM(m) / SUM(n) DESC LIMIT 10")
    assert [str(a) for a in q.aggregations] == ["sum(m)", "sum(n)", "count(*)"]
    table = {k: [v[1], v[3], v[0]] for k, v in TABLE.items()}
    rows = cli.final_rows(q, table)
    assert [name for name, _ in cli.output_columns(q)] == [
        "divide(sum(m),sum(n))", "k", "divide(times(count(*),'100'),sum(n))", "s"]
    # DESC in Double.compare order: NaN first (NaN / 1), +inf (-6 / 0 is -inf, 10 / 2 = 5, -0.0 / 5 = -0.0,
    # 0 / 0 = NaN, 12 / -0.0 = -inf); equal values (the two NaNs, the two -infs) by key ascending
    assert [(r[3], r[1]) for r in rows] == [("a", 2), ("b", 0), ("a", 1), ("c", 0), ("b", 1), ("d", 3)]
    got = {(r[3], r[1]): (r[0], r[2]) for r in rows}
    assert _bits(got[("a", 1)][0]) == _bits(5.0) and got[("a", 1)][1] == 200.0
    assert _bits(got[("c", 0)][0]) == _bits(-0.0) and got[("c", 0)][1] == 40.0
    assert got[("b", 1)][0] == -INF and got[("b", 1)][1] == INF         # 300 / 0.0
    assert got[("d", 3)][0] == -INF and got[("d", 3)][1] == -INF        # 600 / -0.0
    assert math.isnan(got[("a", 2)][0]) and got[("a", 2)][1] == INF


def test_final_rows_expression_ascending_with_having_and_limit():
    q = _q("SELECT s, k, SUM(m) / COUNT(*), AVG(m) FROM t GROUP BY s, k HAVING COUNT(*) > 1 ORDER BY SUM(m) / COUNT(*) LIMIT 3")
    assert [(str(a), a.hidden) for a in q.aggregations] == [("avg(m)", False), ("count(*)", True), ("sum(m)", True)]
    table = {k: [v[2], v[0], v[1]] for k, v in TABLE.items()}
    rows = cli.final_rows(q, table)
    # ("a", 2) has COUNT 1 and is filtered; ascending: -2.0, -0.0, 2.0 (then 2.5, NaN)
    assert rows == [["b", 1, -2.0, -2.0], ["c", 0, -0.0, -0.0], ["d", 3, 2.0, 2.0]]
    assert math.copysign(1.0, rows[1][2]) == -1.0


def test_final_rows_expression_equals_avg_order():
    """ORDER BY SUM(m) / COUNT(*) gives AVG(m)'s rows in AVG(m)'s order (one division of the same two numbers)."""
    for direction in ("", " DESC"):
        a = cli.final_rows(_q(f"SELECT s, k, SUM(m) / COUNT(*) FROM t GROUP BY s, k ORDER BY SUM(m) / COUNT(*){direction}"),
                           {k: [v[1], v[0]] for k, v in TABLE.items()})
        b = cli.final_rows(_q(f"SELECT s, k, AVG(m) FROM t GROUP BY s, k ORDER BY AVG(m){direction}"),
                           {k: [v[2]] for k, v in TABLE.items()})
        assert [(r[0], r[1]) for r in a] == [(r[0], r[1]) for r in b]
        assert [_bits(r[2]) for r in a] == [_bits(r[2]) for r in b]


def test_final_rows_aggregation_only():
    q = _q("SELECT COUNT(*), SUM(m) * 2 - 1 FROM t")
    assert cli.final_rows(q, {(): [4, 10.0]}) == [[4, 19.0]]
    assert [name for name, _ in cli.output_columns(q)] == ["count(*)", "minus(times(sum(m),'2'),'1')"]

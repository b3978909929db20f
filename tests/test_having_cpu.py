"""CPU tests of HAVING: the SQL front end (leaves, hidden aggregations, refusals), the library's predicate
(pinot_b200/csrc/pb200_having.h, shared by the device keep kernel and the host filter) compiled with g++ through
tests/having_probe and checked against a Python reference, and the broker-side filter of pinot_b200.cli.final_rows."""
import ctypes as C
import itertools
import math
import os
import subprocess

import numpy as np
import pytest

from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import having_spec
from pinot_b200.query import Filter

HERE = os.path.dirname(os.path.abspath(__file__))
INF, NAN = float("inf"), float("nan")


def _q(text, **kw):
    return sql.parse(text, **kw)


# ------------------------------------------------------------------------------------------------ SQL front end
def test_having_leaves_in_canonical_form():
    q = _q("SELECT k, SUM(m), COUNT(*) FROM t GROUP BY k HAVING count(*) > 10 AND SUM(m) BETWEEN -1.5 AND 2 "
           "AND NOT (sum(m) <= 0 OR COUNT(*) IN (3, 4)) AND SUM(m) NOT IN (7) AND COUNT(*) <> 5")
    assert [a.hidden for a in q.aggregations] == [False, False]
    assert sql.resolve_having(q) == [
        ("RANGE", 1, 10.0, None, False, True),
        ("RANGE", 0, -1.5, 2.0, True, True),
        ("RANGE", 0, None, 0.0, True, True), ("EQ", 1, 3.0), ("EQ", 1, 4.0), ("OR", 2), ("OR", 2), ("NOT",),
        ("NEQ", 0, 7.0),
        ("NEQ", 1, 5.0),
        ("AND", 5)]


def test_hidden_aggregations_are_added_once_and_orderable():
    q = _q("SELECT k, SUM(m) FROM t GROUP BY k HAVING AVG(m) > 1 AND (MAX(m) < 9 OR AVG(m) < 0) AND PERCENTILE95(x) >= 2 "
           "AND percentile(x, 95) < 5 AND VAR_POP(m) > 0 ORDER BY avg(m) DESC, k LIMIT 3")
    assert [(a.function, a.column, a.arg, a.hidden) for a in q.aggregations] == [
        ("SUM", "m", None, False), ("AVG", "m", None, True), ("MAX", "m", None, True), ("PERCENTILE", "x", 95.0, True),
        ("VARPOP", "m", None, True)]
    assert sql.resolve_order_by(q) == [("AGG", 1, False), ("GROUP_BY", 0, True)]
    assert {n[1] for n in sql.resolve_having(q) if n[0] in ("RANGE", "EQ", "NEQ")} == {1, 2, 3, 4}


def test_having_uses_the_unfiltered_aggregation():
    q = _q("SELECT k, SUM(m) FILTER (WHERE x > 1) FROM t GROUP BY k HAVING SUM(m) > 3")
    assert [(a.function, a.filter is None, a.hidden) for a in q.aggregations] == [("SUM", False, False), ("SUM", True, True)]
    assert sql.resolve_having(q) == [("RANGE", 1, 3.0, None, False, True)]


def test_query_without_having_is_unchanged():
    q = _q("SELECT k, SUM(m) FROM t GROUP BY k ORDER BY SUM(m) LIMIT 5")
    assert q.having is None and sql.resolve_having(q) == [] and having_spec(q) is None


@pytest.mark.parametrize("text", [
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING k > 3",                        # group-by column
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING m > 3",                        # plain column
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING m + 1 > 3",                    # expression of columns
    "SELECT SUM(m) FROM t HAVING SUM(m) > 3",                                 # no GROUP BY
    "SELECT SUM(m) FROM t WHERE m > 1 HAVING COUNT(*) > 3",
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING SUM(m) > 'abc'",               # string literals
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING COUNT(*) IN (1, '2')",
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING SUM(m) BETWEEN '1' AND 2",
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING 3 < SUM(m)",                   # literal on the left
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING 'x' = SUM(m)",
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING SUM(m) / COUNT(*) > 3",        # expression over aggregations
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING SUM(m) > 1 ORDER BY MAX(m)",   # ORDER BY still needs a named aggregation
    "SELECT k, SUM(m) FROM t GROUP BY k HAVING COUNT(*) IN (" + ", ".join(map(str, range(32))) + ")",  # 33 nodes
])
def test_having_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


def test_32_nodes_are_accepted():
    q = _q("SELECT k, SUM(m) FROM t GROUP BY k HAVING COUNT(*) IN (" + ", ".join(map(str, range(31))) + ")")
    assert len(sql.resolve_having(q)) == 32
    assert having_spec(q).num_nodes == 32


# ------------------------------------------------------------------------------------------------ the predicate, g++
@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = tmp_path_factory.mktemp("having_probe") / "libhaving_probe.so"
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", str(out),
                    os.path.join(HERE, "having_probe", "having_probe.cpp")], check=True)
    lib = C.CDLL(str(out))
    lib.probe_having_validate.argtypes = [C.POINTER(_lib.Having), C.c_int32]
    lib.probe_having_eval.argtypes = [C.POINTER(_lib.Having), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.c_void_p]
    return lib


FNS = ["COUNT", "SUM", "AVG", "DISTINCTCOUNT", "MIN", "MAX", "PERCENTILE", "VARPOP", "VARSAMP", "STDDEVPOP", "STDDEVSAMP"]
SELECT = ("SELECT k, COUNT(*), SUM(m), AVG(m), DISTINCTCOUNT(m), MIN(m), MAX(m), PERCENTILE(m, 50), VAR_POP(m), "
          "VAR_SAMP(m), STDDEV_POP(m), STDDEV_SAMP(m) FROM t GROUP BY k HAVING ")
NAMES = ["COUNT(*)", "SUM(m)", "AVG(m)", "DISTINCTCOUNT(m)", "MIN(m)", "MAX(m)", "PERCENTILE(m, 50)", "VAR_POP(m)",
         "VAR_SAMP(m)", "STDDEV_POP(m)", "STDDEV_SAMP(m)"]
EDGE = [NAN, -INF, -1e308, -2.5, -0.0, 0.0, 5e-324, 1.0, 2.5, 3.0, 1e308, INF]
COUNTS = [0, 1, 2, 3, 5, (1 << 53) + 1]


def _rows():
    """(double column, long column) per aggregation and row: every edge value in every double-valued function, every
    count in the count-valued ones, AVG pairs with count 0 and with NaN / inf sums."""
    rows = []
    for i, (x, c) in enumerate(itertools.product(EDGE, COUNTS)):
        dv, lv = [], []
        for a, fn in enumerate(FNS):
            if fn in ("COUNT", "DISTINCTCOUNT"):
                dv.append(float(c)); lv.append(c)
            elif fn == "AVG":
                dv.append(x); lv.append(c)
            else:
                dv.append(EDGE[(EDGE.index(x) + a) % len(EDGE)] if not math.isnan(x) else x); lv.append(c)
        rows.append((dv, lv))
    return rows


def _final(fn, dv, lv):
    if fn in ("COUNT", "DISTINCTCOUNT"):
        return float(lv)
    if fn == "AVG":
        return dv / lv if lv else -INF
    return dv


def _ref(node, vals):
    """The reference: the SQL tree itself, with Python's float comparisons (Java's: NaN only !=, -0.0 == 0.0)."""
    if isinstance(node, Filter):
        outs = [_ref(c, vals) for c in node.children]
        return all(outs) if node.type == "AND" else any(outs) if node.type == "OR" else not outs[0]
    v = vals[[sql.having_name(a) for a in HAVING_AGGS].index(node.column)]
    lits = [float(x) for x in node.values]
    if node.type == "EQ":
        return v == lits[0]
    if node.type == "NEQ":
        return v != lits[0]
    if node.type == "IN":
        return any(v == x for x in lits)
    if node.type == "NOT_IN":
        return all(v != x for x in lits)
    lo_ok = node.lower is None or (v >= float(node.lower) if node.lower_inclusive else v > float(node.lower))
    hi_ok = node.upper is None or (v <= float(node.upper) if node.upper_inclusive else v < float(node.upper))
    return lo_ok and hi_ok


HAVING_AGGS = _q(SELECT + "COUNT(*) > 0").aggregations

CONDITIONS = [f"{n} {op} {lit}" for n in NAMES for op, lit in
              (("=", "0"), ("=", "-0.0"), ("!=", "0"), ("<>", "2.5"), ("<", "2.5"), ("<=", "-0.0"), (">", "0.0"), (">=", "3"),
               ("<", "1.0e400"), (">", "-2.5"), ("=", "1.0e400"))] + [
    "COUNT(*) > 2.5", "COUNT(*) < 2.5", "COUNT(*) = 2.5", "DISTINCTCOUNT(m) >= 0.5", "COUNT(*) = 9007199254740993",
    "AVG(m) BETWEEN -2.5 AND 2.5", "SUM(m) BETWEEN -2.5 AND 1.0e400", "MIN(m) IN (-0.0, 1, 2.5)",
    "MAX(m) NOT IN (0, 3)", "PERCENTILE(m, 50) NOT IN (1.0e400)",
    "NOT SUM(m) > 0", "NOT (SUM(m) = 0 OR AVG(m) < 0)", "COUNT(*) > 1 AND SUM(m) < 0 OR NOT AVG(m) >= 1",
    "(VAR_POP(m) > 0 OR VAR_SAMP(m) <= 0) AND (STDDEV_POP(m) != 0 OR NOT STDDEV_SAMP(m) < 1)",
    "NOT NOT (COUNT(*) > 1 AND (SUM(m) > 0 OR (AVG(m) < 1 AND NOT MAX(m) = 1.0e400)))",
]


def _spec(q):
    s = having_spec(q)
    # the spec indexes q.aggregations; the probe's columns follow FNS, which is the SELECT list's order
    assert [a.function for a in q.aggregations] == FNS
    return s


@pytest.mark.parametrize("cond", CONDITIONS)
def test_predicate_matches_the_reference(probe, cond):
    q = _q(SELECT + cond)
    spec = _spec(q)
    assert probe.probe_having_validate(C.byref(spec), len(FNS)) == 0
    rows = _rows()
    dv = np.array([r[0] for r in rows], dtype=np.float64)
    lv = np.array([r[1] for r in rows], dtype=np.int64)
    fns = np.array([_lib.AGG_CODES[f] for f in FNS], dtype=np.int32)
    out = np.zeros(len(rows), dtype=np.uint8)
    probe.probe_having_eval(C.byref(spec), len(FNS), fns.ctypes.data, dv.ctypes.data, lv.ctypes.data, len(rows), out.ctypes.data)
    want = [_ref(q.having, [_final(f, d, l) for f, d, l in zip(FNS, r[0], r[1])]) for r in rows]
    assert out.tolist() == [int(w) for w in want], cond


def test_nan_matches_only_not_equal(probe):
    fns = np.array([_lib.AGG_CODES[f] for f in FNS], dtype=np.int32)
    dv = np.full((1, len(FNS)), NAN)
    lv = np.ones((1, len(FNS)), dtype=np.int64)
    out = np.zeros(1, dtype=np.uint8)
    for cond, want in (("SUM(m) = 0", 0), ("SUM(m) != 0", 1), ("SUM(m) < 0", 0), ("SUM(m) >= 0", 0),
                       ("SUM(m) BETWEEN -2.5 AND 1.0e400", 0), ("SUM(m) IN (1, 2)", 0), ("SUM(m) NOT IN (1, 2)", 1),
                       ("NOT SUM(m) > 0", 1), ("AVG(m) > -2.5", 0), ("AVG(m) <> 1", 1)):
        spec = having_spec(_q(SELECT + cond))
        probe.probe_having_eval(C.byref(spec), len(FNS), fns.ctypes.data, dv.ctypes.data, lv.ctypes.data, 1, out.ctypes.data)
        assert out[0] == want, cond


def _tree(*nodes):
    h = _lib.Having(len(nodes), 0)
    for i, n in enumerate(nodes):
        h.nodes[i] = _lib.HavingNode(*n)
    return h


R, EQ, NEQ, AND, OR, NOT = (_lib.HAVING_CODES[k] for k in ("RANGE", "EQ", "NEQ", "AND", "OR", "NOT"))


@pytest.mark.parametrize("nodes", [
    [],                                                           # empty
    [(EQ, 0, 0, 0, 1.0, 0.0), (EQ, 0, 0, 0, 2.0, 0.0)],           # two roots
    [(AND, 0, 0, 0, 0.0, 0.0)],                                   # AND without operands
    [(EQ, 0, 0, 0, 1.0, 0.0), (AND, 2, 0, 0, 0.0, 0.0)],          # AND with too few
    [(NOT, 1, 0, 0, 0.0, 0.0)],                                   # NOT without operand
    [(EQ, 0, 3, 0, 1.0, 0.0)],                                    # aggregation out of range
    [(EQ, 0, -1, 0, 1.0, 0.0)],
    [(EQ, 0, 0, 0, NAN, 0.0)],                                    # NaN bounds
    [(NEQ, 0, 0, 0, NAN, 0.0)],
    [(R, 0, 0, 2, NAN, 0.0)],
    [(R, 0, 0, 1, 0.0, NAN)],
    [(R, 0, 0, 3, 0.0, 0.0)],                                     # RANGE without a bound
    [(R, 0, 0, 16, 0.0, 1.0)],                                    # unknown flag
    [(9, 0, 0, 0, 0.0, 0.0)],                                     # unknown node type
])
def test_malformed_trees_are_refused(probe, nodes):
    h = _lib.Having(len(nodes), 0)
    for i, n in enumerate(nodes):
        h.nodes[i] = _lib.HavingNode(*n)
    assert probe.probe_having_validate(C.byref(h), 3) == 1


def test_infinite_bounds(probe):
    """SQL has no literal for -inf; the C ABI takes one.  inf bounds compare as usual: -inf < -inf is false."""
    fns = np.array([_lib.AGG_CODES["MIN"]], dtype=np.int32)
    dv = np.array([-INF, -1e308, INF, NAN])
    lv = np.zeros(4, dtype=np.int64)
    for nodes, want in (([(R, 0, 0, 2 | 4, -INF, 0.0)], [0, 1, 1, 0]),     # v > -inf
                        ([(R, 0, 0, 2, -INF, 0.0)], [1, 1, 1, 0]),         # v >= -inf
                        ([(R, 0, 0, 1 | 8, 0.0, INF)], [1, 1, 0, 0]),      # v < inf
                        ([(EQ, 0, 0, 0, -INF, 0.0)], [1, 0, 0, 0]),
                        ([(NEQ, 0, 0, 0, INF, 0.0)], [1, 1, 0, 1])):
        h = _tree(*nodes)
        assert probe.probe_having_validate(C.byref(h), 1) == 0
        out = np.zeros(4, dtype=np.uint8)
        probe.probe_having_eval(C.byref(h), 1, fns.ctypes.data, dv.ctypes.data, lv.ctypes.data, 4, out.ctypes.data)
        assert out.tolist() == want, nodes


def test_node_limit(probe):
    h = _lib.Having(33, 0)
    assert probe.probe_having_validate(C.byref(h), 3) == 1
    # 32 nodes: 16 leaves, 15 binary ANDs, one NOT -- the deepest stack the limit allows is evaluated too
    nodes = [(R, 0, 0, 2, float(i), 0.0) for i in range(16)] + [(AND, 2, 0, 0, 0.0, 0.0)] * 15 + [(NOT, 1, 0, 0, 0.0, 0.0)]
    h = _tree(*nodes)
    assert probe.probe_having_validate(C.byref(h), 1) == 0
    fns = np.array([_lib.AGG_CODES["SUM"]], dtype=np.int32)
    out = np.zeros(3, dtype=np.uint8)
    dv, lv = np.array([15.0, 14.5, NAN]), np.zeros(3, dtype=np.int64)
    probe.probe_having_eval(C.byref(h), 1, fns.ctypes.data, dv.ctypes.data, lv.ctypes.data, 3, out.ctypes.data)
    assert out.tolist() == [0, 1, 1]   # NOT (v >= 0 AND ... AND v >= 15)
    wide = _tree(*([(EQ, 0, 0, 0, float(i), 0.0) for i in range(31)] + [(OR, 31, 0, 0, 0.0, 0.0)]))
    assert probe.probe_having_validate(C.byref(wide), 1) == 0
    dv = np.array([0.0, 30.0, 31.0, -0.0])
    out = np.zeros(4, dtype=np.uint8)
    probe.probe_having_eval(C.byref(wide), 1, fns.ctypes.data, dv.ctypes.data, np.zeros(4, dtype=np.int64).ctypes.data, 4,
                            out.ctypes.data)
    assert out.tolist() == [1, 1, 0, 1]


# ------------------------------------------------------------------------------------------------ cli.final_rows
TABLE = {  # key values: [COUNT, SUM, AVG (sum, count), DISTINCTCOUNT set, MIN]
    ("a", 1): [3, 10.0, (10.0, 3), {1, 2}, -0.0],
    ("b", 1): [3, -5.0, (-5.0, 3), {1}, 0.0],
    ("a", 2): [1, NAN, (10.0, 1), {1, 2, 3}, 2.0],
    ("c", 0): [7, 0.0, (0.0, 0), set(), INF],
    ("b", 0): [4, 10.0, (9.0, 3), {4, 5}, -INF],
}
BASE = "SELECT COUNT(*), SUM(m), AVG(m), DISTINCTCOUNT(d), MIN(m) FROM t GROUP BY s, k"


def _keys(rows):
    return [tuple(r[:2]) for r in rows]


@pytest.mark.parametrize("having, want", [
    ("COUNT(*) > 2.5", [("a", 1), ("b", 0), ("b", 1), ("c", 0)]),
    ("SUM(m) = 10", [("a", 1), ("b", 0)]),
    ("SUM(m) != 10", [("a", 2), ("b", 1), ("c", 0)]),                    # NaN passes !=
    ("SUM(m) < 100", [("a", 1), ("b", 0), ("b", 1), ("c", 0)]),          # ... and nothing else
    ("MIN(m) = 0", [("a", 1), ("b", 1)]),                                # -0.0 == 0.0
    ("MIN(m) < -1.5", [("b", 0)]),
    ("AVG(m) > 3 OR DISTINCTCOUNT(d) IN (0, 1)", [("a", 1), ("a", 2), ("b", 1), ("c", 0)]),   # empty AVG is -inf
    ("NOT (COUNT(*) BETWEEN 3 AND 4)", [("a", 2), ("c", 0)]),
    ("COUNT(*) > 100", []),
])
def test_final_rows_with_having(having, want):
    rows = cli.final_rows(_q(BASE + " HAVING " + having + " LIMIT 10"), TABLE)
    assert _keys(rows) == want


def test_final_rows_having_then_order_then_limit_and_hidden_columns():
    table = {k: v[:2] + [v[2]] for k, v in TABLE.items()}   # COUNT, SUM, AVG
    q = _q("SELECT s, k, SUM(m) FROM t GROUP BY s, k HAVING COUNT(*) >= 3 AND AVG(m) > -10 ORDER BY AVG(m) DESC LIMIT 2")
    assert [a.hidden for a in q.aggregations] == [False, True, True]
    table = {k: [v[1], v[0], v[2]] for k, v in table.items()}   # the query's aggregation order: SUM, COUNT, AVG
    rows = cli.final_rows(q, table)
    # ('c', 0) has AVG -inf (count 0): filtered by AVG > -10; LIMIT 2 applies after HAVING
    assert rows == [["a", 1, 10.0], ["b", 0, 10.0]]

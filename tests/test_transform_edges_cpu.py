"""CPU: predicates on derived (transform) columns at NaN, -0.0, 0.0 and +-inf, against tests/float_edges_ref.py.

The reference has no dictionary for an arithmetic expression: ExpressionFilterOperator evaluates the expression per row
and compares each DOUBLE value with Java's <, > and == (the raw-value predicate evaluators).  So a predicate on a DOUBLE
derived column selects the rows float_edges_ref.raw_matches selects: NaN matches only NEQ / NOT_IN, and 0 (or '-0.0')
matches both zeros.  The derived column's dictionary is the product's device-built one, sorted in Double.compare order
with one canonical NaN last.

* DOUBLE derived columns: the device leaf (pb200h::leaf_to_device) and pb200h::matching_dict_ids select exactly the
  rows of the value comparisons, and the leaf folds to EMPTY / MATCH_ALL exactly when those rows are none / all.
* INT / LONG derived columns: exact integral comparisons, as before.
* Stored DOUBLE dictionaries keep the oracle's doc set (the reference's binary search of the dictionary, whose `<` / `>`
  call a NaN entry equal to any literal and -0.0 equal to 0.0): tests/test_float_edges_cpu.py pins that parity, and here
  the same column marked derived answers by value instead."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import float_edges_ref as fr
import transform_ref
from oracle import segment_builder as sb
from pinot_b200 import _lib
from pinot_b200.plan_maker import _marshal_query
from pinot_b200.query import Aggregation, Predicate, QueryContext
from test_host_logic_cpu import F_EMPTY, F_MATCH_ALL, F_SCAN_IN, F_SCAN_NOT_IN, F_SCAN_RANGE, _leaf_docs, probe  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

DMAX = 1.7976931348623157e308
NAN = fr.double_of(fr.D_NAN)

# dictionaries in Double.compare order, as the derivation kernel builds them (one canonical NaN, last)
FULL = [-math.inf, -DMAX, -1e308, -1.5, -1.0, -5e-324, -0.0, 0.0, 5e-324, 0.75, 1.5, 1e308, DMAX, math.inf, NAN]
DICTIONARIES = {
    "full": FULL,
    "nan": [NAN],
    "zeros": [-0.0, 0.0],
    "neg_zero": [-0.0],
    "zero_nan": [0.0, NAN],
    "infs_nan": [-math.inf, math.inf, NAN],
    "finite": [-1.5, 0.75, 1.5],
}


@pytest.fixture(scope="module")
def derived_probe(probe):  # noqa: F811  (probe builds the library first)
    src = os.path.join(HERE, "derived_probe", "derived_probe.cpp")
    out = os.path.join(HERE, "derived_probe", "libderived_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.probe_derived_leaf.restype = C.c_int64
    lib.probe_derived_leaf.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                       C.POINTER(_lib.HFilterNode), C.POINTER(_lib.HLiteral), C.c_void_p, C.c_void_p, C.c_int64]
    return lib


def predicates(column, extra=()):
    """EQ / NEQ / IN / NOT_IN over the literals, and RANGE over pairs of them and unbounded sides, with every
    inclusive / exclusive combination."""
    lits = [0, -0.0, 1.5, -1.5, 1e308, -1e308] + list(extra)
    out = []
    for v in lits:
        out += [Predicate("EQ", column, [v]), Predicate("NEQ", column, [v])]
    for vs in ([0], [-0.0], [-0.0, 1.5], [1e308, -1.5], [-1e308, 0, 1.5], [5]):
        out += [Predicate("IN", column, vs), Predicate("NOT_IN", column, vs)]
    bounds = [None, 0, -0.0, 1.5, -1.5, 1e308, -1e308]
    for lo in bounds:
        for hi in bounds:
            if lo is None and hi is None:
                continue
            for li in (True, False):
                for ui in (True, False):
                    if (lo is None and not li) or (hi is None and not ui):
                        continue   # an unbounded side has no inclusiveness
                    out.append(Predicate("RANGE", column, [], lo, hi, li, ui))
    return out


def dict_bytes(entries, data_type):
    np_type = {sb.INT: np.int32, sb.LONG: np.int64, sb.DOUBLE: np.float64}[data_type]
    return np.frombuffer(np.array(entries, dtype=np_type).astype(sb._NP_BE[data_type]).tobytes(), dtype=np.uint8).copy()


def rows_over(card, n, seed):
    """Dictionary ids of n rows: every id at least once, the rest drawn at random."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, card, size=n).astype(np.int64)
    ids[:card] = np.arange(card)
    return ids


def resolve(derived_probe, data_type, derived, synthesized, dict_be, card, n, p):
    """(leaf op, rows the leaf selects, rows matching_dict_ids selects) for `p`, given the rows' dictionary ids."""
    hq, _keep = _marshal_query(QueryContext([Aggregation("COUNT", None)], filter=p), False)
    out4 = np.zeros(4, dtype=np.int32)
    buf = np.zeros(2 * card + 8, dtype=np.int32)

    def call(leaf):
        m = derived_probe.probe_derived_leaf(data_type, int(derived), int(synthesized), dict_be.ctypes.data, card, n, leaf,
                                             hq.filter, hq.literals, out4.ctypes.data, buf.ctypes.data, len(buf))
        assert m >= 0, (p, m)
        return buf[:m].copy()

    leaf_ids = call(1)
    op, lo, hi = int(out4[0]), int(out4[2]), int(out4[3])
    return op, lo, hi, leaf_ids, call(0)


def check_by_value(derived_probe, entries, n, seed, what):
    """A DOUBLE derived column over `entries`: every predicate selects the rows of the value comparisons."""
    dict_be = dict_bytes(entries, sb.DOUBLE)
    card = len(entries)
    ids = rows_over(card, n, seed)
    values = np.array(entries, dtype=np.float64)[ids]
    for p in predicates("e", extra=[5, 0.75, -5e-324]):
        want = np.array([i for i, v in enumerate(values) if fr.raw_matches(v, p, sb.DOUBLE)], dtype=np.int64)
        op, lo, hi, leaf_ids, matching = resolve(derived_probe, sb.DOUBLE, True, False, dict_be, card, n, p)
        got = _leaf_docs(op, lo, hi, leaf_ids, ids, n)
        assert np.array_equal(got, want), (what, p, op, len(got), len(want))
        assert np.array_equal(np.nonzero(np.isin(ids, matching))[0], want), (what, p, "matching_dict_ids")
        # constant folding: every entry has rows, so the leaf is EMPTY / MATCH_ALL exactly when no / every row matches
        assert (op == F_EMPTY) == (len(want) == 0), (what, p, op)
        assert (op == F_MATCH_ALL) == (len(want) == n), (what, p, op)
        if op not in (F_EMPTY, F_MATCH_ALL):   # an unsorted column without an inverted index: a scan
            assert op == (F_SCAN_RANGE if p.type == "RANGE" else F_SCAN_NOT_IN if p.type in ("NEQ", "NOT_IN") else F_SCAN_IN), (what, p, op)


@pytest.mark.parametrize("name", sorted(DICTIONARIES))
def test_double_derived_predicates_compare_values(derived_probe, name):
    check_by_value(derived_probe, DICTIONARIES[name], 700, 11, name)


# (expression, INT source values, predicate): results with NaN, both zeros and both infinities
ISSUE_CASES = [
    ("mod(i,'0')", list(range(-3, 4)), Predicate("EQ", "e", [5])),
    ("mod(i,'0')", list(range(-3, 4)), Predicate("NEQ", "e", [5])),
    ("ceil(divide(i,'7'))", list(range(-13, 14)), Predicate("EQ", "e", [0])),
    ("ceil(divide(i,'7'))", list(range(-13, 14)), Predicate("EQ", "e", [-0.0])),
    ("times(i,'-1')", list(range(-5, 6)), Predicate("RANGE", "e", [], 0, None, True, True)),
    ("times(i,'-1')", list(range(-5, 6)), Predicate("RANGE", "e", [], None, 0, True, False)),
    ("divide(i,'0')", list(range(-4, 5)), Predicate("RANGE", "e", [], -1e308, None, False, True)),
    ("divide(i,'0')", list(range(-4, 5)), Predicate("NOT_IN", "e", [0, 1.5])),
    ("divide('1',i)", list(range(-4, 5)), Predicate("RANGE", "e", [], None, 1e308, True, True)),
    ("mod(i,'3')", list(range(-7, 8)), Predicate("IN", "e", [0])),
]


@pytest.mark.parametrize("expr,source,p", ISSUE_CASES, ids=[f"{e} {p.type}" for e, _, p in ISSUE_CASES])
def test_expression_predicates_over_transform_ref_values(derived_probe, expr, source, p):
    """Expressions over INT values whose results include NaN, -0.0 and +-inf: the derived dictionary is the sorted unique
    results (transform_ref, Double.compare order), the rows those of each source value, and the rows selected are the
    rows whose value compares true."""
    per_value = transform_ref.column(expr, np.array(source, dtype=np.int64), "INT")
    entries = fr.unique_values(per_value, sb.DOUBLE)
    index = {fr.identity(v): k for k, v in enumerate(entries)}
    ids = np.array([index[fr.identity(v)] for v in per_value] * 3, dtype=np.int64)
    values = np.concatenate([per_value] * 3)
    n = len(ids)
    want = np.array([i for i, v in enumerate(values) if fr.raw_matches(v, p, sb.DOUBLE)], dtype=np.int64)
    op, lo, hi, leaf_ids, _ = resolve(derived_probe, sb.DOUBLE, True, False, dict_bytes(entries, sb.DOUBLE), len(entries), n, p)
    assert np.array_equal(_leaf_docs(op, lo, hi, leaf_ids, ids, n), want), (expr, p, op)
    assert (op == F_EMPTY) == (len(want) == 0) and (op == F_MATCH_ALL) == (len(want) == n), (expr, p, op)


def test_the_nan_dictionary_folds_by_value(derived_probe):
    """mod(i, 0) is NaN for every row: `= 5` is EMPTY and `!= 5` MATCH_ALL, whereas the dictionary search (which calls a
    NaN entry equal to any literal) would fold them the other way round."""
    be = dict_bytes([NAN], sb.DOUBLE)
    for p, want in ((Predicate("EQ", "e", [5]), F_EMPTY), (Predicate("NEQ", "e", [5]), F_MATCH_ALL),
                    (Predicate("IN", "e", [0, -0.0]), F_EMPTY), (Predicate("NOT_IN", "e", [0]), F_MATCH_ALL),
                    (Predicate("RANGE", "e", [], None, 0, True, True), F_EMPTY),
                    (Predicate("RANGE", "e", [], -1e308, None, True, True), F_EMPTY)):
        assert resolve(derived_probe, sb.DOUBLE, True, False, be, 1, 4, p)[0] == want, p
        # the same dictionary stored by a segment keeps the reference's search: `= 5` lands on NaN
        if p.type == "EQ":
            assert resolve(derived_probe, sb.DOUBLE, False, False, be, 1, 4, p)[0] == F_MATCH_ALL


def _int_matches(x: int, p) -> bool:
    """An integral value against a predicate by exact numeric value (Python compares int with float exactly)."""
    if p.type == "RANGE":
        if p.lower is not None and not (x >= p.lower if p.lower_inclusive else x > p.lower):
            return False
        return p.upper is None or (x <= p.upper if p.upper_inclusive else x < p.upper)
    hit = any(x == v for v in p.values)
    return hit if p.type in ("EQ", "IN") else not hit


@pytest.mark.parametrize("data_type", [sb.INT, sb.LONG])
def test_integral_derived_predicates_are_exact(derived_probe, data_type):
    """INT / LONG derived columns (calendar fields, DATETRUNC, ...) keep their exact integral comparisons, fractional
    and out-of-range literals included."""
    big = 2 ** 31 - 1 if data_type == sb.INT else 2 ** 63 - 1
    entries = sorted({-big - 1, -(2 ** 20), -7, -1, 0, 1, 2, 7, 2 ** 20, big} | ({2 ** 53 + 1, -(2 ** 53) - 1} if data_type == sb.LONG else set()))
    dict_be = dict_bytes(entries, data_type)
    ids = rows_over(len(entries), 400, 5)
    values = [entries[i] for i in ids]
    for p in predicates("e", extra=[7, -7, 0.5, -0.5, 2.5, 1e19, -1e19, 2 ** 20, 2 ** 53 + 1]):
        want = np.array([i for i, v in enumerate(values) if _int_matches(v, p)], dtype=np.int64)
        for derived in (True, False):
            op, lo, hi, leaf_ids, _ = resolve(derived_probe, data_type, derived, False, dict_be, len(entries), len(ids), p)
            assert np.array_equal(_leaf_docs(op, lo, hi, leaf_ids, ids, len(ids)), want), (data_type, derived, p)


def test_stored_double_dictionary_keeps_the_reference_search(oracle, derived_probe):
    """The same DOUBLE dictionary stored by a segment (neither derived nor synthesised): the oracle's doc set, the
    reference's search quirk included; marked derived, the value comparisons.  The two differ on this dictionary."""
    entries = FULL
    ids = rows_over(len(entries), 600, 3)
    values = np.array(entries, dtype=np.float64)[ids]
    col = fr.build_dict_column("e", values)
    seg = sb.SegmentData("stored", len(values), [col])
    assert [fr.identity(v) for v in col.dict_values] == [fr.identity(v) for v in entries]
    differ = 0
    for p in predicates("e", extra=[5]):
        q = QueryContext([Aggregation("COUNT", None)], filter=p)
        op, lo, hi, leaf_ids, _ = resolve(derived_probe, sb.DOUBLE, False, False, col.dict, col.cardinality, len(values), p)
        stored = _leaf_docs(op, lo, hi, leaf_ids, col.dict_ids, len(values))
        assert np.array_equal(stored, fr.doc_ids(oracle, seg, q)), p
        op, lo, hi, leaf_ids, _ = resolve(derived_probe, sb.DOUBLE, True, False, col.dict, col.cardinality, len(values), p)
        by_value = _leaf_docs(op, lo, hi, leaf_ids, col.dict_ids, len(values))
        assert np.array_equal(by_value, [i for i, v in enumerate(values) if fr.raw_matches(v, p, sb.DOUBLE)]), p
        differ += not np.array_equal(stored, by_value)
    assert differ > 0

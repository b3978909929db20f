"""Value-space reference of the filter: which docs of a segment a filter tree matches, computed from the stored values.

It reads every doc's value straight from the segment's columns (exact_ref.column_values) and compares it with the
predicate's literal exactly, in the column's own type; it never calls the oracle's filter and never looks at dictIds:

* INT / LONG: Python integers, a float literal by its exact value (Fraction): `x = 2.5` matches nothing, `x >= 2.5` is
  `x >= 3`, a literal beyond the column's range makes the comparison constant.  This is what the reference's broker
  (NumericalFilterOptimizer) rewrites such predicates to before a server sees them.
* FLOAT: np.float32 against (float)literal; DOUBLE: float.
* STRING: unpadded UTF-8 bytes, ordered bytewise.

NaN and -0.0 are out of scope (see exact_ref)."""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

from exact_ref import column_values
from oracle import segment_builder as sb
from pinot_b200.query import Filter, Predicate

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _exact(v) -> Fraction:
    return Fraction(int(v)) if isinstance(v, (int, np.integer)) else Fraction(float(v))


def _at_least(x: np.ndarray, k: int) -> np.ndarray:
    """x >= k for int64 x and any Python integer k."""
    if k > INT64_MAX:
        return np.zeros(len(x), dtype=bool)
    return x >= np.int64(max(k, INT64_MIN))


def _at_most(x: np.ndarray, k: int) -> np.ndarray:
    if k < INT64_MIN:
        return np.zeros(len(x), dtype=bool)
    return x <= np.int64(min(k, INT64_MAX))


def _integral_leaf(x: np.ndarray, p: Predicate) -> np.ndarray:
    if p.type == "RANGE":
        m = np.ones(len(x), dtype=bool)
        if p.lower is not None:
            lo = _exact(p.lower)
            m &= _at_least(x, math.ceil(lo) if p.lower_inclusive else math.floor(lo) + 1)
        if p.upper is not None:
            hi = _exact(p.upper)
            m &= _at_most(x, math.floor(hi) if p.upper_inclusive else math.ceil(hi) - 1)
        return m
    hit = np.zeros(len(x), dtype=bool)
    for v in p.values:
        e = _exact(v)
        if e.denominator == 1 and INT64_MIN <= e.numerator <= INT64_MAX:
            hit |= x == np.int64(e.numerator)
    return hit if p.type in ("EQ", "IN") else ~hit


def _ordered_leaf(x: np.ndarray, p: Predicate, lit) -> np.ndarray:
    """FLOAT / DOUBLE / STRING: plain comparisons of x with lit(literal)."""
    if p.type == "RANGE":
        m = np.ones(len(x), dtype=bool)
        if p.lower is not None:
            lo = lit(p.lower)
            m &= (x >= lo) if p.lower_inclusive else (x > lo)
        if p.upper is not None:
            hi = lit(p.upper)
            m &= (x <= hi) if p.upper_inclusive else (x < hi)
        return m
    hit = np.zeros(len(x), dtype=bool)
    for v in p.values:
        hit |= x == lit(v)
    return hit if p.type in ("EQ", "IN") else ~hit


class _Values:
    """Every doc's stored value per column, read once."""

    def __init__(self, oracle, seg: sb.SegmentData):
        self.oracle, self.seg, self.cache = oracle, seg, {}

    def __call__(self, column: str):
        if column not in self.cache:
            c = self.seg.column(column)
            x = column_values(self.oracle, self.seg, column, np.arange(self.seg.num_docs))
            if c.data_type in (sb.INT, sb.LONG):
                x = x.astype(np.int64)
            elif c.data_type == sb.FLOAT:
                x = x.astype(np.float32)
            elif c.data_type == sb.DOUBLE:
                x = x.astype(np.float64)
            self.cache[column] = (c.data_type, x)
        return self.cache[column]


def _leaf(values: _Values, p: Predicate) -> np.ndarray:
    dt, x = values(p.column)
    if dt in (sb.INT, sb.LONG):
        return _integral_leaf(x, p)
    if dt == sb.FLOAT:
        return _ordered_leaf(x, p, lambda v: np.float32(float(v)))
    if dt == sb.DOUBLE:
        return _ordered_leaf(x, p, float)
    return _ordered_leaf(x, p, lambda v: v.encode("utf-8") if isinstance(v, str) else bytes(v))


def _evaluate(values: _Values, node, n: int) -> np.ndarray:
    if node is None:
        return np.ones(n, dtype=bool)
    if isinstance(node, Predicate):
        return _leaf(values, node)
    assert isinstance(node, Filter), node
    kids = [_evaluate(values, c, n) for c in node.children]
    if node.type == "NOT":
        assert len(kids) == 1
        return ~kids[0]
    out = kids[0].copy()
    for k in kids[1:]:
        if node.type == "AND":
            out &= k
        else:
            out |= k
    return out


def matching_docs(oracle, seg: sb.SegmentData, node) -> np.ndarray:
    """bool[num_docs]: the docs of `seg` the filter tree `node` (a QueryContext.filter, None = all) matches."""
    return _evaluate(_Values(oracle, seg), node, seg.num_docs)


def matching_docs_many(oracle, seg: sb.SegmentData, nodes) -> list:
    """matching_docs of several trees over one segment, reading each column once."""
    values = _Values(oracle, seg)
    return [_evaluate(values, t, seg.num_docs) for t in nodes]

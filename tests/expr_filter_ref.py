"""Value-space reference of filters with leaves on expressions over two or more columns (DESIGN.md section 3.16).

tests/filter_ref.py decides every ordinary leaf.  A leaf whose column is an expression with two or more distinct columns
is decided per row the way the reference's ExpressionFilterOperator does: the expression evaluated as a DOUBLE by
tests/expr_ref.evaluate on the stored values, then compared by tests/float_edges_ref.raw_matches.  Nothing here looks at
the product."""
from __future__ import annotations

import numpy as np

import filter_ref
from exact_ref import column_values
from expr_ref import columns, evaluate, parse
from float_edges_ref import raw_matches
from oracle import segment_builder as sb
from pinot_b200.query import Filter, Predicate


def is_expression(column: str) -> bool:
    return bool(column) and "(" in column and len(set(columns(parse(column)))) >= 2


_VALUES = {}


def expression_values(oracle, seg: sb.SegmentData, text: str) -> list:
    """The expression's DOUBLE value at every doc of `seg` (kept per segment object and text)."""
    key = (id(seg), seg.name, text)
    if key not in _VALUES:
        tree = parse(text)
        cols = sorted(set(columns(tree)))
        docs = np.arange(seg.num_docs)
        vals = {c: column_values(oracle, seg, c, docs) for c in cols}
        _VALUES[key] = [evaluate(tree, {c: vals[c][i] for c in cols}) for i in range(seg.num_docs)]
    return _VALUES[key]


def matching_docs(oracle, seg: sb.SegmentData, node) -> np.ndarray:
    """bool[num_docs]: the docs of `seg` the filter tree `node` matches (None = all)."""
    values = filter_ref._Values(oracle, seg)

    def walk(n):
        if n is None:
            return np.ones(seg.num_docs, dtype=bool)
        if isinstance(n, Predicate):
            if is_expression(n.column):
                xs = expression_values(oracle, seg, n.column)
                return np.array([raw_matches(x, n, sb.DOUBLE) for x in xs], dtype=bool).reshape(seg.num_docs)
            return filter_ref._leaf(values, n)
        assert isinstance(n, Filter), n
        kids = [walk(c) for c in n.children]
        if n.type == "NOT":
            return ~kids[0]
        out = kids[0].copy()
        for k in kids[1:]:
            out = (out & k) if n.type == "AND" else (out | k)
        return out
    return walk(node)

"""Per-row reference of aggregations over CASE WHEN (DESIGN.md section 3.19), in Python values.

A CASE text `case(c1,v1,...,e)` is evaluated on each matched row: the first condition that holds picks its value, else
the ELSE value.  A condition compares the row's stored value with its literals by value: INT / LONG exactly (the literal
as a Fraction of its text), FLOAT as (float) value against (float) literal, DOUBLE as doubles, STRING as strings; LIKE
through sql.like_to_regexp and REGEXP_LIKE with re.search.  Values are tests/expr_ref.py's arithmetic.  The doc set comes
from tests/filter_ref.py and the values from exact_ref.column_values; nothing here looks at the product."""
from __future__ import annotations

import re
from fractions import Fraction
from typing import Dict, List, Sequence

import numpy as np

import expr_ref
from exact_ref import column_values
from filter_ref import matching_docs
from pinot_b200.sql import like_to_regexp

_TOKEN = re.compile(r"'(?:[^']|'')*'|[A-Za-z_$][\w$.]*|[-+]?[0-9.][0-9.]*(?:[eE][+-]?[0-9]+)?|\S")


def parse(text: str):
    """CASE text -> ("case", [cond, value, ..., else]); conditions ("and" | "or" | "not", [kids]) or (fn, column,
    [literal texts]); values expr_ref trees."""
    toks = _TOKEN.findall(text)
    pos = 0

    def node():
        nonlocal pos
        t = toks[pos]
        pos += 1
        if t.startswith("'"):
            return ("lit", t[1:-1].replace("''", "'"))
        if t[0].isdigit() or t[0] in "+-.":
            return ("lit", t)
        if pos < len(toks) and toks[pos] == "(":
            pos += 1
            args = []
            while toks[pos] != ")":
                args.append(node())
                if toks[pos] == ",":
                    pos += 1
            pos += 1
            return (t, args)
        return ("col", t)

    tree = node()
    assert pos == len(toks) and tree[0] == "case", text
    return tree


def _value_tree(t):
    """A branch value as an expr_ref tree (literals as floats)."""
    if t[0] == "lit":
        return ("lit", float(t[1]))
    if t[0] == "col":
        return t
    return (t[0], [_value_tree(a) for a in t[1]])


def _compare(v, lit: str):
    """-1, 0, 1: the stored value v against the literal text, by the column's type (numpy dtype of v)."""
    if isinstance(v, (bytes, str)):
        s = v.decode("utf-8") if isinstance(v, bytes) else v
        return (s > lit) - (s < lit)
    if isinstance(v, (np.integer, int)):
        a, b = Fraction(int(v)), Fraction(lit)
    elif isinstance(v, np.float32):
        a, b = np.float32(v), np.float32(float(lit))
    else:
        a, b = float(v), float(lit)
    return int(a > b) - int(a < b)


def holds(c, row) -> bool:
    fn, args = c
    if fn in ("and", "or", "not"):
        kids = [holds(a, row) for a in args]
        return all(kids) if fn == "and" else any(kids) if fn == "or" else not kids[0]
    v = row[args[0][1]]
    lits = [a[1] for a in args[1:]]
    if fn in ("like", "regexp_like"):
        s = v.decode("utf-8") if isinstance(v, bytes) else v
        return re.search(like_to_regexp(lits[0]) if fn == "like" else lits[0], s) is not None
    cmp = [_compare(v, x) for x in lits]
    return {"equals": lambda: cmp[0] == 0, "not_equals": lambda: cmp[0] != 0, "less_than": lambda: cmp[0] < 0,
            "less_than_or_equal": lambda: cmp[0] <= 0, "greater_than": lambda: cmp[0] > 0,
            "greater_than_or_equal": lambda: cmp[0] >= 0, "between": lambda: cmp[0] >= 0 and cmp[1] <= 0,
            "in": lambda: 0 in cmp, "not_in": lambda: 0 not in cmp}[fn]()


def columns(tree) -> List[str]:
    if tree[0] == "col":
        return [tree[1]]
    if tree[0] == "lit":
        return []
    return [c for a in tree[1] for c in columns(a)]


def evaluate(tree, row) -> float:
    args = tree[1]
    for k in range(0, len(args) - 1, 2):
        if holds(args[k], row):
            return expr_ref.evaluate(_value_tree(args[k + 1]), row)
    return expr_ref.evaluate(_value_tree(args[-1]), row)


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def row_values(oracle, segs: Sequence, flt, group_by: Sequence[str], text: str) -> Dict[tuple, List[float]]:
    """{group key values: the CASE's value on every matched row of the group} (aggregation only: the key ())."""
    tree = parse(text)
    cols = sorted(set(columns(tree)))
    out: Dict[tuple, List[float]] = {} if group_by else {(): []}
    for seg in segs:
        docs = np.nonzero(matching_docs(oracle, seg, flt))[0]
        if not len(docs):
            continue
        vals = {c: column_values(oracle, seg, c, docs) for c in cols}
        keys = [column_values(oracle, seg, g, docs) for g in group_by]
        for i in range(len(docs)):
            out.setdefault(tuple(_py(k[i]) for k in keys), []).append(evaluate(tree, {c: vals[c][i] for c in cols}))
    return out

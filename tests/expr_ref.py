"""Per-row reference of aggregations over multi-column expressions (DESIGN.md section 3.15).

An expression is evaluated on each matched row with Python floats: each leaf value converted with float() (an int64
beyond 2^53 rounds to nearest), +, -, *, / one IEEE-754 step each (x / 0: +-inf, 0 / 0 and NaN / 0: NaN), MOD math.fmod
(NaN where C's fmod is NaN), FLOOR / CEIL keeping the sign of a zero, ABS math.fabs.  The doc set comes from
tests/filter_ref.py and the values from exact_ref.column_values; nothing here looks at the product.

Checks: SUM / AVG within gamma_n * sum|x| of the exact sum of the row values (NaN when a row is NaN or both infinities
occur, otherwise the infinity that occurs, an exact zero as +0.0); MIN / MAX bit for bit in Double.compare order."""
from __future__ import annotations

import math
import re
import struct
from fractions import Fraction
from typing import Dict, List, Sequence

import numpy as np

from exact_ref import column_values, gamma, same_double
from filter_ref import matching_docs

_TOKEN = re.compile(r"'(?:[^']|'')*'|[A-Za-z_$][\w$.]*|[-+]?[0-9.][0-9.]*(?:[eE][+-]?[0-9]+)?|\S")
_ALIASES = {"add": "plus", "sub": "minus", "mult": "times", "div": "divide"}


def parse(text: str):
    """Expression text -> tree: ("col", name) | ("lit", float) | (function, [args])."""
    toks = _TOKEN.findall(text)
    pos = 0

    def node():
        nonlocal pos
        t = toks[pos]
        pos += 1
        if t.startswith("'"):
            return ("lit", float(t[1:-1].replace("''", "'")))
        if t[0].isdigit() or t[0] in "+-.":
            return ("lit", float(t))
        if pos < len(toks) and toks[pos] == "(":
            pos += 1
            name = t.lower().replace("_", "")
            args = []
            while toks[pos] != ")":
                args.append(node())
                if toks[pos] == ",":
                    pos += 1
            pos += 1
            return (_ALIASES.get(name, name), args)
        return ("col", t)
    tree = node()
    assert pos == len(toks), text
    return tree


def columns(tree) -> List[str]:
    if tree[0] == "col":
        return [tree[1]]
    if tree[0] == "lit":
        return []
    return [c for a in tree[1] for c in columns(a)]


def _div(x: float, y: float) -> float:
    if y != 0 or math.isnan(y):
        return x / y if not math.isnan(y) else math.nan
    if math.isnan(x) or x == 0:
        return math.nan
    return math.copysign(math.inf, x) * math.copysign(1.0, y)


def _fmod(x: float, y: float) -> float:
    if math.isnan(x) or math.isnan(y) or math.isinf(x) or y == 0:
        return math.nan
    return math.fmod(x, y)


def _round(f, x: float) -> float:
    if not math.isfinite(x):
        return x
    r = float(f(x))
    return math.copysign(0.0, x) if r == 0 else r


_OPS = {"plus": lambda x, y: x + y, "minus": lambda x, y: x - y, "times": lambda x, y: x * y, "divide": _div, "mod": _fmod,
        "floor": lambda x: _round(math.floor, x), "ceil": lambda x: _round(math.ceil, x), "abs": math.fabs}


def evaluate(tree, row: Dict[str, object]) -> float:
    """The expression on one row: row maps a column name to its stored value."""
    if tree[0] == "col":
        v = row[tree[1]]
        return float(v.item() if hasattr(v, "item") else v)
    if tree[0] == "lit":
        return tree[1]
    return _OPS[tree[0]](*[evaluate(a, row) for a in tree[1]])


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def row_values(oracle, segs: Sequence, flt, group_by: Sequence[str], text: str) -> Dict[tuple, List[float]]:
    """{group key values: the expression's value on every matched row of the group} (aggregation only: the key ())."""
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
            key = tuple(_py(k[i]) for k in keys)
            out.setdefault(key, []).append(evaluate(tree, {c: vals[c][i] for c in cols}))
    return out


def order_key(x: float) -> int:
    """Double.compare order as an unsigned key (every NaN one value after +inf)."""
    u = struct.unpack("<Q", struct.pack("<d", math.nan if math.isnan(x) else x))[0]
    return (~u & (2 ** 64 - 1)) if u >> 63 else u | (1 << 63)


def check_sum(got: float, xs: List[float]) -> bool:
    """The SUM contract over the row values xs."""
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return math.isnan(got)
    if math.inf in xs or -math.inf in xs:
        return got == (math.inf if math.inf in xs else -math.inf)
    s = sum(Fraction(x) for x in xs)
    if s == 0 and all(x == 0 for x in xs):
        return same_double(got, 0.0)
    if not math.isfinite(got):
        return False
    a = sum(Fraction(abs(x)) for x in xs)
    return abs(Fraction(got) - s) <= gamma(max(len(xs), 1)) * a


def check_value(fn: str, got_double: float, got_long: int, xs: List[float]) -> bool:
    """One aggregation of one group: its double (and for SUM / AVG its count) against the row values."""
    if fn in ("SUM", "AVG"):
        return check_sum(got_double, xs) and (fn == "SUM" or got_long == len(xs))
    if not xs:
        return same_double(got_double, math.inf if fn == "MIN" else -math.inf)
    want = (min if fn == "MIN" else max)(xs, key=order_key)
    return order_key(got_double) == order_key(want)

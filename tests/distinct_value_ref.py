"""Exact reference of DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG from stored values: the distinct values of a group
(integers exactly, floats by identity: -0.0 and 0.0 apart, one NaN), summed as Fractions and rounded once.  DISTINCTSUM
of no value is 0.0, DISTINCTAVG -inf.  The values come from tests/percentile_ref.group_values; nothing here comes from the
product."""
import math
from fractions import Fraction

from pinot_b200.query import value_key


def distinct_values(values):
    """The distinct stored values: integers exactly, floats by identity (ValueKey: -0.0 and 0.0 apart, one NaN)."""
    return {value_key(v) for v in (x.item() if hasattr(x, "item") else x for x in values)}


def ref_final(fn, values):
    """The exact reference: the distinct stored values summed as Fractions, rounded once."""
    s = distinct_values(values)
    if fn == "DISTINCTCOUNT":
        return float(len(s))
    if not s:
        return 0.0 if fn == "DISTINCTSUM" else -math.inf
    total = sum((Fraction(v) for v in s), Fraction(0))
    return float(total / len(s) if fn == "DISTINCTAVG" else total)

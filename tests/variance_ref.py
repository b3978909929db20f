"""Exact reference of VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP from stored values.

The values come from tests/percentile_ref.group_values (the doc set of tests/filter_ref.py, the column's stored values at
those docs, grouped by the group-by columns' values).  Every sum is a Fraction, so M2 = sum (v - mean)^2 is exact; the
variance is rounded once to double, and STDDEV is the correctly rounded sqrt of that double.  The final-value rules of
VarianceAggregationFunction are restated here: n == 0, and *SAMP with n == 1, give -inf.  Nothing here comes from the
product."""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Sequence

import numpy as np

FUNCTIONS = ("VARPOP", "VARSAMP", "STDDEVPOP", "STDDEVSAMP")


def exact_sums(values: np.ndarray):
    """(n, sum v, sum v^2) of the stored values, exact."""
    if values.dtype.kind in "iu":
        ints = [int(x) for x in values]
        return len(ints), Fraction(sum(ints)), Fraction(sum(x * x for x in ints))
    fr = [Fraction(float(x)) for x in values]
    return len(fr), sum(fr, Fraction(0)), sum((x * x for x in fr), Fraction(0))


def exact_variance(function: str, sums) -> Fraction:
    n, s1, s2 = sums
    m2 = s2 - s1 * s1 / n
    return m2 / (n - 1 if function in ("VARSAMP", "STDDEVSAMP") else n)


def final(function: str, sums) -> float:
    n = sums[0]
    if n == 0 or (function in ("VARSAMP", "STDDEVSAMP") and n == 1):
        return float("-inf")
    var = float(exact_variance(function, sums))
    return math.sqrt(var) if function.startswith("STDDEV") else var


def within_one_ulp(got: float, function: str, sums) -> bool:
    """The variance within 1 ulp of the exact rational; STDDEV the correctly rounded sqrt of a variance within 1 ulp."""
    want = final(function, sums)
    if math.isinf(want) or math.isinf(got):
        return got == want
    exact = exact_variance(function, sums)
    var = float(exact)
    if function.startswith("VAR"):
        return abs(Fraction(got) - exact) <= Fraction(math.ulp(var))
    candidates = (math.nextafter(var, -math.inf), var, math.nextafter(var, math.inf))
    return any(v >= 0 and abs(Fraction(v) - exact) <= Fraction(math.ulp(var)) and got == math.sqrt(v) for v in candidates)


def merge(parts: Sequence[tuple]) -> tuple:
    n, s1, s2 = 0, Fraction(0), Fraction(0)
    for a, b, c in parts:
        n, s1, s2 = n + a, s1 + b, s2 + c
    return n, s1, s2

"""CPU checks of tests/exact_ref.py, the exact COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT reference the -m gpu tests
hold the device to."""
import math
from fractions import Fraction

import numpy as np

from exact_ref import ExactSum, U, _exact_int_sums, assert_exact, check_sum, gamma, reference, same_double, sum_within_bound
from pinot_b200 import sql
from reduce_util import normalise

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1


def test_exact_sums_of_a_hand_made_table(oracle):
    k = np.array([0, 1, 0, 1, 2, 2, 0, 1], dtype=np.int32)
    v = np.array([INT_MAX, INT_MIN, INT_MAX, -1, 5, 6, INT_MAX, INT_MIN], dtype=np.int32)
    w = np.array([1, 1, 1, 1, 0, 1, 1, 1], dtype=np.int32)
    lv = np.array([1 << 62, -(1 << 62), 3, -3, (1 << 63) - 1, -(1 << 63), 7, 1], dtype=np.int64)
    d = np.array([1e15, 1.0, -1e15, 0.5, 2.0, -2.0, 0.25, 3.0], dtype=np.float64)
    seg = oracle.build_segment("hand", {"k": k, "v": v, "w": w, "lv": lv, "d": d, "rv": v.copy()}, raw=["rv"])
    q = sql.parse("SELECT SUM(v), COUNT(*), AVG(v), SUM(lv), SUM(d), SUM(rv), SUM(v) FILTER(WHERE v < 0) FROM t "
                  "WHERE w = 1 GROUP BY k")
    ref = reference(oracle, [seg], q)
    assert set(ref) == {(0,), (1,), (2,)}
    g0, g1, g2 = ref[(0,)], ref[(1,)], ref[(2,)]
    assert g0[0] == ExactSum("int", 3 * INT_MAX, None, 3) and g0[1] == 3 and g0[2].n == 3
    assert g1[0].s == 2 * INT_MIN - 1 and g1[1] == 3
    assert g2[0].s == 6 and g2[1] == 1              # row 4 (w = 0) is filtered out
    assert g0[3].s == (1 << 62) + 3 + 7 and g0[3].a == (1 << 62) + 10
    assert g2[3].s == -(1 << 63) and g2[3].a == 1 << 63   # |INT64_MIN| does not wrap
    assert g0[4].s == 0.25 and g0[4].a == 2e15 + 0.25      # cancellation: S exact, A keeps the magnitude
    assert g0[5] == g0[0] and g1[5] == g1[0]                # raw INT column: same values
    assert g0[6] == ExactSum("int", 0, None, 0) and g1[6] == ExactSum("int", 2 * INT_MIN - 1, None, 3)
    # merged: the union of the segments' rows, by value
    seg2 = oracle.build_segment("hand2", {"k": k + 1, "v": v, "w": w, "lv": lv, "d": d, "rv": v.copy()}, raw=["rv"])
    both = reference(oracle, [seg, seg2], q)
    assert set(both) == {(0,), (1,), (2,), (3,)}
    assert both[(1,)][0].s == 2 * INT_MIN - 1 + 3 * INT_MAX and both[(1,)][1] == 6
    # aggregation only, nothing matches: one row of zeros
    empty = reference(oracle, [seg], sql.parse("SELECT SUM(v), COUNT(*) FROM t WHERE w > 5"))
    assert empty == {(): [ExactSum("int", 0, None, 0), 0]}


def test_comparator_int_sums_are_bit_exact():
    q = sql.parse("SELECT SUM(v), AVG(v), COUNT(*) FROM t")
    s = (1 << 53) + 1                        # float(s) rounds to 2^53 (ties to even)
    ref = {(): [ExactSum("int", s, None, 4), ExactSum("int", s, None, 4), 4]}
    assert_exact(q, {(): [float(1 << 53), (float(1 << 53), 4), 4]}, ref)
    for bad in ([float((1 << 53) + 2), (float(1 << 53), 4), 4],      # next double up: within 1e-6, not exact
                [float(1 << 53), (float(1 << 53), 5), 4],            # AVG count
                [float(1 << 53), (float(1 << 53), 4), 3]):           # COUNT
        try:
            assert_exact(q, {(): bad}, ref)
        except AssertionError:
            continue
        raise AssertionError(f"accepted {bad}")


def test_gamma_bound():
    assert gamma(0) == 0 and gamma(1) == U / (1 - U)
    assert gamma(3) - gamma(2) >= U
    def left_to_right(values):   # not sum(): Python 3.12 compensates float sums
        acc = 0.0
        for t in values:
            acc += t
        return acc

    x = [1e15, 1.0, -1e15, 1e-3, 3.0, -1.0] * 50
    ref = ExactSum("approx", math.fsum(x), math.fsum(abs(t) for t in x), len(x))
    orders = (x, sorted(x), sorted(x, key=abs), sorted(x, key=lambda t: -abs(t)), x[::-1])
    # any summation order stays within the bound ...
    for order in orders:
        assert sum_within_bound(left_to_right(order), ref)
    # ... where 1e-6 relative to the (small) exact sum is a false alarm for some order
    assert any(abs(left_to_right(o) - ref.s) > 1e-6 * abs(ref.s) for o in orders)
    # and it is far tighter than 1e-6 relative when nothing cancels
    y = [float(i % 1000) + 0.5 for i in range(10_000)]
    ry = ExactSum("approx", math.fsum(y), math.fsum(y), len(y))
    assert not sum_within_bound(ry.s * (1 + 1e-9), ry)
    assert not sum_within_bound(math.inf, ry) and not sum_within_bound(math.nan, ry)
    # LONG: exact integer S and A; the bound is evaluated without rounding
    big = ExactSum("approx", (1 << 62) + 1, (1 << 62) + 1, 2)
    assert check_sum(float(1 << 62), big)
    assert Fraction(float(1 << 62)) != big.s


def test_bincount_is_not_an_exact_integer_sum_above_2_53():
    """np.bincount(weights=...) accumulates in float64: past 2^53 every further odd addend is rounded.  The reference's
    int64 sum is exact, and its correctly rounded double is what the device must return."""
    n = (1 << 22) + 4096
    v = np.full(n, INT_MAX, dtype=np.int32)
    v[::3] = INT_MAX - 2
    g = np.zeros(n, dtype=np.int64)
    exact = int(np.sum(v.astype(object)))
    assert exact > 1 << 53
    assert _exact_int_sums(v, g, 1) == [exact]
    in_float = float(np.bincount(g, weights=v.astype(np.float64))[0])
    assert in_float != float(exact)
    assert not check_sum(in_float, ExactSum("int", exact, None, n))
    assert check_sum(float(exact), ExactSum("int", exact, None, n))


INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
FLT_MAX, FLT_TRUE_MIN = float(np.finfo(np.float32).max), float(np.finfo(np.float32).smallest_subnormal)
DBL_MAX, DBL_TRUE_MIN = float(np.finfo(np.float64).max), 5e-324


def _extremes_table(oracle, name, shift=0):
    """Groups (w = 1 only): k = 0 holds INT_MAX only in the raw column, k = 1 INT_MIN / -1 / 0, k = 2 one row (its
    filtered-out twin holds every extreme), k = 3 INT_MIN only.  LONG at INT64_MIN / INT64_MAX and 2^53 + 1, FLOAT /
    DOUBLE at +-inf, +-max and the smallest subnormal."""
    k = np.array([0, 1, 0, 1, 2, 2, 0, 1, 3], dtype=np.int32) + shift
    w = np.array([1, 1, 1, 1, 0, 1, 1, 1, 1], dtype=np.int32)
    ri = np.array([INT_MAX, INT_MIN, INT_MAX, -1, INT_MAX, 5, INT_MAX, 0, INT_MIN], dtype=np.int32)
    lv = np.array([INT64_MAX, INT64_MIN, (1 << 53) + 1, 3, INT64_MIN, 7, 1, (1 << 53) - 1, INT64_MAX], dtype=np.int64)
    f = np.array([np.inf, -np.inf, -FLT_MAX, FLT_MAX, np.inf, FLT_TRUE_MIN, -FLT_TRUE_MIN, 0.5, 1.0], dtype=np.float32)
    d = np.array([-np.inf, DBL_MAX, 2.5, -DBL_MAX, np.inf, -DBL_TRUE_MIN, DBL_TRUE_MIN, np.inf, -1.0], dtype=np.float64)
    s = np.array([b"b", b"a", b"b", b"c", b"zz", b"a", b"d", b"a", b"e"])
    return oracle.build_segment(name, {"k": k, "w": w, "ri": ri, "lv": lv, "f": f, "d": d, "s": s}, raw=["ri"])


EXTREME_QUERY = ("SELECT MIN(ri), MAX(ri), MIN(lv), MAX(lv), MIN(f), MAX(f), MIN(d), MAX(d), DISTINCTCOUNT(s), "
                 "DISTINCTCOUNT(lv), MAX(ri) FILTER(WHERE ri > 0), MIN(d) FILTER(WHERE ri > 0), "
                 "DISTINCTCOUNT(s) FILTER(WHERE ri > 0) FROM t WHERE w = 1 GROUP BY k")


def test_min_max_distinct_of_a_hand_made_table(oracle):
    seg = _extremes_table(oracle, "ext")
    q = sql.parse(EXTREME_QUERY)
    ref = reference(oracle, [seg], q)
    assert set(ref) == {(0,), (1,), (2,), (3,)}
    inf = math.inf
    assert ref[(0,)][:8] == [INT_MAX, INT_MAX, 1, INT64_MAX, -FLT_MAX, inf, -inf, 2.5]
    assert ref[(1,)][:8] == [INT_MIN, 0, INT64_MIN, (1 << 53) - 1, -inf, FLT_MAX, -DBL_MAX, inf]
    assert ref[(2,)][:8] == [5, 5, 7, 7, FLT_TRUE_MIN, FLT_TRUE_MIN, -DBL_TRUE_MIN, -DBL_TRUE_MIN]   # row 4 is filtered out
    assert ref[(3,)][:8] == [INT_MIN, INT_MIN, INT64_MAX, INT64_MAX, 1.0, 1.0, -1.0, -1.0]
    assert type(ref[(0,)][3]) is int and float(ref[(0,)][3]) == 2.0 ** 63      # the exact value; the device's double rounds to nearest
    assert ref[(0,)][8] == frozenset({"b", "d"}) and ref[(1,)][8] == frozenset({"a", "c"})
    assert ref[(1,)][9] == frozenset({INT64_MIN, 3, (1 << 53) - 1})
    # FILTER (WHERE ri > 0): groups 1 and 3 match the main filter only -- the functions' empty values
    assert ref[(0,)][10:] == [INT_MAX, -inf, frozenset({"b", "d"})] and ref[(2,)][10:] == [5, -DBL_TRUE_MIN, frozenset({"a"})]
    for g in ((1,), (3,)):
        assert ref[g][10:] == [-inf, inf, frozenset()]
    # the oracle (double MIN / MAX, dictId sets) agrees on every one of them
    r = oracle.execute(seg, q)
    want = normalise(seg, q, r.num_groups, r.keys, r.doubles, r.longs, r.distinct)
    assert_exact(q, want, ref, "oracle")
    # merged: the union of the rows, keyed by value; a group present in one segment only keeps its own extremes
    both = reference(oracle, [seg, _extremes_table(oracle, "ext2", shift=3)], q)
    assert set(both) == {(i,) for i in range(7)}
    assert both[(3,)][:2] == [INT_MIN, INT_MAX] and both[(3,)][2:4] == [1, INT64_MAX]
    assert both[(3,)][4:8] == [-FLT_MAX, inf, -inf, 2.5] and both[(3,)][8] == frozenset({"b", "d", "e"})
    assert both[(6,)] == ref[(3,)] and both[(1,)] == ref[(1,)]
    # aggregation only, nothing matches: the empty values
    empty = reference(oracle, [seg], sql.parse("SELECT MIN(ri), MAX(lv), DISTINCTCOUNT(s), COUNT(*) FROM t WHERE w > 5"))
    assert empty == {(): [inf, -inf, frozenset(), 0]}


def test_comparator_min_max_bit_exact_and_distinct_sets():
    q = sql.parse("SELECT MIN(v), MAX(v), DISTINCTCOUNT(v) FROM t")
    ref = {(): [float(INT_MIN), float(INT_MAX), frozenset({INT_MIN, 0, INT_MAX})]}
    assert_exact(q, {(): [float(INT_MIN), float(INT_MAX), frozenset({INT_MIN, 0, INT_MAX})]}, ref)
    for bad in ([float(INT_MIN), -math.inf, ref[()][2]],                          # MAX of a non-empty group read as empty
                [math.inf, float(INT_MAX), ref[()][2]],                           # MIN likewise
                [float(INT_MIN), float(INT_MAX - 1), ref[()][2]],                 # the second-largest value
                [float(INT_MIN), float(INT_MAX), frozenset({INT_MIN, INT_MAX})]):  # a value missing from the set
        try:
            assert_exact(q, {(): bad}, ref)
        except AssertionError:
            continue
        raise AssertionError(f"accepted {bad}")
    assert same_double(math.inf, math.inf) and not same_double(0.0, -0.0)
    assert not same_double(2.0 ** 63, float(INT64_MAX - 1024))   # one ulp below 2^63: == on doubles tells them apart too

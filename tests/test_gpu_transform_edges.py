"""-m gpu: DOUBLE transform expressions whose results include NaN, -0.0, +-inf and subnormals, end to end on the device,
against a per-row reference that shares no code with the product.

Per-row values come from tests/transform_ref.py over the source column's values; the reference then follows the
contract of tests/float_edges_ref.py (DESIGN.md section 5): identity is doubleToLongBits (one NaN, two zeros), order is
Double.compare (NaN after +inf), and predicates on an expression compare each row's value with Java's <, > and ==
(float_edges_ref.raw_matches: NaN matches only NEQ / NOT IN, 0 matches both zeros).  Filter trees are evaluated per row
(stored-column leaves by tests/filter_ref.py); NOT complements the doc set, so NaN rows satisfy NOT (E > 0).

Sources: INT and LONG columns with 0, negatives and the type's extremes; DOUBLE and FLOAT columns holding several NaN bit
patterns, both zeros, both infinities, subnormals and +-max, stored as dictionaries (the first NaN's bits kept), and a raw
DOUBLE column that gets a dictionary at load.  Every expression is checked on its derived column and on a raw DOUBLE
"twin" column that stores the expression's per-row values: both must equal the reference.

Checks: filter leaves alone and in AND / OR / NOT trees and FILTER clauses (COUNT, num_docs_scanned and the doc set read
back through DISTINCTCOUNT(rid)); GROUP BY E on the default, hash and global-table routes (the NaN key's bits are the
canonical NaN's); COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT / PERCENTILE of E by a small key; VAR / STDDEV refused on
a non-finite dictionary and exact otherwise; ORDER BY E and MIN(E), selection ORDER BY E, rid and DISTINCT E ORDER BY E;
HAVING on MIN(E) / MAX(E); three segments whose stored NaN bits differ, merged on the device over a bound source and over
the bound expression, with the merged DataTable."""
import math
from fractions import Fraction

import numpy as np
import pytest

import datatable_util
import filter_ref
import float_edges_ref as fr
import transform_ref
from gpu_util import to_device, tuned
from oracle import segment_builder as sb
from pinot_b200 import sql
from pinot_b200._lib import UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext
from test_gpu_float_edges import assert_matches, product_table
from test_gpu_order_by import execute_ordered

pytestmark = pytest.mark.gpu

SIZES = [1, 33, 8_193, 100_003]
DMAX, FMAX = 1.7976931348623157e308, 3.4028234663852886e38
D_NANS = [fr.D_NAN, fr.D_NEG_NAN, fr.D_PAYLOAD_NAN, fr.D_SIGNALLING_NAN]
F_NANS = [fr.F_NAN, fr.F_NEG_NAN, fr.F_PAYLOAD_NAN, fr.F_SIGNALLING_NAN]
INT_POOL = [-(1 << 31), -(1 << 31) + 1, -10 ** 9] + list(range(-13, 14)) + [10 ** 9, (1 << 31) - 1]
LONG_POOL = [-(1 << 63), -(1 << 53) - 1, -(1 << 40)] + list(range(-7, 8)) + [1 << 40, (1 << 53) + 1, (1 << 63) - 1]
D_POOL = [-math.inf, -DMAX, -1e300, -7.25, -2.5, -1.5, -0.75, -5e-324, -0.0, 0.0, 5e-324, 1e-310, 0.75, 1.5, 2.5, 3.0,
          7.25, 1e300, DMAX, math.inf]
F_POOL = [-math.inf, -FMAX, -7.25, -2.5, -1.5, -1e-45, -0.0, 0.0, 1e-45, 0.75, 1.5, 2.5, FMAX, math.inf]
SOURCE_TYPES = {"i": "INT", "l": "LONG", "d": "DOUBLE", "f": "FLOAT", "dr": "DOUBLE"}

# (expression, source): each one produces at least one of NaN, -0.0, +-inf or a subnormal on these sources
EXPRS = [("divide(i,'0')", "i"), ("divide('1',i)", "i"), ("mod(i,'0')", "i"), ("times(i,'-1')", "i"),
         ("ceil(divide(i,'7'))", "i"), ("mod(i,'3')", "i"), ("times(i,'1e300')", "i"),
         ("times(l,'-1')", "l"), ("divide(l,'0')", "l"),
         ("abs(d)", "d"), ("floor(d)", "d"), ("ceil(divide(d,'4'))", "d"), ("plus(d,'0')", "d"), ("times(d,'0')", "d"),
         ("divide(d,'0')", "d"), ("divide('1',d)", "d"), ("mod(d,'2.5')", "d"),
         ("abs(f)", "f"), ("divide('1',f)", "f"), ("times(f,'0')", "f"),
         ("floor(dr)", "dr"), ("divide('1',dr)", "dr"), ("times(dr,'0')", "dr"),
         ("ceil(times(mod(d,'2.5'),'-1'))", "d")]
TWIN = {e: f"tw{k}" for k, (e, _) in enumerate(EXPRS)}


def _draw(rng, pool, n, dtype):
    v = np.array(pool, dtype=dtype)[rng.integers(0, len(pool), size=n)]
    k = min(n, len(pool))
    v[:k] = np.array(pool, dtype=dtype)[rng.permutation(len(pool))[:k]]
    return v


def _floats(rng, pool, nans, n, dtype, first_nan):
    """Values of `pool` and NaNs of every pattern in `nans`; row 0 is the NaN `first_nan` (the bits a stored dictionary
    keeps) and the other NaN rows take the other patterns."""
    of = fr.float_of if dtype == np.float32 else fr.double_of
    v = _draw(rng, pool, n, dtype)
    nan_rows = rng.random(n) < 0.1
    v[nan_rows] = np.array([of(b) for b in nans], dtype=dtype)[rng.integers(0, len(nans), size=int(nan_rows.sum()))]
    v[0] = of(first_nan)
    return v


class Seg:
    """One segment: its device columns (stored, raw, twins), the per-row values of each expression, and the reference's
    view of them (a SegmentData whose expression columns are raw columns named by the expression)."""

    def __init__(self, ctx, name, n, seed, nan_index):
        rng = np.random.default_rng(seed)
        self.n = n
        src = {"i": _draw(rng, INT_POOL, n, np.int32), "l": _draw(rng, LONG_POOL, n, np.int64),
               "d": _floats(rng, D_POOL, D_NANS, n, np.float64, D_NANS[nan_index]),
               "f": _floats(rng, F_POOL, F_NANS, n, np.float32, F_NANS[nan_index]),
               "dr": _floats(rng, D_POOL, D_NANS, n, np.float64, D_NANS[(nan_index + 1) % 4])}
        self.src = src
        self.rid = np.arange(n, dtype=np.int32)
        self.g = rng.integers(0, 5, size=n).astype(np.int32)
        self.m = rng.integers(0, 10, size=n).astype(np.int32)
        self.values = {e: transform_ref.column(e, src[s], SOURCE_TYPES[s]) for e, s in EXPRS}
        stored = [sb.build_column("rid", self.rid), sb.build_column("g", self.g), sb.build_column("m", self.m),
                  sb.build_column("i", src["i"]), sb.build_column("l", src["l"]),
                  fr.build_dict_column("d", src["d"]), fr.build_dict_column("f", src["f"]), sb.build_raw_column("dr", src["dr"])]
        self.data = sb.SegmentData(name, n, stored)
        twins = [sb.build_raw_column(TWIN[e], self.values[e]) for e, _ in EXPRS]
        self.ref = sb.SegmentData(name, n, stored[:3] + [sb.ColumnData(e, sb.DOUBLE, False, 0, 0, False, 0, None, None, None,
                                                                       raw_values=self.values[e]) for e, _ in EXPRS])
        self.full = sb.SegmentData(name, n, stored + twins)
        self.ctx = ctx
        self.dev = to_device(ctx, self.full)

    def reload(self):
        return to_device(self.ctx, self.full)


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def segs(ctx):
    out = [Seg(ctx, f"te{n}", n, 17 + n, k % 4) for k, n in enumerate(SIZES)]
    yield out
    for s in out:
        s.dev.destroy()


def _names(e):
    return [e, TWIN[e]]


# ------------------------------------------------------------------------------------------------------------ filters
def leaves(c):
    out = [Predicate("EQ", c, [0]), Predicate("EQ", c, [-0.0]), Predicate("NEQ", c, [0]), Predicate("EQ", c, [1.5]),
           Predicate("NEQ", c, [-1.5]), Predicate("IN", c, [-0.0, 1.5, 1e308]), Predicate("NOT_IN", c, [0, -1.5]),
           Predicate("EQ", c, [5])]
    for lo, hi in ((0, None), (None, 0), (-0.0, 0.0), (-1e308, None), (None, 1e308), (-1.5, 1.5), (1e308, None)):
        for inc in (True, False):
            out.append(Predicate("RANGE", c, [], lo, hi, inc if lo is not None else True, inc if hi is not None else True))
    return out


def _rename(node, name, old="E"):
    """The tree with `name` in place of the column `old`."""
    if node is None:
        return None
    if isinstance(node, Predicate):
        return Predicate(node.type, name if node.column == old else node.column, list(node.values), node.lower, node.upper,
                         node.lower_inclusive, node.upper_inclusive)
    return Filter(node.type, [_rename(c, name, old) for c in node.children])


_IDENTITIES = {}


def expr_mask(s, e, p):
    """raw_matches over the distinct values of the expression's rows (by identity), spread back to the rows."""
    if (s.n, e) not in _IDENTITIES:
        ids = np.array([fr.identity(v) for v in s.values[e].tolist()], dtype=np.uint64)
        _IDENTITIES[(s.n, e)] = np.unique(ids, return_inverse=True)
    uniq, inverse = _IDENTITIES[(s.n, e)]
    hit = np.array([fr.raw_matches(fr.double_of(int(u)), p, sb.DOUBLE) for u in uniq], dtype=bool)
    return hit[inverse] if s.n else np.zeros(0, dtype=bool)


_STORED = {}


def ref_docs(oracle, s, e, node):
    """bool[n]: the rows the tree selects; E leaves by value, stored leaves by filter_ref, NOT as the complement."""
    if isinstance(node, Predicate):
        if node.column == "E":
            return expr_mask(s, e, node)
        if (s.n, repr(node)) not in _STORED:
            _STORED[(s.n, repr(node))] = filter_ref.matching_docs(oracle, s.data, node)
        return _STORED[(s.n, repr(node))]
    kids = [ref_docs(oracle, s, e, c) for c in node.children]
    if node.type == "NOT":
        return ~kids[0]
    out = kids[0].copy()
    for k in kids[1:]:
        out = out & k if node.type == "AND" else out | k
    return out


def _docs_of(block, a, g=0):
    return np.sort(np.asarray(block.distinct.get((a, g), np.zeros(0)), dtype=np.int64))


def test_filters(oracle, pm, segs):
    """Leaves on E alone, in AND / OR / NOT trees with stored columns, and as FILTER clauses."""
    for s in segs:
        for e, _ in EXPRS:
            for leaf in leaves("E"):
                trees = [leaf, Filter("AND", [leaf, Predicate("RANGE", "g", [], None, 2, True, False)]),
                         Filter("OR", [leaf, Predicate("EQ", "m", [3])]), Filter("NOT", [leaf])]
                wants = [ref_docs(oracle, s, e, t) for t in trees]
                for name in _names(e):
                    for t, want in zip(trees, wants):
                        q = QueryContext([Aggregation("COUNT"), Aggregation("DISTINCTCOUNT", "rid")], filter=_rename(t, name))
                        b = pm.execute_segments([s.dev], q)[0]
                        what = (s.n, name, e, t)
                        k = int(want.sum())
                        assert b.stats.num_docs_scanned == k, what
                        assert int(b.longs[0][0]) == k, what
                        assert np.array_equal(_docs_of(b, 1), np.nonzero(want)[0]), what
                    clause = _rename(leaf, name)
                    q = QueryContext([Aggregation("COUNT"), Aggregation("COUNT", filter=clause),
                                      Aggregation("DISTINCTCOUNT", "rid", filter=clause)])
                    b = pm.execute_segments([s.dev], q)[0]
                    assert int(b.longs[0][0]) == s.n and int(b.longs[1][0]) == int(wants[0].sum()), (s.n, name, leaf)
                    assert np.array_equal(_docs_of(b, 2), np.nonzero(wants[0])[0]), (s.n, name, leaf)


# ----------------------------------------------------------------------------------------------- groups, aggregates
_REF = {}


def reference(s, q, key):
    k = (s.n, key)
    if k not in _REF:
        _REF[k] = fr.reference(None, [s.ref], q)
    return _REF[k]


def _swap(q, e, name):
    sub = lambda c: name if c == e else c  # noqa: E731
    return QueryContext([Aggregation(a.function, sub(a.column), arg=a.arg) for a in q.aggregations],
                        filter=_rename(q.filter, name, e), group_by=[sub(g) for g in q.group_by],
                        order_by=[(sub(c), asc) for c, asc in q.order_by], limit=q.limit, num_groups_limit=1_000_000)


def test_group_by_expression_on_every_route(ctx, pm, segs):
    """GROUP BY E: -0.0 and 0.0 are two groups, every NaN one group whose key is the canonical NaN."""
    for s in segs:
        for e, _ in EXPRS:
            base = QueryContext([Aggregation("COUNT"), Aggregation("SUM", "m"), Aggregation("DISTINCTCOUNT", "g")],
                                group_by=[e], num_groups_limit=1_000_000)
            want = reference(s, base, ("gb", e))
            for knobs in ({}, {"dense_max": 1}, {"smem_groups": 0}):
                with tuned(ctx, **knobs):
                    for name in _names(e):
                        q = _swap(base, e, name)
                        b = pm.execute_segments([s.dev], q)[0]
                        got = product_table(s.dev, q, b)
                        assert_matches(q, got, want, f"n={s.n} {name} {e} {knobs}")
                        if name == e:
                            nan_ids = [int(b.keys[g, 0]) for g in range(b.num_groups)
                                       if math.isnan(s.dev.dictionary_value(e, int(b.keys[g, 0])))]
                            assert len(nan_ids) == (1 if np.isnan(s.values[e]).any() else 0), (s.n, e)
                            for i in nan_ids:
                                assert fr.bits_of(s.dev.dictionary_value(e, i)) == fr.D_NAN, (s.n, e)


def test_aggregates_of_the_expression(pm, segs):
    """COUNT / SUM / AVG by check_sum, MIN / MAX / PERCENTILE bit for bit (any NaN for NaN), DISTINCTCOUNT as identities."""
    for s in segs:
        for e, _ in EXPRS:
            # a finite sum that overflows (+-max twice) is +-inf or finite by the order of the additions: SUM / AVG only
            # where no sum of the finite values can leave the double range
            finite = np.abs(s.values[e][np.isfinite(s.values[e])])
            sums = [Aggregation("SUM", e), Aggregation("AVG", e)] if not len(finite) or finite.max() < DMAX / s.n else []
            qs = [QueryContext([Aggregation("COUNT"), Aggregation("MIN", e), Aggregation("MAX", e),
                                Aggregation("DISTINCTCOUNT", e)] + sums, group_by=["g"], num_groups_limit=1_000_000),
                  QueryContext([Aggregation("MIN", e), Aggregation("MAX", e), Aggregation("DISTINCTCOUNT", e)] + sums[:1]),
                  QueryContext([Aggregation("PERCENTILE", e, arg=0.0), Aggregation("PERCENTILE", e, arg=50.0),
                                Aggregation("PERCENTILE", e, arg=100.0)], group_by=["g"], num_groups_limit=1_000_000),
                  QueryContext([Aggregation("COUNT"), Aggregation("MIN", e), Aggregation("MAX", e)],
                               filter=Predicate("RANGE", e, [], 0, None, True, True))]
            for k, q0 in enumerate(qs):
                want = reference(s, q0, ("agg", e, k))
                for name in _names(e):
                    q = _swap(q0, e, name)
                    assert_matches(q, product_table(s.dev, q, pm.execute_segments([s.dev], q)[0]), want, f"n={s.n} {name} {e} #{k}")


def test_variance_refuses_non_finite_and_is_exact_otherwise(pm, segs):
    for s in segs:
        for e, _ in EXPRS:
            v = s.values[e]
            q = QueryContext([Aggregation("VARPOP", e), Aggregation("STDDEVSAMP", e)])
            if not np.all(np.isfinite(v)):
                with pytest.raises(UnsupportedQueryError):
                    pm.execute_segments([s.dev], q)
                continue
            xs = [Fraction(float(x)) for x in v]
            lo, hi = min(xs), max(xs)
            # the grid's step 2^e: the lowest set bit over the differences from the smallest value (dyadic rationals)
            e2 = min(((d.numerator & -d.numerator).bit_length() - d.denominator.bit_length() for d in {x - lo for x in xs} - {0}),
                     default=0)
            if (hi - lo) / Fraction(2) ** e2 >= 2 ** 32:
                # values no grid of 2^32 steps holds (DESIGN.md section 3.9): refused rather than rounded
                with pytest.raises(UnsupportedQueryError):
                    pm.execute_segments([s.dev], q)
                continue
            b = pm.execute_segments([s.dev], QueryContext([Aggregation("VARPOP", e)]))[0]
            mean = sum(xs) / len(xs)
            assert float(b.doubles[0][0]) == float(sum((x - mean) ** 2 for x in xs) / len(xs)), (s.n, e)


# ------------------------------------------------------------------------------------------------------------- order
def _keys(dev, q, b):
    return [tuple(fr.Key(dev.dictionary_value(c, int(b.keys[g, j]))) for j, c in enumerate(q.group_by)) for g in range(b.num_groups)]


def test_order_by_expression_and_its_minimum(pm, segs):
    for s in segs:
        for e, _ in EXPRS:
            for asc in (True, False):
                base = QueryContext([Aggregation("COUNT"), Aggregation("SUM", "m")], group_by=[e], order_by=[(e, asc)], limit=5,
                                    num_groups_limit=1_000_000)
                want = fr.ordered(base, reference(s, base, ("gb2", e)), sql.resolve_order_by(base))
                for name in _names(e):
                    q = _swap(base, e, name)
                    for trim in (0, 3):
                        got = _keys(s.dev, q, execute_ordered(pm, [s.dev], q, trim)[0])
                        assert got == [k for k, _ in (want if trim == 0 else want[:trim])], (s.n, name, asc, trim)
                base = QueryContext([Aggregation("MIN", e), Aggregation("COUNT")], group_by=["g"], order_by=[(f"MIN({e})", asc)],
                                    limit=5, num_groups_limit=1_000_000)
                want = fr.ordered(base, reference(s, base, ("min", e, asc)), sql.resolve_order_by(base))
                for name in _names(e):
                    q = QueryContext([Aggregation("MIN", name), Aggregation("COUNT")], group_by=["g"],
                                     order_by=[(f"MIN({name})", asc)], limit=5, num_groups_limit=1_000_000)
                    got = _keys(s.dev, q, execute_ordered(pm, [s.dev], q, 0)[0])
                    assert got == [k for k, _ in want], (s.n, name, asc)


def _sort_key(x, asc):
    k = transform_ref.double_order_key(float(x))
    return k if asc else -k


def test_selection_and_distinct_order(pm, segs):
    """SELECT E, rid ORDER BY E, rid and SELECT DISTINCT E ORDER BY E: Double.compare order, NaN after +inf."""
    for s in segs:
        for e, _ in EXPRS:
            v = s.values[e]
            for asc in (True, False):
                order = sorted(range(s.n), key=lambda r: (_sort_key(v[r], asc), r))[:60]
                uniq = sorted(fr.unique_values(v, sb.DOUBLE), key=fr.ORDER, reverse=not asc)
                for name in _names(e):
                    b = pm.execute_selection([s.dev], sql.SelectionQuery(columns=[name, "rid"], order_by=[(name, asc), ("rid", True)],
                                                                         limit=60))[0]
                    assert [fr.identity(float(x)) for x in b.columns[0]] == [fr.identity(v[r]) for r in order], (s.n, name, asc)
                    assert [int(r) for r in b.columns[1]] == order, (s.n, name, asc)
                    d = pm.execute_distinct([s.dev], sql.DistinctQuery(columns=[name], order_by=[(name, asc)], limit=1000))[0]
                    assert [fr.identity(float(x)) for x in d.columns[0]] == [fr.identity(x) for x in uniq[:1000]], (s.n, name, asc)


def test_having_on_the_expression(pm, segs):
    """HAVING MIN(E) = 0 and MAX(E) > 0 compare the final values like Java: -0.0 = 0, NaN matches neither."""
    for s in segs:
        for e, _ in EXPRS:
            base = QueryContext([Aggregation("MIN", e), Aggregation("MAX", e), Aggregation("COUNT")], group_by=["g"],
                                num_groups_limit=1_000_000)
            table = reference(s, base, ("having", e))
            for cond, test in (("MIN({}) = 0", lambda r: r[0] == 0), ("MAX({}) > 0", lambda r: r[1] > 0)):
                want = sorted(k[0].v for k, r in table.items() if test(r))
                for name in _names(e):
                    q = sql.parse(f"SELECT g, MIN({name}), MAX({name}), COUNT(*) FROM t GROUP BY g HAVING {cond.format(name)}",
                                  num_groups_limit=1_000_000)
                    b = pm.execute_segments([s.dev], q)[0]
                    got = sorted(int(s.dev.dictionary_value("g", int(b.keys[g, 0]))) for g in range(b.num_groups))
                    assert got == want, (s.n, name, cond)


# ------------------------------------------------------------------------------------------------------------ merged
@pytest.mark.parametrize("bound", ["source", "expression"])
def test_merged_segments_with_different_nan_bits(ctx, pm, bound):
    """Three segments whose stored d dictionaries keep three different NaN bit patterns, merged on the device: one NaN
    group, two zero groups, the reference's values over the union; the DataTable of the merged GROUP BY too."""
    parts = [Seg(ctx, f"mg{k}", n, 500 + k, k) for k, n in enumerate((8_193, 3_333, 997))]
    assert len({fr.bits_of(p.full.column("d").dict_values[-1]) for p in parts}) == 3
    exprs = [e for e, src in EXPRS if src == "d"]
    try:
        for e in exprs:
            devs = [p.reload() for p in parts]
            try:
                dom = DictionaryDomain.build(ctx, devs, ["d"] if bound == "source" else [e])
                for d in devs:
                    d.bind_domain(dom)
                dom.release()
                q = QueryContext([Aggregation("COUNT"), Aggregation("SUM", "m"), Aggregation("MIN", e), Aggregation("MAX", e),
                                  Aggregation("DISTINCTCOUNT", "g")], group_by=[e], num_groups_limit=1_000_000)
                want = fr.reference(None, [p.ref for p in parts], q)
                block = pm.execute_segments(devs, q, merge=True, keep_handle=True, defer=False)[0]
                try:
                    assert_matches(q, product_table(devs[0], q, block), want, f"{bound} {e}")
                    dt = datatable_util.parse(pm.to_datatable(devs[0], q, block))
                finally:
                    block.release(ctx)
                keys = [r[0] for r in dt["rows"]]
                assert sorted(fr.identity(k) for k in keys) == sorted(k[0]._id() for k in want), (bound, e)
                nan_rows = [k for k in keys if math.isnan(k)]
                assert len(nan_rows) == 1 and fr.bits_of(nan_rows[0]) == fr.D_NAN, (bound, e)
                zeros = [fr.bits_of(k) for k in keys if k == 0]
                assert sorted(zeros) == sorted({fr.bits_of(z) for z in np.concatenate([p.values[e] for p in parts]) if z == 0}), (bound, e)
            finally:
                for d in devs:
                    d.destroy()
    finally:
        for p in parts:
            p.dev.destroy()

"""Host-side query model: the slice of Pinot's ``QueryContext`` the scan -> filter -> group-by path consumes.

Mirrors (names and meaning, not code) ``pinot-core/src/main/java/org/apache/pinot/core/query/request/context/
QueryContext.java``: a filter tree (``FilterContext`` with AND / OR / NOT / PREDICATE nodes,
``pinot-common/.../request/context/FilterContext.java``), group-by expressions (identifiers only on this path),
aggregation functions and the two server options that shape group-by execution (``numGroupsLimit`` and
``maxInitialResultHolderCapacity``: ``core/plan/maker/InstancePlanMakerImplV2.java:68-91``).

Predicates are in VALUE space here (as the broker sends them); turning them into dictId space is the plan maker's job
(``pinot_b200/plan_maker.py``), exactly where the reference runs its ``PredicateEvaluator``s.
"""
from __future__ import annotations

import math
import re
import struct
from dataclasses import dataclass, field
from fractions import Fraction
from typing import List, Optional, Sequence, Union

# InstancePlanMakerImplV2 defaults (core/plan/maker/InstancePlanMakerImplV2.java:68-82)
DEFAULT_MAX_INITIAL_RESULT_HOLDER_CAPACITY = 10_000
DEFAULT_NUM_GROUPS_LIMIT = 100_000

Literal = Union[int, float, str]


@dataclass
class Predicate:
    """Leaf of the filter tree: ``Predicate.Type`` EQ / NOT_EQ / IN / NOT_IN / RANGE / REGEXP_LIKE on an identifier."""
    type: str  # "EQ" | "NEQ" | "IN" | "NOT_IN" | "RANGE" | "REGEXP_LIKE"
    column: str
    values: List[Literal] = field(default_factory=list)  # EQ/NEQ: [v]; IN/NOT_IN: [v...]; REGEXP_LIKE: [pattern]
    lower: Optional[Literal] = None  # RANGE; None = unbounded ("*")
    upper: Optional[Literal] = None
    lower_inclusive: bool = True
    upper_inclusive: bool = True


@dataclass
class Filter:
    """AND / OR / NOT node (``FilterContext.Type``)."""
    type: str  # "AND" | "OR" | "NOT"
    children: List[Union["Filter", Predicate]] = field(default_factory=list)


FilterNode = Union[Filter, Predicate]


@dataclass(frozen=True)
class AggFunction:
    family: str       # as a refusal shared by the family names it ("VAR/STDDEV", "MIN/MAX", ...)
    arg: Optional[str]  # the argument besides the column: None, "percentile", "log2m" or "time" (the time column)
    dict_ids: bool    # reads its column's dictIds: a merged submission needs one dictionary for that column


# What each aggregation function is, in PB200_AGG_* code order (_lib.AGG_CODES): the package's half of
# pinot_b200/csrc/pb200_aggfn.h.  FIRST/LASTWITHTIME's data column is bound with its time column, not through dict_ids.
AGG_FUNCTIONS = {
    "COUNT": AggFunction("COUNT", None, False),
    "SUM": AggFunction("SUM/AVG", None, False),
    "MIN": AggFunction("MIN/MAX", None, True),
    "MAX": AggFunction("MIN/MAX", None, True),
    "AVG": AggFunction("SUM/AVG", None, False),
    "DISTINCTCOUNT": AggFunction("DISTINCTCOUNT", None, True),
    "PERCENTILE": AggFunction("PERCENTILE", "percentile", True),
    "VARPOP": AggFunction("VAR/STDDEV", None, True),
    "VARSAMP": AggFunction("VAR/STDDEV", None, True),
    "STDDEVPOP": AggFunction("VAR/STDDEV", None, True),
    "STDDEVSAMP": AggFunction("VAR/STDDEV", None, True),
    "FIRSTWITHTIME": AggFunction("FIRST/LASTWITHTIME", "time", False),
    "LASTWITHTIME": AggFunction("FIRST/LASTWITHTIME", "time", False),
    "DISTINCTSUM": AggFunction("DISTINCTSUM/DISTINCTAVG", None, True),
    "DISTINCTAVG": AggFunction("DISTINCTSUM/DISTINCTAVG", None, True),
    "DISTINCTCOUNTHLL": AggFunction("DISTINCTCOUNTHLL", "log2m", True),
}


def functions_where(test) -> tuple:
    """The names of the functions whose AggFunction passes `test`, in code order."""
    return tuple(name for name, f in AGG_FUNCTIONS.items() if test(f))


WITHTIME_FUNCTIONS = functions_where(lambda f: f.arg == "time")
MOMENT_FUNCTIONS = functions_where(lambda f: f.family == "VAR/STDDEV")
# functions whose intermediate is the set of distinct values (merged by union)
DISTINCT_SET_FUNCTIONS = functions_where(lambda f: f.family in ("DISTINCTCOUNT", "DISTINCTSUM/DISTINCTAVG"))


@dataclass
class Aggregation:
    function: str  # COUNT | SUM | MIN | MAX | AVG | DISTINCTCOUNT | PERCENTILE | VARPOP | VARSAMP | STDDEVPOP | STDDEVSAMP
    #                | FIRSTWITHTIME | LASTWITHTIME | DISTINCTSUM | DISTINCTAVG | DISTINCTCOUNTHLL
    column: Optional[str] = None  # None for COUNT(*)
    # FILTER (WHERE ...) clause of this function (QueryContext.getFilteredAggregationFunctions: Pair<function, FilterContext>);
    # evaluated together with the query's own filter (AggregationFunctionUtils.buildFilteredAggregationInfos)
    filter: Optional["FilterNode"] = None
    arg: Optional[float] = None  # PERCENTILE: the percentile, 0 <= p <= 100; DISTINCTCOUNTHLL: log2m (an int, default 8)
    # FIRSTWITHTIME / LASTWITHTIME(column, time_column, 'value_type'): the time column and the type literal (upper case)
    time_column: Optional[str] = None
    value_type: Optional[str] = None
    # named only in HAVING: computed like the others, never an output column (Pinot's QueryContext adds such functions too)
    hidden: bool = False

    def __str__(self):
        if self.function == "PERCENTILE":
            return f"percentile({self.column}, {self.arg:g})"
        if self.function == "DISTINCTCOUNTHLL" and self.arg != HLL_DEFAULT_LOG2M:
            return f"distinctcounthll({self.column}, {self.arg})"
        if self.function in WITHTIME_FUNCTIONS:
            return f"{self.function.lower()}({self.column},{self.time_column},'{self.value_type}')"
        return f"{self.function.lower()}({self.column or '*'})"


@dataclass
class PostAggregation:
    """Arithmetic over the final values of aggregations (Pinot's post-aggregation expression), e.g. SUM(a) / SUM(b)
    (DESIGN.md section 3.18).  `program` is postfix, root last: ("AGG", a) with a indexing QueryContext.aggregations,
    ("LIT", float), ("NEG",), ("ADD",), ("SUB",), ("MUL",), ("DIV",).  `text` is its normalised name
    (divide(sum(a),sum(b))): what an ORDER BY item is matched with and the CLI's column header."""
    text: str
    program: List[tuple]

    def __str__(self):
        return self.text


def java_divide(x: float, y: float) -> float:
    """x / y as one IEEE-754 double division, as Java computes it: a division by zero gives +-inf (the sign of x times
    the sign of the zero), and NaN for 0 / 0 or a NaN operand; Python raises there instead."""
    if y != 0.0:
        return x / y
    if x == 0.0 or math.isnan(x):
        return math.nan
    return math.copysign(math.inf, x) * math.copysign(1.0, y)


def post_eval(program, value) -> float:
    """The value of a post-aggregation program (PostAggregation.program) for one row; value(a) = the final value of
    aggregation a.  Each operand is read as a float and each operator is one IEEE-754 double operation, rounded to
    nearest (pinot_b200/csrc/pb200_postagg.h is the library's copy of this rule)."""
    st: List[float] = []
    for n in program:
        op = n[0]
        if op == "AGG":
            st.append(float(value(n[1])))
        elif op == "LIT":
            st.append(float(n[1]))
        elif op == "NEG":
            st.append(-st.pop())
        else:
            y = st.pop()
            x = st.pop()
            st.append(x + y if op == "ADD" else x - y if op == "SUB" else x * y if op == "MUL" else java_divide(x, y))
    return st[0]


# the type literal of FIRST/LASTWITHTIME -> the stored type it names (BOOLEAN is stored as INT)
WITHTIME_TYPES = {"INT": 0, "BOOLEAN": 0, "LONG": 1, "FLOAT": 2, "DOUBLE": 3, "STRING": 4}


def withtime_pick(function: str, cur, new):
    """By-value merge of two FIRST/LASTWITHTIME intermediates (time value, data value); None is an empty one.  `new`
    comes later in the call's row order: LAST keeps it on a tie, FIRST keeps `cur`."""
    if cur is None:
        return new
    if new is None:
        return cur
    if function == "LASTWITHTIME":
        return new if new[0] >= cur[0] else cur
    return new if new[0] < cur[0] else cur


def percentile_index(n: int, p: float) -> int:
    """PercentileAggregationFunction.extractFinalResult's index among n > 0 sorted values: the largest at p == 100,
    otherwise int((double)n * p / 100.0) -- product, division, truncation -- clamped to n - 1."""
    if p == 100.0:
        return n - 1
    return min(int(float(n) * float(p) / 100.0), n - 1)


def value_order(v):
    """Sort key of a value in the reference's total order: a float in Double.compare order (-0.0 before 0.0, every NaN
    one value after +inf), any other value as it is."""
    if isinstance(v, float):
        u = struct.unpack("<Q", struct.pack("<d", v))[0]
        if u & 0x7FFFFFFFFFFFFFFF > 0x7FF0000000000000:
            u = 0x7FF8000000000000
        return u ^ 0xFFFFFFFFFFFFFFFF if u >> 63 else u | (1 << 63)
    return v


class ValueKey(float):
    """A float compared by identity, as the reference's group keys, DISTINCTCOUNT sets and histograms are
    (Double.equals / doubleToLongBits): all NaNs are one value, -0.0 and 0.0 are two.  Prints and sums as the float."""
    __slots__ = ()

    def __eq__(self, other):
        return isinstance(other, float) and value_order(float(self)) == value_order(float(other))

    def __ne__(self, other):
        return not self == other

    def __hash__(self):
        return hash(value_order(float(self)))


def value_key(v):
    """`v` as a key of a by-value merge: floats by identity (ValueKey), other values as they are."""
    return ValueKey(v) if isinstance(v, float) else v


def percentile_of_counts(counts) -> float:
    """PERCENTILE over a {value: count} multiset (the by-value merge of per-segment histograms); -inf when empty.
    `counts` is (p, {value: count}); values rank in Double.compare order."""
    p, hist = counts
    n = sum(hist.values())
    if n == 0:
        return float("-inf")
    k = percentile_index(n, p)
    for v in sorted(hist, key=value_order):
        k -= hist[v]
        if k < 0:
            return float(v)
    raise AssertionError("unreachable")


def distinct_final(function: str, values) -> float:
    """The final DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG of a set of distinct values (DESIGN.md section 3.14):
    the set size, or the exact sum (divided by the size) rounded once to the nearest double.  Empty: 0.0 / -inf.  NaN
    in the set, or both infinities: NaN; otherwise an infinity in the set wins.  Integer members (INT / LONG values) stay
    Python integers: a LONG beyond 2^53 is summed exactly, not rounded to a double first."""
    if function == "DISTINCTCOUNT":
        return len(values)
    values = [v.item() if hasattr(v, "item") else v for v in values]
    floats = [float(v) for v in values if isinstance(v, float)]
    if any(math.isnan(v) for v in floats) or (math.inf in floats and -math.inf in floats):
        return math.nan
    if math.inf in floats or -math.inf in floats:
        return math.inf if math.inf in floats else -math.inf
    if not values:
        return 0.0 if function == "DISTINCTSUM" else -math.inf
    exact = sum((Fraction(v) for v in values), Fraction(0))
    if function == "DISTINCTAVG":
        exact /= len(values)
    try:
        return float(exact)   # numerator / denominator of ints: correctly rounded, subnormals included
    except OverflowError:
        return math.inf if exact > 0 else -math.inf


# DISTINCTCOUNTHLL (DESIGN.md section 3.17): its intermediate is DISTINCTCOUNT's set of distinct values too, merged by union
HLL_DEFAULT_LOG2M = 8
_M32 = 0xFFFFFFFF
_MURMUR_M = 0x5BD1E995


def _hll_hash_long(data: int) -> int:
    """stream-lib MurmurHash.hashLong of a Java long (any Python int, taken mod 2^64)."""
    data &= 0xFFFFFFFFFFFFFFFF
    h = 0
    k = ((data & _M32) * _MURMUR_M) & _M32
    k ^= k >> 24
    h ^= (k * _MURMUR_M) & _M32
    k = ((data >> 32) * _MURMUR_M) & _M32
    k ^= k >> 24
    h = (h * _MURMUR_M) & _M32
    h ^= (k * _MURMUR_M) & _M32
    h ^= h >> 13
    h = (h * _MURMUR_M) & _M32
    return h ^ (h >> 15)


def _hll_hash_bytes(b: bytes, seed: int = -1) -> int:
    """stream-lib MurmurHash.hash(byte[], length, seed): the tail bytes are sign-extended, as a Java byte is."""
    n = len(b)
    h = (seed ^ n) & _M32
    for i in range(n >> 2):
        k = (int.from_bytes(b[4 * i:4 * i + 4], "little") * _MURMUR_M) & _M32
        k ^= k >> 24
        k = (k * _MURMUR_M) & _M32
        h = ((h * _MURMUR_M) & _M32) ^ k
    left = n & 3
    if left:
        sx = [x - 256 if x > 127 else x for x in b[n - left:]]
        if left >= 3:
            h ^= (sx[-3] << 16) & _M32
        if left >= 2:
            h ^= (sx[-2] << 8) & _M32
        h ^= sx[-1] & _M32
        h = (h * _MURMUR_M) & _M32
    h ^= h >> 13
    h = (h * _MURMUR_M) & _M32
    return h ^ (h >> 15)


def hll_hash(value, data_type: Optional[str] = None) -> int:
    """MurmurHash.hash(Object) of a dictionary value: INT / LONG as a long, FLOAT through floatToRawIntBits
    (sign-extended), DOUBLE through doubleToRawLongBits, STRING over its UTF-8 bytes.  data_type ("INT" ... "STRING")
    tells a FLOAT from a DOUBLE; without it a float is a DOUBLE."""
    value = value.item() if hasattr(value, "item") else value
    if isinstance(value, str):
        return _hll_hash_bytes(value.encode("utf-8"))
    if isinstance(value, float):
        if data_type == "FLOAT":
            return _hll_hash_long(struct.unpack("<i", struct.pack("<f", value))[0])
        return _hll_hash_long(struct.unpack("<q", struct.pack("<d", value))[0])
    return _hll_hash_long(int(value))


_TYPE_NAMES = {0: "INT", 1: "LONG", 2: "FLOAT", 3: "DOUBLE", 4: "STRING"}


class HllSet(set):
    """The distinct values of a DISTINCTCOUNTHLL intermediate and the column's stored type (a FLOAT hashes other bits
    than the same DOUBLE); unions in place keep the type."""

    def __init__(self, values=(), data_type=None):
        super().__init__(values)
        self.data_type = _TYPE_NAMES.get(data_type, data_type)


def hll_final(values, log2m: int = HLL_DEFAULT_LOG2M, data_type: Optional[str] = None) -> int:
    """DISTINCTCOUNTHLL of a set of distinct values (DESIGN.md section 3.17): the estimate of stream-lib's HyperLogLog with
    2^log2m registers offered every member (HyperLogLog.cardinality, registerSum summed exactly, Java's Math.round).  An
    empty set gives 0."""
    p = int(log2m)
    m = 1 << p
    reg = [0] * m
    for v in values:
        x = hll_hash(v, data_type)
        y = ((x << p) & _M32) | ((1 << (p - 1)) + 1)
        j = x >> (32 - p)
        reg[j] = max(reg[j], 33 - y.bit_length())
    register_sum = math.ldexp(sum(1 << (33 - p - r) for r in reg), -(33 - p))   # exact: an integer below 2^34, scaled
    zeros = reg.count(0)
    alpha_mm = {4: 0.673 * m * m, 5: 0.697 * m * m, 6: 0.709 * m * m}.get(p, (0.7213 / (1 + 1.079 / m)) * m * m)
    estimate = alpha_mm * (1 / register_sum)
    if estimate <= 2.5 * m:
        if zeros == 0:
            return (1 << 63) - 1   # m * log(+inf): Math.round(+inf)
        estimate = m * math.log(m / zeros)
    f = math.floor(estimate)
    return f + (1 if estimate - f >= 0.5 else 0)


@dataclass(frozen=True)
class Moments:
    """Exact moments of n values v_i = c + k_i * 2^e (c = c_mant * 2^c_exp): s1 = sum k_i, s2 = sum k_i^2 -- the
    intermediate of VAR / STDDEV that per-segment results are merged by (pb200_result_moments)."""
    n: int
    c_mant: int
    c_exp: int
    e: int
    s1: int
    s2: int

    def value_sums(self):
        """(n, sum v, sum v^2) as exact Fractions."""
        from fractions import Fraction
        c = Fraction(self.c_mant) * Fraction(2) ** self.c_exp
        u = Fraction(2) ** self.e
        return self.n, self.n * c + self.s1 * u, self.n * c * c + 2 * c * self.s1 * u + self.s2 * u * u


def merge_moments(parts) -> tuple:
    """By-value merge of Moments: (n, sum v, sum v^2), exact."""
    from fractions import Fraction
    n, s1, s2 = 0, Fraction(0), Fraction(0)
    for m in parts:
        a, b, c = m.value_sums()
        n, s1, s2 = n + a, s1 + b, s2 + c
    return n, s1, s2


def moments_final(function: str, sums) -> float:
    """VarianceAggregationFunction's final value from exact (n, sum v, sum v^2), rounded once: -inf for n == 0, and for
    the *SAMP functions at n == 1; STDDEV is the sqrt of the rounded variance."""
    import math
    from fractions import Fraction
    n, s1, s2 = sums
    samp = function in ("VARSAMP", "STDDEVSAMP")
    if n == 0 or (samp and n == 1):
        return float("-inf")
    m2 = Fraction(s2) - Fraction(s1) * Fraction(s1) / n   # sum (v - mean)^2
    var = float(m2 / (n - 1 if samp else n))              # Fraction -> float rounds to nearest
    return math.sqrt(var) if function.startswith("STDDEV") else var


@dataclass
class QueryContext:
    aggregations: List[Aggregation]
    filter: Optional[FilterNode] = None
    group_by: List[str] = field(default_factory=list)
    table: str = "testTable"
    limit: int = 10
    order_by: List[tuple] = field(default_factory=list)  # (expression string, ascending)
    num_groups_limit: int = DEFAULT_NUM_GROUPS_LIMIT
    max_initial_result_holder_capacity: int = DEFAULT_MAX_INITIAL_RESULT_HOLDER_CAPACITY
    and_scan_reordering: bool = False
    use_star_tree: bool = True  # query option useStarTree
    # GROUP BY ... ORDER BY ... LIMIT n trims to max(5 * n, option) groups (option > 0; else no trim): the merged result
    # (query options minServerGroupTrimSize, default 5000) and per-segment results (minSegmentGroupTrimSize, default off)
    min_server_group_trim_size: int = 5000
    min_segment_group_trim_size: int = -1
    # HAVING: a filter tree whose leaves name aggregations by sql.having_name and compare them with numeric literals
    # (sql.resolve_having gives the library's postfix form); applied to final rows, before ORDER BY and LIMIT
    having: Optional[FilterNode] = None
    # arithmetic over aggregations in the SELECT list (PostAggregation; an ORDER BY expression is one of them), and the
    # SELECT list in its order: ("COLUMN", name), ("AGG", index into aggregations), ("POST", index into post_aggregations)
    post_aggregations: List[PostAggregation] = field(default_factory=list)
    select: List[tuple] = field(default_factory=list)

    @property
    def is_group_by(self) -> bool:
        return len(self.group_by) > 0


def having_eval(nodes, values) -> bool:
    """The outcome of a HAVING postfix tree (sql.resolve_having) for one row; values[a] = the final value of aggregation a
    as a float.  Python's float comparisons are Java's: a NaN matches only NEQ, -0.0 == 0.0 (pinot_b200/csrc/pb200_having.h
    is the library's copy of this rule)."""
    stack = []
    for n in nodes:
        op = n[0]
        if op in ("AND", "OR"):
            args = stack[len(stack) - n[1]:]
            del stack[len(stack) - n[1]:]
            stack.append(all(args) if op == "AND" else any(args))
        elif op == "NOT":
            stack.append(not stack.pop())
        elif op == "EQ":
            stack.append(values[n[1]] == n[2])
        elif op == "NEQ":
            stack.append(not values[n[1]] == n[2])
        else:  # RANGE: (agg, lo or None, hi or None, lo inclusive, hi inclusive)
            _, a, lo, hi, lo_inc, hi_inc = n
            v = values[a]
            stack.append((lo is None or (v >= lo if lo_inc else v > lo)) and (hi is None or (v <= hi if hi_inc else v < hi)))
    return stack[0]


# ----------------------------------------------------------------------------------------------------------------------
# Broker-side filter optimizers that shape what the server receives
# (core/query/optimizer/filter/{FlattenAndOr,MergeEqIn,MergeRange}FilterOptimizer.java)
# ----------------------------------------------------------------------------------------------------------------------
def flatten(node: Optional[FilterNode]) -> Optional[FilterNode]:
    if node is None or isinstance(node, Predicate):
        return node
    kids = [flatten(c) for c in node.children]
    if node.type in ("AND", "OR"):
        flat = []
        for k in kids:
            if isinstance(k, Filter) and k.type == node.type:
                flat.extend(k.children)
            else:
                flat.append(k)
        kids = flat
        if len(kids) == 1:
            return kids[0]
    return Filter(node.type, kids)


def merge_eq_in(node: Optional[FilterNode]) -> Optional[FilterNode]:
    """OR of EQ/IN on the same column -> one IN (MergeEqInFilterOptimizer)."""
    if node is None or isinstance(node, Predicate):
        return node
    kids = [merge_eq_in(c) for c in node.children]
    if node.type != "OR":
        return Filter(node.type, kids)
    by_col = {}
    rest = []
    for k in kids:
        if isinstance(k, Predicate) and k.type in ("EQ", "IN"):
            by_col.setdefault(k.column, []).append(k)
        else:
            rest.append(k)
    merged = []
    for col, preds in by_col.items():
        if len(preds) == 1:
            merged.append(preds[0])
        else:
            vals = []
            for p in preds:
                for v in p.values:
                    if v not in vals:
                        vals.append(v)
            merged.append(Predicate("EQ", col, vals) if len(vals) == 1 else Predicate("IN", col, vals))
    out = merged + rest
    return out[0] if len(out) == 1 else Filter("OR", out)


def merge_range(node: Optional[FilterNode]) -> Optional[FilterNode]:
    """AND of several RANGE predicates on the same column -> their intersection (MergeRangeFilterOptimizer)."""
    if node is None or isinstance(node, Predicate):
        return node
    kids = [merge_range(c) for c in node.children]
    if node.type != "AND":
        return Filter(node.type, kids)
    ranges = {}
    others = []
    recreate = False
    for k in kids:
        if isinstance(k, Predicate) and k.type == "RANGE":
            cur = ranges.get(k.column)
            if cur is None:
                ranges[k.column] = Predicate("RANGE", k.column, [], k.lower, k.upper, k.lower_inclusive, k.upper_inclusive)
            else:
                recreate = True
                if k.lower is not None and (cur.lower is None or k.lower > cur.lower or
                                            (k.lower == cur.lower and not k.lower_inclusive)):
                    cur.lower, cur.lower_inclusive = k.lower, k.lower_inclusive
                if k.upper is not None and (cur.upper is None or k.upper < cur.upper or
                                            (k.upper == cur.upper and not k.upper_inclusive)):
                    cur.upper, cur.upper_inclusive = k.upper, k.upper_inclusive
        else:
            others.append(k)
    if not recreate:
        return Filter("AND", kids)
    out = others + list(ranges.values())
    return out[0] if len(out) == 1 else Filter("AND", out)


def optimize_filter(node: Optional[FilterNode]) -> Optional[FilterNode]:
    return merge_range(merge_eq_in(flatten(node)))


def filter_columns(node: Optional[FilterNode]) -> List[str]:
    out: List[str] = []

    def walk(n):
        if n is None:
            return
        if isinstance(n, Predicate):
            if n.column not in out:
                out.append(n.column)
        else:
            for c in n.children:
                walk(c)

    walk(node)
    return out


def postfix(node: Optional[FilterNode]) -> Sequence[FilterNode]:
    """Children-before-parent order (what both the C-ABI and the oracle consume)."""
    out = []

    def walk(n):
        if isinstance(n, Filter):
            for c in n.children:
                walk(c)
        out.append(n)

    if node is not None:
        walk(node)
    return out


_EXPR_TOKEN = re.compile(r"'(?:[^']|'')*'|[A-Za-z_$][\w$.]*|[0-9.][0-9.]*(?:[eE][+-]?[0-9]+)?|\S")


def is_multi_column_expression(function: str, column) -> bool:
    """SUM / AVG / MIN / MAX over an expression with two or more column leaves (DESIGN.md section 3.15) or over CASE: computed per row
    on the device, not derived; the same test as the library's (a name followed by '(' is a function, a quoted or numeric
    token a literal, any other name a column)."""
    if function not in ("SUM", "AVG", "MIN", "MAX") or not column or "(" not in column:
        return False
    if column.startswith("case("):   # CASE WHEN (DESIGN.md section 3.19) is computed per row whatever its column count
        return True
    tokens = _EXPR_TOKEN.findall(column)
    leaves = 0
    for k, t in enumerate(tokens):
        if (t[0].isalpha() or t[0] in "_$") and not (k + 1 < len(tokens) and tokens[k + 1] == "("):
            leaves += 1
    return leaves >= 2

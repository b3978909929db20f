"""Reference for FLOAT / DOUBLE columns at NaN, -0.0 and +-inf, sharing nothing with the product.

The contract it restates (DESIGN.md section 5):

* Identity is Double.doubleToLongBits (FLOAT: Float.floatToIntBits): every NaN is one value, -0.0 and 0.0 are two.
  Dictionaries, group keys, DISTINCTCOUNT and by-value merges follow it.
* Order is Double.compare / Float.compare: -inf < ... < -0.0 < 0.0 < ... < +inf < NaN.  Dictionary order, MIN / MAX,
  PERCENTILE ranks and every ORDER BY follow it.
* SUM / AVG follow IEEE: NaN when the group has a NaN row or both infinities, else +-inf when it has that infinity, else the
  exact sum within the gamma_n bound of tests/exact_ref.py.  A sum that is exactly zero is +0.0 (the reference starts at
  0.0).  NaN results are compared as "is NaN", not bit for bit.
* Predicates on a dictionary column are the oracle's (the reference's binary search of the dictionary, oracle.filter_doc_ids);
  predicates on a raw column compare each value with Java's <, > and ==, so NaN matches only NEQ / NOT_IN and 0 matches
  both zeros (restated here, raw_doc_ids).

The dictionary builder is Pinot's: unique values by bit identity, the raw bits of the first NaN seen kept as the entry,
sorted by Double.compare.  oracle.segment_builder merges -0.0 with 0.0 (np.unique), so it cannot build these columns.
"""
from __future__ import annotations

import functools
import math
import struct
from typing import Dict, List, Optional, Sequence

import numpy as np

from exact_ref import ExactSum, same_double, sum_within_bound
from oracle import segment_builder as sb

D_NAN, D_NEG_NAN = 0x7FF8000000000000, 0xFFF8000000000000
D_PAYLOAD_NAN, D_SIGNALLING_NAN = 0x7FF80000DEADBEEF, 0x7FF0000000000001
F_NAN, F_NEG_NAN, F_PAYLOAD_NAN, F_SIGNALLING_NAN = 0x7FC00000, 0xFFC00000, 0x7FC0BEEF, 0x7F800001


def double_of(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def float_of(bits: int) -> np.float32:
    return np.frombuffer(struct.pack("<I", bits), dtype=np.float32)[0]


def bits_of(x, data_type: int = sb.DOUBLE) -> int:
    if data_type == sb.FLOAT:
        return struct.unpack("<I", np.float32(x).tobytes())[0]
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def identity(x, data_type: int = sb.DOUBLE) -> int:
    """doubleToLongBits / floatToIntBits (as unsigned): NaNs collapse to the canonical NaN."""
    if math.isnan(float(x)):
        return F_NAN if data_type == sb.FLOAT else D_NAN
    return bits_of(x, data_type)


def java_compare(a: float, b: float) -> int:
    """Double.compare: numeric < / > first, then the signed doubleToLongBits (so -0.0 < 0.0 and NaN == NaN > +inf)."""
    a, b = float(a), float(b)
    if a < b:
        return -1
    if a > b:
        return 1
    ia, ib = identity(a), identity(b)
    sa = ia - (1 << 64) if ia >> 63 else ia
    sb_ = ib - (1 << 64) if ib >> 63 else ib
    return (sa > sb_) - (sa < sb_)


ORDER = functools.cmp_to_key(java_compare)


def unique_values(values: np.ndarray, data_type: int) -> list:
    """Pinot's dictionary content: one entry per identity, the first NaN's own bits, sorted by Double.compare."""
    first = {}
    for v in values:
        first.setdefault(identity(v, data_type), v)
    return sorted(first.values(), key=ORDER)


def build_dict_column(name: str, values: np.ndarray, inverted: bool = False, lib=None) -> sb.ColumnData:
    """A dictionary-encoded FLOAT / DOUBLE column as a Pinot segment stores it (sorted index when the values are sorted
    in dictionary order, an inverted index when asked)."""
    values = np.asarray(values)
    dt = sb.FLOAT if values.dtype == np.float32 else sb.DOUBLE
    entries = unique_values(values, dt)
    index = {identity(v, dt): i for i, v in enumerate(entries)}
    dict_ids = np.array([index[identity(v, dt)] for v in values], dtype=np.int32)
    card = len(entries)
    bits = sb.num_bits_per_value(card - 1)
    dict_values = np.array(entries, dtype=values.dtype)
    dbytes = np.frombuffer(dict_values.astype(sb._NP_BE[dt]).tobytes(), dtype=np.uint8).copy()
    n = len(values)
    is_sorted = bool(n > 0 and np.all(dict_ids[1:] >= dict_ids[:-1]))
    if is_sorted:
        starts = np.searchsorted(dict_ids, np.arange(card), side="left")
        ends = np.searchsorted(dict_ids, np.arange(card), side="right") - 1
        fwd = np.frombuffer(np.stack([starts, ends], axis=1).astype(">i4").tobytes(), dtype=np.uint8).copy()
    else:
        fwd = sb.pack_fixed_bits(dict_ids, bits)
    inv = lib.inverted_index_build(dict_ids, card) if inverted and not is_sorted else None
    return sb.ColumnData(name, dt, True, bits, card, is_sorted, dbytes.size // card, fwd, dbytes, inv, dict_values, dict_ids)


def sorted_rows(values: np.ndarray) -> np.ndarray:
    """`values` in Double.compare order (the row order of a column with a sorted index)."""
    return values[sorted(range(len(values)), key=lambda i: ORDER(float(values[i])))]   # indexing keeps the NaN bits


def column_values(seg: sb.SegmentData, column: str) -> np.ndarray:
    c = seg.column(column)
    if not c.has_dictionary:
        return np.asarray(c.raw_values)
    return np.asarray(c.dict_values)[np.asarray(c.dict_ids)]


# ------------------------------------------------------------------------------------------------------------ filters
def raw_matches(v, p, data_type: int) -> bool:
    """A raw value against a value-space predicate with Java's <, > and == in the column's type."""
    x = float(np.float32(v)) if data_type == sb.FLOAT else float(v)
    cast = (lambda t: float(np.float32(t))) if data_type == sb.FLOAT else float
    if p.type == "RANGE":
        if p.lower is not None and not (x >= cast(p.lower) if p.lower_inclusive else x > cast(p.lower)):
            return False
        if p.upper is not None and not (x <= cast(p.upper) if p.upper_inclusive else x < cast(p.upper)):
            return False
        return not math.isnan(x)
    hit = any(x == cast(t) for t in p.values)
    return hit if p.type in ("EQ", "IN") else not hit


def raw_doc_ids(seg: sb.SegmentData, p) -> np.ndarray:
    c = seg.column(p.column)
    return np.array([i for i, v in enumerate(c.raw_values) if raw_matches(v, p, c.data_type)], dtype=np.int64)


def doc_ids(oracle, seg: sb.SegmentData, q) -> np.ndarray:
    """The rows `q`'s filter (one predicate or none) selects: the oracle's on a dictionary column, raw_doc_ids on a raw one."""
    p = q.filter
    if p is None:
        return np.arange(seg.num_docs, dtype=np.int64)
    if getattr(p, "column", None) is not None and not seg.column(p.column).has_dictionary:
        return raw_doc_ids(seg, p)
    return oracle.filter_doc_ids(seg, q)[0].astype(np.int64)


# ------------------------------------------------------------------------------------------------------- aggregates
@functools.total_ordering
class Key:
    """A group-key value compared by identity and ordered by Double.compare (ints and strings as they are)."""
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = v

    def _id(self):
        return identity(self.v) if isinstance(self.v, float) else self.v

    def __eq__(self, o):
        return self._id() == o._id()

    def __lt__(self, o):
        return java_compare(self.v, o.v) < 0 if isinstance(self.v, float) else self.v < o.v

    def __hash__(self):
        return hash(self._id())

    def __repr__(self):
        return repr(self.v)


def float_sum(xs: Sequence[float]):
    """The SUM contract: 'nan', +-inf, or an ExactSum for the gamma_n bound."""
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return "nan"
    if math.inf in xs:
        return math.inf
    if -math.inf in xs:
        return -math.inf
    s = math.fsum(xs)
    return ExactSum("approx", s if s != 0 else 0.0, math.fsum(abs(x) for x in xs), len(xs))


def percentile(xs: Sequence[float], p: float) -> float:
    """PercentileAggregationFunction over the group's values in Double.compare order (-inf when empty)."""
    if not xs:
        return -math.inf
    n = len(xs)
    k = n - 1 if p == 100 else min(int(float(n) * float(p) / 100.0), n - 1)
    return sorted(xs, key=ORDER)[k]


def reference(oracle, segs: Sequence[sb.SegmentData], q) -> Dict[tuple, list]:
    """{(Key, ...): [per aggregation]} over the union of the segments' selected rows: COUNT int, SUM / AVG float_sum
    (AVG: with its count), MIN / MAX / PERCENTILE float, DISTINCTCOUNT frozenset of identities."""
    groups: Dict[tuple, List[int]] = {}
    cols = {}
    rows = []
    for s in segs:
        docs = doc_ids(oracle, s, q)
        names = set(q.group_by) | {a.column for a in q.aggregations if a.column}
        vals = {c: column_values(s, c)[docs] for c in names}
        for i in range(len(docs)):
            rows.append({c: (float(v[i]) if v.dtype.kind == "f" else v[i].item()) for c, v in vals.items()})
        for c in names:
            cols[c] = s.column(c).data_type
    for r, row in enumerate(rows):
        groups.setdefault(tuple(Key(row[c]) for c in q.group_by), []).append(r)
    if not q.group_by:
        groups.setdefault((), [])
    out = {}
    for key, members in groups.items():
        vals = []
        for agg in q.aggregations:
            fn = agg.function
            xs = [rows[r][agg.column] for r in members] if agg.column else []
            if fn == "COUNT":
                vals.append(len(members))
            elif fn in ("SUM", "AVG"):
                vals.append(float_sum(xs) if fn == "SUM" else (float_sum(xs), len(xs)))
            elif fn == "MIN":
                vals.append(min(xs, key=ORDER) if xs else math.inf)
            elif fn == "MAX":
                vals.append(max(xs, key=ORDER) if xs else -math.inf)
            elif fn == "DISTINCTCOUNT":
                vals.append(frozenset(identity(x, cols[agg.column]) for x in xs))
            elif fn == "PERCENTILE":
                vals.append(percentile(xs, agg.arg))
            else:
                raise ValueError(fn)
        out[key] = vals
    return out


def check_sum(got: float, want) -> bool:
    if want == "nan":
        return math.isnan(got)
    if isinstance(want, float):
        return got == want
    if want.s == 0 and want.a == 0:
        return same_double(got, 0.0)    # only zeros: +0.0, also when every row is -0.0
    return sum_within_bound(got, want)


def check_value(got: float, want: float) -> bool:
    """MIN / MAX / PERCENTILE: bit for bit (so -0.0 is not 0.0), any NaN for a NaN."""
    return math.isnan(got) if math.isnan(want) else same_double(got, float(want))


def final(fn: str, v) -> float:
    """The final value of a reference intermediate (what ORDER BY compares)."""
    if fn == "COUNT":
        return v
    if fn == "DISTINCTCOUNT":
        return len(v)
    if fn in ("SUM", "AVG"):
        s, n = (v, None) if fn == "SUM" else v
        x = math.nan if s == "nan" else s if isinstance(s, float) else float(s.s)
        return x if fn == "SUM" else (x / n if n else -math.inf)
    return float(v)


def ordered(q, table: Dict[tuple, list], items) -> List[tuple]:
    """[(key, finals)] in ORDER BY order (items: sql.resolve_order_by), ties by the key values ascending."""
    rows = sorted(((k, [final(a.function, v) for a, v in zip(q.aggregations, vals)]) for k, vals in table.items()),
                  key=lambda r: r[0])
    for kind, index, asc in reversed(items):
        if kind == "GROUP_BY":
            rows.sort(key=lambda r: r[0][index], reverse=not asc)
        else:
            rows.sort(key=lambda r: ORDER(float(r[1][index])), reverse=not asc)
    return rows

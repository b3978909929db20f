"""Exact reference for COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT, independent of the oracle's aggregation code, and the
comparator that holds the device's results to it.

The oracle accumulates SUM in Java order in a `double`, so it states parity with the reference but cannot tell an exact
integer sum from a nearly exact one; its MIN / MAX fold doubles, so it cannot tell which row won either.  Here the rows
come from the oracle's filter (pinned to the reference's goldens), the values and group keys straight from the segment's
columns, and the arithmetic is exact:

* INT columns (dictionary or raw): per-group sums in int64 (exact while rows x 2^31 < 2^63); the device must return
  `float(exact)`, the correctly rounded double, bit for bit.
* LONG, FLOAT, DOUBLE: the device sums these in double in no fixed order, so the reference keeps per group the exact sum
  S (Python int for LONG, `math.fsum` for floats), A = sum |x| and the row count n; the device's sum must lie within
  gamma_n * A of S, gamma_n = n u / (1 - n u), u = 2^-53.  That bound holds for every summation order (a LONG's
  rounding to double included) and does not depend on |S|, so cancelling values are no false alarm.
* COUNT and the AVG count: equal.
* MIN / MAX: the stored value of the group's smallest / largest row (int for INT / LONG, float for FLOAT / DOUBLE).  A
  dictionary column is ordered by its dictionary (the smallest / largest dictId, Pinot's order for every type); a raw
  column numerically.  A group without a row: +inf / -inf.  The device must return `float(value)` (round to nearest:
  LONG beyond 2^53), bit for bit.  STRING MIN / MAX come back as dictIds, not values, and are left to the oracle
  comparison.
* DISTINCTCOUNT: the set of the group's distinct values, equal.

Merged results: the reference runs over the union of the segments' rows, keyed by value (not a sum of per-segment floats).

NaN and -0.0 in FLOAT / DOUBLE columns are held by tests/float_edges_ref.py: np.unique (the test segment builder) merges
-0.0 with +0.0, so this reference is fed columns without them, and sum_within_bound takes finite sums only.
"""
from __future__ import annotations

import dataclasses
import math
import struct
from dataclasses import dataclass
from fractions import Fraction
from typing import Dict, List, Optional, Sequence

import numpy as np

from oracle import segment_builder as sb

U = Fraction(1, 1 << 53)   # unit roundoff of binary64


@dataclass(frozen=True)
class ExactSum:
    """One group's SUM / AVG argument: kind "int" (INT columns: exact is `s`, device == float(s)) or "approx" (LONG /
    FLOAT / DOUBLE: `s` the exact (LONG) or correctly rounded (floats) sum, `a` = sum |x|)."""
    kind: str
    s: object     # int (INT, LONG) or float (FLOAT, DOUBLE)
    a: object     # int or float; unused for "int"
    n: int


def gamma(n: int) -> Fraction:
    """gamma_n = n u / (1 - n u): bound on the relative error of any sum of n terms in binary64 (Higham, Lemma 3.1)."""
    assert 0 <= n and n * U < 1
    return n * U / (1 - n * U)


def _dictionary(c: sb.ColumnData) -> np.ndarray:
    if c.dict_values is not None:
        return np.asarray(c.dict_values)
    if c.data_type == sb.STRING:
        return np.frombuffer(c.dict.tobytes(), dtype=f"S{c.dict_entry_bytes}")
    return np.frombuffer(c.dict.tobytes(), dtype=sb._NP_BE[c.data_type]).astype(sb._NP_BE[c.data_type][1:])


def _dict_ids(oracle, seg: sb.SegmentData, c: sb.ColumnData, docs: np.ndarray) -> np.ndarray:
    if c.dict_ids is not None:
        return np.asarray(c.dict_ids)[docs]
    if c.is_sorted:   # (start, end) doc pairs per dictId
        starts = np.frombuffer(c.fwd.tobytes(), dtype=">i4").reshape(-1, 2)[:, 0].astype(np.int64)
        return (np.searchsorted(starts, docs, side="right") - 1).astype(np.int32)
    return oracle.read_dict_ids(c.fwd, seg.num_docs, c.bits, docs)


def column_values(oracle, seg: sb.SegmentData, column: str, docs: np.ndarray) -> np.ndarray:
    """The stored value of `column` at every doc of `docs`."""
    c = seg.column(column)
    if not c.has_dictionary:
        return np.asarray(c.raw_values)[docs]
    return _dictionary(c)[_dict_ids(oracle, seg, c, docs)]


def _key_value(v):
    return v.decode("utf-8") if isinstance(v, bytes) else v


def _exact_int_sums(values: np.ndarray, gidx: np.ndarray, groups: int) -> List[int]:
    v = values.astype(np.int64)
    # int64 accumulation is exact while no partial sum can leave int64: rows x 2^31 < 2^63
    assert len(v) < (1 << 32)
    out = np.zeros(groups, dtype=np.int64)
    np.add.at(out, gidx, v)
    return [int(x) for x in out]


def _split_u32(x: np.ndarray, gidx: np.ndarray, groups: int, signed: bool) -> List[int]:
    """Exact per-group sums of 64-bit integers: high and low 32-bit halves summed apart in int64 (exact below 2^31 rows)."""
    assert len(x) < (1 << 31)
    hi = (x >> np.int64(32)).astype(np.int64) if signed else (x >> np.uint64(32)).astype(np.int64)
    lo = (x & (0xFFFFFFFF if signed else np.uint64(0xFFFFFFFF))).astype(np.int64)
    sh, sl = np.zeros(groups, dtype=np.int64), np.zeros(groups, dtype=np.int64)
    np.add.at(sh, gidx, hi)
    np.add.at(sl, gidx, lo)
    return [(int(h) << 32) + int(l) for h, l in zip(sh, sl)]


def _long_sums(values: np.ndarray, gidx: np.ndarray, groups: int):
    v = values.astype(np.int64)
    u = v.view(np.uint64)
    mag = np.where(v < 0, (~u) + np.uint64(1), u)   # |v| as uint64 (also for INT64_MIN)
    return _split_u32(v, gidx, groups, True), _split_u32(mag, gidx, groups, False)


def _float_sums(values: np.ndarray, gidx: np.ndarray, groups: int):
    v = values.astype(np.float64)
    order = np.argsort(gidx, kind="stable")
    bounds = np.searchsorted(gidx[order], np.arange(groups + 1))
    sv = v[order]
    s = [math.fsum(sv[bounds[g]:bounds[g + 1]].tolist()) for g in range(groups)]
    a = [math.fsum(np.abs(sv[bounds[g]:bounds[g + 1]]).tolist()) for g in range(groups)]
    return s, a


def _extremes(oracle, segs, docs, column: str, sel: np.ndarray, gidx: np.ndarray, groups: int, fn: str) -> list:
    """Per group, the MIN / MAX stored value of `column` over the selected rows (+-inf: no row).
    Inside a segment the order is its dictionary's (smallest / largest dictId) or, raw, the numeric one; across segments
    the winners are compared by value."""
    pick = np.minimum if fn == "MIN" else np.maximum
    best, have = None, np.zeros(groups, dtype=bool)
    at = 0
    for s, d in zip(segs, docs):
        m = sel[at:at + len(d)]
        g = gidx[at:at + len(d)][m]
        at += len(d)
        if not len(g):
            continue
        c = s.column(column)
        present = np.zeros(groups, dtype=bool)
        present[g] = True
        some_row = np.zeros(groups, dtype=np.int64)   # the start value of a present group is one of its own rows
        some_row[g] = np.arange(len(g))
        if c.has_dictionary:
            ids = _dict_ids(oracle, s, c, d[m]).astype(np.int64)
            win = ids[some_row]
            pick.at(win, g, ids)
            v = _dictionary(c)[win]
        else:
            vals = np.asarray(c.raw_values)[d[m]]
            v = vals[some_row]
            pick.at(v, g, vals)
        if best is None:
            best = v.copy()
        else:
            both = have & present
            best[both] = pick(best[both], v[both])
            best[present & ~have] = v[present & ~have]
        have |= present
    empty = math.inf if fn == "MIN" else -math.inf
    if best is None:
        return [empty] * groups
    return [best[i].item() if have[i] else empty for i in range(groups)]


def _distinct_sets(values: np.ndarray, gidx: np.ndarray, groups: int) -> List[frozenset]:
    order = np.argsort(gidx, kind="stable")
    bounds = np.searchsorted(gidx[order], np.arange(groups + 1))
    sv = values[order]
    return [frozenset(_key_value(x) for x in np.unique(sv[bounds[g]:bounds[g + 1]]).tolist()) for g in range(groups)]


def reference(oracle, segs: Sequence[sb.SegmentData], q) -> Dict[tuple, list]:
    """{group key values: [per aggregation]} over the union of the segments' rows: COUNT -> int, SUM / AVG -> ExactSum,
    MIN / MAX -> stored value or +-inf (None for STRING), DISTINCTCOUNT -> frozenset of values.  Keys are the value tuples
    reduce_util.normalise produces."""
    docs = [oracle.filter_doc_ids(s, q)[0].astype(np.int64) for s in segs]
    # group index of every matched row: per column, values -> codes over the union, then mixed radix
    if q.group_by:
        code = np.zeros(sum(len(d) for d in docs), dtype=np.int64)
        uniqs, mult = [], 1
        for col in q.group_by:
            vals = np.concatenate([column_values(oracle, s, col, d) for s, d in zip(segs, docs)])
            uniq, inv = np.unique(vals, return_inverse=True)
            code += inv.reshape(-1).astype(np.int64) * mult
            uniqs.append(uniq)
            mult *= max(len(uniq), 1)
            assert mult < (1 << 62)
        gcodes, gidx = np.unique(code, return_inverse=True)
        gidx = gidx.reshape(-1)
        keys = []
        for c in gcodes.tolist():
            key = []
            for uniq in uniqs:
                c, i = divmod(c, len(uniq))
                key.append(_key_value(uniq[i].item()))
            keys.append(tuple(key))
    else:
        gidx = np.zeros(sum(len(d) for d in docs), dtype=np.int64)
        keys = [()]
    groups = len(keys)
    cols = [[None] * groups for _ in q.aggregations]
    for a, agg in enumerate(q.aggregations):
        dt = segs[0].column(agg.column).data_type if agg.column is not None else None
        if agg.function not in ("COUNT", "SUM", "AVG", "MIN", "MAX", "DISTINCTCOUNT"):
            continue
        if agg.function in ("MIN", "MAX") and dt == sb.STRING:
            continue
        if agg.filter is not None:   # FILTER (WHERE ...): the main filter's rows that the clause matches too
            cq = dataclasses.replace(q, filter=agg.filter)
            sel = np.concatenate([np.isin(d, oracle.filter_doc_ids(s, cq)[0]) for s, d in zip(segs, docs)])
        else:
            sel = np.ones(len(gidx), dtype=bool)
        if agg.function in ("MIN", "MAX"):
            cols[a] = _extremes(oracle, segs, docs, agg.column, sel, gidx, groups, agg.function)
            continue
        g = gidx[sel]
        counts = [int(x) for x in np.bincount(g, minlength=groups)]
        if agg.function == "COUNT":
            cols[a] = counts
            continue
        vals = np.concatenate([column_values(oracle, s, agg.column, d) for s, d in zip(segs, docs)])[sel]
        if agg.function == "DISTINCTCOUNT":
            cols[a] = _distinct_sets(vals, g, groups)
            continue
        if dt == sb.INT:
            cols[a] = [ExactSum("int", s, None, n) for s, n in zip(_exact_int_sums(vals, g, groups), counts)]
        elif dt == sb.LONG:
            s, m = _long_sums(vals, g, groups)
            cols[a] = [ExactSum("approx", x, y, n) for x, y, n in zip(s, m, counts)]
        else:
            s, m = _float_sums(vals, g, groups)
            cols[a] = [ExactSum("approx", x, y, n) for x, y, n in zip(s, m, counts)]
    return {key: [cols[a][i] for a in range(len(q.aggregations))] for i, key in enumerate(keys)}


def sum_within_bound(got: float, ref: ExactSum) -> bool:
    """|got - S| <= gamma_n * A, evaluated in exact rational arithmetic.  For floats S is the correctly rounded sum: its own
    error (<= u A) fits in gamma_n - gamma_{n-1} >= u, since n values take n - 1 additions."""
    if not math.isfinite(got):
        return False
    a = Fraction(ref.a) if isinstance(ref.a, int) else Fraction(math.nextafter(ref.a, math.inf))
    return abs(Fraction(got) - Fraction(ref.s)) <= gamma(ref.n) * a


def check_sum(got: float, ref: ExactSum) -> bool:
    if ref.kind == "int":
        return got == float(ref.s)   # float(int) rounds to nearest, ties to even: what (double)int64 does
    return sum_within_bound(got, ref)


def same_double(got: float, ref: float) -> bool:
    """Bit-for-bit equality of two doubles (0.0 and -0.0 differ, an infinity only equals itself)."""
    return struct.pack("<d", got) == struct.pack("<d", ref)


def assert_exact(q, got: Dict[tuple, list], ref: Dict[tuple, list], what: str = "") -> None:
    """Per aggregation: COUNT equal; SUM / AVG over INT bit-exact (AVG: and its count equal); over LONG / FLOAT / DOUBLE
    within gamma_n * A of the exact sum; MIN / MAX bit-exact; DISTINCTCOUNT the same set of values."""
    assert set(got) == set(ref), f"{what}: group keys differ from the exact reference: {len(got)} vs {len(ref)}"
    for key, rv in ref.items():
        gv = got[key]
        for a, agg in enumerate(q.aggregations):
            fn, r = agg.function, rv[a]
            if fn in ("COUNT", "DISTINCTCOUNT"):
                assert gv[a] == r, (what, key, fn, agg.column, gv[a], r)
            elif fn in ("SUM", "AVG"):
                s = gv[a] if fn == "SUM" else gv[a][0]
                if fn == "AVG":
                    assert gv[a][1] == r.n, (what, key, "AVG count", gv[a][1], r.n)
                assert check_sum(s, r), (what, key, fn, agg.column, r.kind, repr(s), r.s, r.n)
            elif fn in ("MIN", "MAX") and r is not None:
                assert same_double(gv[a], float(r)), (what, key, fn, agg.column, float(gv[a]).hex(), float(r).hex(), r)


def check_exact(oracle, segs: Sequence[sb.SegmentData], q, got: Dict[tuple, list], what: str = "") -> Dict[tuple, list]:
    ref = reference(oracle, segs, q)
    assert_exact(q, got, ref, what)
    return ref

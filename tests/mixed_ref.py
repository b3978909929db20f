"""One reference for every aggregation function in any query, so that queries mixing the families can be held to it.

This module only dispatches: the rows, values and rules come from the per-family modules, and nothing here looks at the
product beyond the result block it is handed.

* Groups: exact_ref.reference (the doc set of tests/filter_ref.py, keyed by the group-by columns' values; aggregation only:
  the one key ()).  Each function's matched values per group come from percentile_ref.group_values, expressions from
  expr_ref.row_values and FIRST/LASTWITHTIME from withtime_ref.withtime.  A FILTER (WHERE ...) clause adds its
  predicate to the query's filter for that aggregation alone.
* Final values: COUNT / SUM / AVG / MIN / MAX by exact_ref, DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG by
  distinct_value_ref, PERCENTILE by percentile_ref, VAR / STDDEV by variance_ref, DISTINCTCOUNTHLL by hll_ref,
  expression aggregations by expr_ref.

Comparison contract:

* bit for bit: COUNT, SUM / AVG over INT columns (and the AVG count), MIN, MAX (not over STRING columns: the plan maker
  refuses them, and reference() raises), DISTINCTCOUNT (the count and the set of
  values), DISTINCTSUM, DISTINCTAVG, PERCENTILE (and its row count), DISTINCTCOUNTHLL, FIRST/LASTWITHTIME (time, value
  and dictId), expression MIN / MAX;
* within gamma_n * sum |x| of the exact sum: SUM / AVG over LONG, FLOAT and DOUBLE columns and over expressions (their
  atomics add in any order);
* within one ulp of the exact rational: VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP (their row count exactly)."""
from __future__ import annotations

import dataclasses
import math
import struct
from typing import Callable, Dict, List, Optional, Sequence

import exact_ref
import hll_ref
import numpy as np
import variance_ref
from distinct_value_ref import distinct_values, ref_final
from expr_ref import check_value, order_key, row_values
from oracle import segment_builder as sb
from percentile_ref import group_values, percentile, pick
from pinot_b200.query import Filter, value_key
from withtime_ref import withtime

DISTINCT_SET = ("DISTINCTCOUNT", "DISTINCTSUM", "DISTINCTAVG")
WITHTIME = ("FIRSTWITHTIME", "LASTWITHTIME")
TYPE_NAMES = {sb.INT: "INT", sb.LONG: "LONG", sb.FLOAT: "FLOAT", sb.DOUBLE: "DOUBLE", sb.STRING: "STRING"}


def is_expression(agg) -> bool:
    return "(" in (agg.column or "")


def _plain(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _bits(x: float) -> bytes:
    return struct.pack("<d", x)


def summed_in_any_order(segs, agg) -> bool:
    """SUM / AVG whose result depends on the order of its additions: floating and expression sums."""
    if agg.function not in ("SUM", "AVG"):
        return False
    return is_expression(agg) or segs[0].column(agg.column).data_type != sb.INT


def _filter_of(q, agg):
    if agg.filter is None:
        return q.filter
    return agg.filter if q.filter is None else Filter("AND", [q.filter, agg.filter])


@dataclasses.dataclass
class Want:
    """The reference state of one aggregation in one group: `kind` names the rule that checks it."""
    kind: str
    value: object
    extra: object = None
    memo: dict = dataclasses.field(default_factory=dict)   # DISTINCTCOUNTHLL estimates by log2m, computed once


def reference(oracle, segs: Sequence, q) -> Dict[tuple, List[Want]]:
    """{group key values: [Want per aggregation]} over the union of the segments' rows."""
    # exact_ref keys the groups and answers COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT over plain columns; the other
    # aggregations stand in as COUNT(*) there
    plain = [a if (a.function in ("COUNT", "SUM", "AVG", "MIN", "MAX") and not is_expression(a)) else
             dataclasses.replace(a, function="COUNT", column=None, filter=None) for a in q.aggregations]
    base = exact_ref.reference(oracle, segs, dataclasses.replace(q, aggregations=plain))
    cols = []
    for a, agg in enumerate(q.aggregations):
        fn, flt = agg.function, _filter_of(q, agg)
        if is_expression(agg):
            rows = row_values(oracle, segs, flt, q.group_by, agg.column)
            cols.append({k: Want("expr", rows.get(k, [])) for k in base})
        elif fn in ("MIN", "MAX") and segs[0].column(agg.column).data_type == sb.STRING:
            # the plan maker refuses them ("aggregation over STRING column"): no block of this layer holds one to check
            raise ValueError(f"{fn} over STRING column {agg.column} is not answered")
        elif fn in ("COUNT", "SUM", "AVG", "MIN", "MAX"):
            cols.append({k: Want("exact", v[a]) for k, v in base.items()})
        elif fn in WITHTIME:
            won = withtime(oracle, segs, flt, q.group_by, fn, agg.column, agg.time_column)
            cols.append({k: Want("withtime", won.get(k)) for k in base})
        else:
            values = group_values(oracle, segs, flt, q.group_by, agg.column)
            dtype = TYPE_NAMES[segs[0].column(agg.column).data_type]
            cols.append({k: Want(fn, values.get(k, np.zeros(0)), dtype) for k in base})
    return {k: [c[k] for c in cols] for k in base}


def _hll(want: Want, log2m) -> int:
    if log2m not in want.memo:
        members = {value_key(_plain(v)) for v in want.value}
        want.memo[log2m] = hll_ref.hll([float(v) if isinstance(v, float) else v for v in members], int(log2m), want.extra)
    return want.memo[log2m]


def final(agg, want: Want) -> float:
    """The final value of an aggregation as ORDER BY and HAVING compare it (AVG = sum / count, -inf when empty)."""
    fn, v = agg.function, want.value
    if want.kind == "expr":
        if fn in ("SUM", "AVG"):
            raise ValueError("expression sums have no exact final value")
        return min(v, key=order_key) if fn == "MIN" and v else max(v, key=order_key) if v else \
            (math.inf if fn == "MIN" else -math.inf)
    if want.kind == "exact":
        if fn == "COUNT":
            return float(v)
        if fn in ("SUM", "AVG"):
            if v.kind != "int":
                raise ValueError("floating sums have no exact final value")
            return float(v.s) if fn == "SUM" else (v.s / v.n if v.n else -math.inf)
        return float(v)
    if want.kind == "withtime":
        return -math.inf if v is None else float(v[1])
    if fn in DISTINCT_SET:
        return ref_final(fn, v)
    if fn == "PERCENTILE":
        return percentile(v, agg.arg)
    if fn in variance_ref.FUNCTIONS:
        return variance_ref.final(fn, variance_ref.exact_sums(v))
    if fn == "DISTINCTCOUNTHLL":
        return float(_hll(want, agg.arg))
    raise ValueError(fn)


def check_one(agg, want: Want, d: float, n: int, dict_id: Optional[int], members, decode: Callable, what: str):
    """One aggregation of one group: d its double, n its long, dict_id its dictId (PERCENTILE, WITHTIME) and members the
    dictIds of its set (DISTINCTCOUNT, None when the block has none).  Returns what must not change with the aggregation's
    position in the query (None: an order-dependent sum, held to its bound only)."""
    fn, v = agg.function, want.value
    if want.kind == "expr":
        assert check_value(fn, d, n, v), f"{what}: {fn}({agg.column}) = {d!r} ({n}) over {len(v)} rows"
        return None if fn in ("SUM", "AVG") else _bits(d)
    if want.kind == "exact":
        if fn == "COUNT":
            assert n == v, f"{what}: COUNT {n} != {v}"
            return n
        if fn in ("SUM", "AVG"):
            assert exact_ref.check_sum(d, v), f"{what}: {fn}({agg.column}) {d!r} vs exact {v.s} over {v.n} rows ({v.kind})"
            if fn == "AVG":
                assert n == v.n, f"{what}: AVG count {n} != {v.n}"
            return None if v.kind != "int" else (_bits(d), n)
        assert exact_ref.same_double(d, float(v)), f"{what}: {fn}({agg.column}) {d!r} != {float(v)!r}"
        return _bits(d)
    if want.kind == "withtime":
        if v is None:
            assert dict_id == -1 and d == -math.inf, f"{what}: {fn} expected no row, got {d!r} id {dict_id}"
            return (_bits(d), dict_id)
        assert n == v[0], f"{what}: {fn} time {n} != {v[0]}"
        assert _plain(decode(agg.column, dict_id)) == v[1], f"{what}: {fn} value of id {dict_id} != {v[1]!r}"
        if not isinstance(v[1], str):
            assert exact_ref.same_double(d, float(v[1])), f"{what}: {fn} double {d!r} != {v[1]!r}"
        return (_bits(d), n, dict_id)
    if fn in DISTINCT_SET:
        want_d = ref_final(fn, v)
        got_d = float(n) if fn == "DISTINCTCOUNT" else d
        assert _bits(got_d) == _bits(want_d), f"{what}: {fn}({agg.column}) {got_d!r} != {want_d!r}"
        assert n == len(distinct_values(v)), f"{what}: {fn}({agg.column}) count {n} != {len(distinct_values(v))}"
        if members is not None:
            got = {value_key(_plain(decode(agg.column, int(i)))) for i in members}
            assert got == {value_key(_plain(x)) for x in v}, f"{what}: {fn}({agg.column}) members differ"
        return (_bits(got_d), n)
    if fn == "PERCENTILE":
        want_d = percentile(v, agg.arg)
        assert _bits(d) == _bits(want_d), f"{what}: PERCENTILE({agg.column}, {agg.arg:g}) {d!r} != {want_d!r}"
        assert n == len(v), f"{what}: PERCENTILE row count {n} != {len(v)}"
        p = pick(v, agg.arg)
        if p is None:
            assert dict_id == -1, what
        else:
            assert _plain(decode(agg.column, dict_id)) == _plain(p), f"{what}: PERCENTILE dictId {dict_id} is not {p!r}"
        return (_bits(d), n, dict_id)
    if fn in variance_ref.FUNCTIONS:
        sums = variance_ref.exact_sums(v)
        assert variance_ref.within_one_ulp(d, fn, sums), f"{what}: {fn}({agg.column}) {d!r} vs {variance_ref.final(fn, sums)!r}"
        assert n == sums[0], f"{what}: {fn} row count {n} != {sums[0]}"
        return (_bits(d), n)
    if fn == "DISTINCTCOUNTHLL":
        want_n = _hll(want, agg.arg)
        assert n == want_n and d == float(want_n), f"{what}: DISTINCTCOUNTHLL({agg.column}, {agg.arg}) {n} / {d!r} != {want_n}"
        return n
    raise ValueError(fn)


def block_rows(q, b, decode: Callable) -> List[tuple]:
    """The group key values of every row of block b, in the block's order (aggregation only: [()])."""
    if b.num_groups < 0:
        return [()]
    return [tuple(_plain(decode(c, int(b.keys[g][j]))) for j, c in enumerate(q.group_by)) for g in range(b.num_groups)]


def check_block(q, b, ref: Dict[tuple, List[Want]], decode: Callable, what: str, all_groups: bool = True) -> Dict[tuple, list]:
    """Every aggregation of every row of block b against the reference; decode(column, id) gives the value of a dictId of
    the block (group keys, set members, selected rows).  all_groups: the block holds every reference group (no ORDER BY
    trim, no HAVING).  Returns {key: [position-independent value per aggregation]}."""
    keys = block_rows(q, b, decode)
    assert len(set(keys)) == len(keys), f"{what}: a group key twice"
    if all_groups:
        assert set(keys) == set(ref), f"{what}: groups differ: {len(keys)} vs {len(ref)}"
    else:
        assert set(keys) <= set(ref), f"{what}: groups the reference does not have"
    out = {}
    for g, key in enumerate(keys):
        row = []
        for a, agg in enumerate(q.aggregations):
            members = b.distinct.get((a, g)) if agg.function == "DISTINCTCOUNT" else None
            row.append(check_one(agg, ref[key][a], float(b.doubles[a][g]), int(b.longs[a][g]), int(b.dict_ids[a][g]), members,
                                 decode, f"{what} a={a} {agg} key={key}"))
        out[key] = row
    return out

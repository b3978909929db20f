"""Command line face of the path: load Pinot segment directories into HBM and run one aggregation / group-by query on them.

    python -m pinot_b200.cli --segment-dir /data/myTable_0 --segment-dir /data/myTable_1 \\
        "SELECT SUM(m), COUNT(*) FROM myTable WHERE d > 10 GROUP BY k LIMIT 20"

What happens: ``pb200h_segment_load_dir`` per directory (v1 file-per-index or v3 columns.psf + index_map, raw columns decoded
and dictionary-encoded at load, star-trees attached), ``pb200h_execute`` over all segments in one submission, then -- what the
reference's combine + broker reduce do, in a few lines of Python -- the per-segment results blocks are merged by key VALUES
(``AggregationFunction.merge``), final results extracted (AVG = sum / count, DISTINCTCOUNT = set size, DISTINCTSUM /
DISTINCTAVG = the set's exact sum / mean rounded once, DISTINCTCOUNTHLL = the set's estimate), filtered by HAVING,
expressions over aggregations computed, ordered, and the first LIMIT rows printed.  With ``--merge-on-device`` the segments are first bound to one dictionary domain
and combined on the GPU, where HAVING, ORDER BY and the trim run too.

Needs a GPU: the product has no CPU fallback.  Queries outside the accelerated set exit with the library's message (a Pinot
server would run the stock operator for them)."""
from __future__ import annotations

import argparse
import json
import sys
from typing import Dict, List


def merge_blocks(query, segments, blocks) -> Dict[tuple, list]:
    """{key values: [intermediate per aggregation]} over all blocks: COUNT -> int, SUM / MIN / MAX -> float,
    AVG -> (sum, count), DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG -> set of values, DISTINCTCOUNTHLL -> query.HllSet of
    values, or its final estimate for a block merged on the device, PERCENTILE -> (p, {value: count}) from the per-segment
    histograms, or its final float for a block merged on the device, VAR / STDDEV -> exact (n, sum v, sum v^2) from the
    blocks' moments, each shifted from its own grid (c, e) to values, or the final float of a block merged on the device,
    FIRST/LASTWITHTIME -> (time value, data value) of the winning row or None for an empty block (query.withtime_pick: ties
    go to the later segment for LAST, to the earlier one for FIRST)
    (GroupByCombineOperator / AggregationFunction.merge).  Float keys, set members and histogram values are compared by
    identity (query.ValueKey: one NaN, -0.0 apart from 0.0) and MIN / MAX merge in Double.compare order, as the reference's
    Double.equals / doubleToLongBits keyed tables and its dictionary order do."""
    from .query import (DISTINCT_SET_FUNCTIONS, MOMENT_FUNCTIONS, WITHTIME_FUNCTIONS, HllSet, merge_moments, value_key, value_order,
                        withtime_pick)
    out: Dict[tuple, list] = {}
    for seg, b in zip(segments, blocks):
        rows = 1 if b.num_groups < 0 else b.num_groups
        for g in range(rows):
            key = () if b.num_groups < 0 else tuple(value_key(seg.dictionary_value(c, int(b.keys[g, j]))) for j, c in enumerate(query.group_by))
            vals = []
            for a, agg in enumerate(query.aggregations):
                fn = agg.function
                if fn == "COUNT":
                    vals.append(int(b.longs[a][g]))
                elif fn == "AVG":
                    vals.append((float(b.doubles[a][g]), int(b.longs[a][g])))
                elif fn in DISTINCT_SET_FUNCTIONS:
                    vals.append({value_key(seg.dictionary_value(agg.column, int(d))) for d in b.distinct[(a, g)]})
                elif fn == "DISTINCTCOUNTHLL":
                    if (a, g) in b.distinct:
                        vals.append(HllSet((value_key(seg.dictionary_value(agg.column, int(d))) for d in b.distinct[(a, g)]),
                                           seg.column_info(agg.column)["data_type"]))
                    else:
                        vals.append(int(b.longs[a][g]))
                elif fn == "PERCENTILE" and (a, g) in b.histograms:
                    ids, counts = b.histograms[(a, g)]
                    hist: Dict[float, int] = {}
                    for d, c in zip(ids, counts):
                        v = value_key(float(seg.dictionary_value(agg.column, int(d))))
                        hist[v] = hist.get(v, 0) + int(c)
                    vals.append((agg.arg, hist))
                elif fn in MOMENT_FUNCTIONS and (a, g) in b.moments:
                    vals.append(merge_moments([b.moments[(a, g)]]))
                elif fn in WITHTIME_FUNCTIONS:
                    vals.append(b.withtime(a, g, seg, agg.column))
                else:
                    vals.append(float(b.doubles[a][g]))
            cur = out.get(key)
            if cur is None:
                out[key] = vals
                continue
            for a, agg in enumerate(query.aggregations):
                fn = agg.function
                if fn in ("COUNT", "SUM"):
                    cur[a] += vals[a]
                elif fn == "MIN":
                    cur[a] = min(cur[a], vals[a], key=value_order)
                elif fn == "MAX":
                    cur[a] = max(cur[a], vals[a], key=value_order)
                elif fn == "AVG":
                    cur[a] = (cur[a][0] + vals[a][0], cur[a][1] + vals[a][1])
                elif fn == "PERCENTILE" and isinstance(cur[a], tuple):
                    for v, c in vals[a][1].items():
                        cur[a][1][v] = cur[a][1].get(v, 0) + c
                elif fn in MOMENT_FUNCTIONS and isinstance(cur[a], tuple):
                    cur[a] = tuple(x + y for x, y in zip(cur[a], vals[a]))
                elif fn in WITHTIME_FUNCTIONS:
                    cur[a] = withtime_pick(fn, cur[a], vals[a])
                else:
                    cur[a] |= vals[a]
    return out


def output_columns(query) -> List[tuple]:
    """(header, position) of each printed column; positions index a row of key values, then the final value of every
    aggregation, then the value of every post-aggregation expression.  A query with expressions over aggregations prints
    its SELECT list in its order; the others print the GROUP BY columns, then their aggregations.  Hidden aggregations
    (named only in HAVING or in expressions) are never printed."""
    k, m = len(query.group_by), len(query.aggregations)
    if query.post_aggregations:
        at = {"COLUMN": lambda c: query.group_by.index(c), "AGG": lambda a: k + a, "POST": lambda i: k + m + i}
        names = {"COLUMN": str, "AGG": lambda a: str(query.aggregations[a]), "POST": lambda i: str(query.post_aggregations[i])}
        return [(names[kind](x), at[kind](x)) for kind, x in query.select]
    return ([(c, j) for j, c in enumerate(query.group_by)] +
            [(str(a), k + j) for j, a in enumerate(query.aggregations) if not a.hidden])


def final_rows(query, table: Dict[tuple, list]) -> List[list]:
    """Broker-side extraction of final results + HAVING + ORDER BY + LIMIT.  HAVING keeps the rows whose final values pass
    it (Java's comparisons: query.having_eval).  Expressions over aggregations are computed from the final values as
    Python floats, one IEEE-754 operation per operator (query.post_eval).  ORDER BY compares final values (AVG = sum /
    count, DISTINCTCOUNT = set size) or expression values and breaks ties by the key values ascending, in GROUP BY column
    order -- the library's order.  Without ORDER BY Pinot returns an arbitrary LIMIT-sized subset; here the rows are sorted
    by key to make the output stable.  Rows hold the columns of output_columns."""
    from .query import (DISTINCT_SET_FUNCTIONS, MOMENT_FUNCTIONS, distinct_final, having_eval, hll_final, moments_final, percentile_of_counts,
                        post_eval, value_order)
    from .sql import resolve_having, resolve_order_by
    items = resolve_order_by(query) if query.is_group_by else []
    having = resolve_having(query)
    rows = []
    keys = sorted(table, key=lambda k: tuple(value_order(x) for x in k)) if items else sorted(table, key=lambda k: tuple(str(x) for x in k))
    for key in keys:
        vals = []
        for agg, v in zip(query.aggregations, table[key]):
            if agg.function == "AVG":
                vals.append(v[0] / v[1] if v[1] else float("-inf"))
            elif agg.function in DISTINCT_SET_FUNCTIONS:
                vals.append(distinct_final(agg.function, v))
            elif agg.function == "DISTINCTCOUNTHLL":
                vals.append(hll_final(v, agg.arg, v.data_type) if isinstance(v, set) else v)
            elif agg.function == "PERCENTILE" and isinstance(v, tuple):
                vals.append(percentile_of_counts(v))
            elif agg.function in MOMENT_FUNCTIONS and isinstance(v, tuple):
                vals.append(moments_final(agg.function, v))
            elif agg.function in ("FIRSTWITHTIME", "LASTWITHTIME"):
                vals.append(float("-inf") if v is None else v[1])
            else:
                vals.append(v)
        # HAVING compares numbers; a STRING FIRST/LASTWITHTIME value is never one of its operands (sql.resolve_having
        # refuses that), so it stands in as -inf, the value the device compares for it when empty
        if having and not having_eval(having, [float("-inf") if isinstance(x, (bytes, str)) else float(x) for x in vals]):
            continue
        posts = [post_eval(p.program, lambda a: float(vals[a])) for p in query.post_aggregations]
        rows.append(list(key) + vals + posts)
    k, m = len(query.group_by), len(query.aggregations)
    for kind, index, asc in reversed(items):  # stable passes, last item first
        col = index if kind == "GROUP_BY" else k + index if kind == "AGG" else k + m + index
        rows.sort(key=lambda r: value_order(r[col]), reverse=not asc)
    shown = [c for _, c in output_columns(query)]
    return [[r[c] for c in shown] for r in rows[: query.limit]]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m pinot_b200.cli", description=__doc__.split("\n\n")[0])
    ap.add_argument("sql")
    ap.add_argument("--segment-dir", action="append", required=True, help="a Pinot segment directory (repeatable)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--merge-on-device", action="store_true", help="bind the segments to one dictionary domain and combine on the GPU")
    ap.add_argument("--num-groups-limit", type=int, default=100_000)
    ap.add_argument("--json", action="store_true", help="print one JSON object instead of a table")
    ap.add_argument("--star-tree", action="append", default=[], metavar="JSON",
                    help="a StarTreeIndexConfig (an entry of the table config's starTreeIndexConfigs): build that tree on "
                         "the device on every loaded segment (repeatable)")
    args = ap.parse_args(argv)
    from .plan_maker import parse_star_tree_config
    try:
        args.star_tree = [parse_star_tree_config(c) for c in args.star_tree]
    except ValueError as e:
        ap.error(str(e))

    from . import sql
    from ._lib import Pb200Error
    from .plan_maker import B200Context, B200PlanMaker, DictionaryDomain
    from .query import functions_where, is_multi_column_expression

    if sql.is_distinct(args.sql):
        return _distinct(args, sql.parse_distinct(args.sql))
    if sql.is_selection(args.sql):
        return _selection(args, sql.parse_selection(args.sql))
    query = sql.parse(args.sql, num_groups_limit=args.num_groups_limit)
    ctx = B200Context(args.device)
    segments, domain = [], None
    try:
        for d in args.segment_dir:
            segments.append(_load(ctx, d, args.star_tree))
        pm = B200PlanMaker(ctx)
        try:
            if args.merge_on_device and len(segments) > 1:
                cols = list(dict.fromkeys(list(query.group_by) + [a.column for a in query.aggregations
                                                                  if a.column and not is_multi_column_expression(a.function, a.column)
                                                                  and a.function in functions_where(lambda f: f.dict_ids or f.arg == "time")]
                                           + [a.time_column for a in query.aggregations if a.time_column and "(" not in a.time_column]))
                if cols:
                    domain = DictionaryDomain.build(ctx, segments, cols)
                    for s in segments:
                        s.bind_domain(domain)
                blocks = pm.execute_segments(segments, query, merge=True)
                table = merge_blocks(query, segments[:1], blocks)
            else:
                blocks = pm.execute_segments(segments, query)
                table = merge_blocks(query, segments, blocks)
        except Pb200Error as e:
            sys.stderr.write(f"{e}\n")
            return 2
        rows = final_rows(query, table)
        names = [name for name, _ in output_columns(query)]
        stats = {"numDocsScanned": sum(b.stats.num_docs_scanned for b in blocks), "totalDocs": sum(s.num_docs for s in segments),
                 "numSegments": len(segments), "deviceMs": round(sum(b.device_ms for b in blocks[:1]), 4),
                 "operators": sorted({b.operator_kind for b in blocks})}
        if args.json:
            print(json.dumps({"columns": names, "rows": rows, "stats": stats}, default=str))
        else:
            print("\t".join(names))
            for r in rows:
                print("\t".join(str(x) for x in r))
            print(f"-- {json.dumps(stats)}", file=sys.stderr)
        return 0
    finally:
        blocks = None
        for s in segments:
            s.destroy()
        if domain is not None:
            domain.release()
        ctx.close()


def _load(ctx, index_dir, star_trees):
    """A segment directory in HBM, with the configured star-trees built on the device."""
    from .plan_maker import IndexSegment
    seg = IndexSegment.load(ctx, index_dir)
    try:
        for cfg in star_trees:
            seg.build_star_tree(**cfg)
    except BaseException:
        seg.destroy()
        raise
    return seg


def _selection(args, query) -> int:
    """SELECT columns ... LIMIT n: one device submission, segments taken in the order given (their dictionaries may
    differ: values are decoded per row's segment)."""
    from ._lib import Pb200Error
    from .plan_maker import B200Context, B200PlanMaker

    ctx = B200Context(args.device)
    segments = []
    try:
        for d in args.segment_dir:
            segments.append(_load(ctx, d, args.star_tree))
        try:
            block = B200PlanMaker(ctx).execute_selection(segments, query, merge=True)
        except Pb200Error as e:
            sys.stderr.write(f"{e}\n")
            return 2
        rows = [[c[i].item() if hasattr(c[i], "item") else c[i] for c in block.columns] for i in range(block.num_rows)]
        stats = {"numDocsScanned": block.stats.num_docs_scanned, "totalDocs": sum(s.num_docs for s in segments),
                 "numSegments": len(segments), "deviceMs": round(block.device_ms, 4), "operators": ["SELECTION"]}
        if args.json:
            print(json.dumps({"columns": block.names, "rows": rows, "stats": stats}, default=str))
        else:
            print("\t".join(block.names))
            for r in rows:
                print("\t".join(str(x) for x in r))
            print(f"-- {json.dumps(stats)}", file=sys.stderr)
        return 0
    finally:
        for s in segments:
            s.destroy()
        ctx.close()


def _distinct(args, query) -> int:
    """SELECT DISTINCT columns ... LIMIT n.  --merge-on-device: the segments are bound to one domain over the DISTINCT
    columns and answered in one merged call; otherwise one per-segment call, merged by value (merge_distinct_blocks)."""
    from ._lib import Pb200Error
    from .plan_maker import B200Context, B200PlanMaker, DictionaryDomain, merge_distinct_blocks

    ctx = B200Context(args.device)
    segments, domain = [], None
    try:
        for d in args.segment_dir:
            segments.append(_load(ctx, d, args.star_tree))
        pm = B200PlanMaker(ctx)
        try:
            if args.merge_on_device and len(segments) > 1:
                domain = DictionaryDomain.build(ctx, segments, list(dict.fromkeys(query.columns)))
                for s in segments:
                    s.bind_domain(domain)
                block = pm.execute_distinct(segments, query, merge=True)
            else:
                block = merge_distinct_blocks(pm.execute_distinct(segments, query), query.order_by, query.limit)
        except Pb200Error as e:
            sys.stderr.write(f"{e}\n")
            return 2
        rows = [[c[i].item() if hasattr(c[i], "item") else c[i] for c in block.columns] for i in range(block.num_rows)]
        stats = {"numDocsScanned": block.stats.num_docs_scanned, "totalDocs": sum(s.num_docs for s in segments),
                 "numSegments": len(segments), "deviceMs": round(block.device_ms, 4), "operators": ["DISTINCT"]}
        if args.json:
            print(json.dumps({"columns": block.names, "rows": rows, "stats": stats}, default=str))
        else:
            print("\t".join(block.names))
            for r in rows:
                print("\t".join(str(x) for x in r))
            print(f"-- {json.dumps(stats)}", file=sys.stderr)
        return 0
    finally:
        block = None
        for s in segments:
            s.destroy()
        if domain is not None:
            domain.release()
        ctx.close()


if __name__ == "__main__":
    sys.exit(main())

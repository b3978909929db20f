#!/usr/bin/env python
"""What DISTINCT queries cost on ONE GPU, on bench.py's table (8 segments x 100 M rows, c0..c7 of cardinality 10 ..
1 000 000, synthetic, resident in HBM), every segment in one merged submission (the synthetic segments share one
dictionary per column, which is what binding them to a domain gives):

    SELECT DISTINCT c3 FROM benchTable WHERE c6 > K LIMIT 10                     (the prefix route)
    SELECT DISTINCT c3 FROM benchTable WHERE c6 > K ORDER BY c3 DESC LIMIT 10
    SELECT DISTINCT c0 FROM benchTable WHERE c6 > K LIMIT 10                     (10 values: every SM hits the same entries)
    SELECT DISTINCT c1, c3 FROM benchTable WHERE c6 > K ORDER BY c1, c3 LIMIT 100   (1 M key space)
    SELECT DISTINCT c6 FROM benchTable WHERE c6 > K ORDER BY c6 LIMIT 1000       (1 M values)

at 10 % and 1 % selectivity, each next to the equivalent GROUP BY ... COUNT(*) (same filter, same keys).  Per query:
step ms (host clock around the call, which ends in a device synchronisation), device ms (DISTINCT: scan launches + table
builds; GROUP BY: the scan), the scan alone (the same filter as a selection ORDER BY ... LIMIT 0, which scans every doc:
build ms = device ms - scan ms for the shapes that scan every doc), extract ms (pb200_last_phases "extract"), rows and
docs scanned; plus the card's name and power limit, read in the same run.  Prints one JSON object.

    python tests/workloads/run_distinct.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_distinct.py --dry-run     # no GPU: the queries and table shape it would run
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

COLUMNS = ["c0", "c1", "c3", "c6"]


def query_texts(selectivity: float):
    """{shape: (DISTINCT text, GROUP BY text)}"""
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k}"
    return {"c3 limit 10": (f"SELECT DISTINCT c3 {w} LIMIT 10", f"SELECT COUNT(*) {w} GROUP BY c3 LIMIT 10"),
            "c3 order by desc limit 10": (f"SELECT DISTINCT c3 {w} ORDER BY c3 DESC LIMIT 10",
                                          f"SELECT COUNT(*) {w} GROUP BY c3 ORDER BY c3 DESC LIMIT 10"),
            "c0 limit 10": (f"SELECT DISTINCT c0 {w} LIMIT 10", f"SELECT COUNT(*) {w} GROUP BY c0 LIMIT 10"),
            "c1, c3 order by limit 100": (f"SELECT DISTINCT c1, c3 {w} ORDER BY c1, c3 LIMIT 100",
                                          f"SELECT COUNT(*) {w} GROUP BY c1, c3 ORDER BY c1, c3 LIMIT 100"),
            "c6 order by limit 1000": (f"SELECT DISTINCT c6 {w} ORDER BY c6 LIMIT 1000",
                                       f"SELECT COUNT(*) {w} GROUP BY c6 ORDER BY c6 LIMIT 1000")}


def timed(run, steps):
    for _ in range(2):
        run()
    total, out = 0.0, None
    dev = extract = 0.0
    for _ in range(steps):
        t = time.perf_counter()
        out = run()
        total += time.perf_counter() - t
        dev += out[0]
        extract += out[1]
    return total / steps * 1e3, dev / steps, extract / steps, out


def measure(pm, segs, distinct_text, group_text, steps):
    from pinot_b200 import sql
    from pinot_b200.sql import SelectionQuery
    dq = sql.parse_distinct(distinct_text)
    gq = sql.parse(group_text, num_groups_limit=2_000_000)
    scan_q = SelectionQuery(columns=[], filter=dq.filter, order_by=[(dq.columns[0], True)], limit=0)

    def run_distinct():
        b = pm.execute_distinct(segs, dq, merge=True)
        return b.device_ms, pm.ctx.last_phases()["extract"], b

    def run_group():
        b = pm.execute_segments(segs, gq, merge=True)[0]
        return b.device_ms, pm.ctx.last_phases()["extract"], b

    def run_scan():
        b = pm.execute_selection(segs, scan_q, merge=True)
        return b.device_ms, 0.0, b
    d_step, d_dev, d_ext, (_, _, db) = timed(run_distinct, steps)
    g_step, g_dev, g_ext, (_, _, gb) = timed(run_group, steps)
    _, s_dev, _, _ = timed(run_scan, steps)
    return {"distinct": {"step_ms": round(d_step, 4), "device_ms": round(d_dev, 4), "extract_ms": round(d_ext, 4),
                         "rows": db.num_rows, "docs_scanned": db.stats.num_docs_scanned},
            "full_scan_ms": round(s_dev, 4),
            "group_by": {"step_ms": round(g_step, 4), "device_ms": round(g_dev, 4), "extract_ms": round(g_ext, 4),
                         "groups": gb.num_groups, "docs_scanned": gb.stats.num_docs_scanned}}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--dry-run", action="store_true", help="print the plan of the run without a GPU")
    args = ap.parse_args(argv)
    from pinot_b200 import sql
    plan = {f"{int(sel * 100)} %": query_texts(sel) for sel in (0.10, 0.01)}
    for texts in plan.values():
        for d, g in texts.values():
            sql.parse_distinct(d)   # every query parses
            sql.parse(g)
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {COLUMNS}", "queries": plan,
                          "measured": "not measured (dry run, no GPU)"}))
        return 0
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    segs = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, bench.column_specs(0, s, COLUMNS)) for s in range(args.segments)]
    out = {"gpu": card, "table": f"{args.segments} x {args.rows} rows", "steps": args.steps}
    try:
        for label, texts in plan.items():
            out[label] = {name: measure(pm, segs, d, g, args.steps) for name, (d, g) in texts.items()}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""What VAR / STDDEV queries cost on ONE GPU, on bench.py's table (8 segments x 100 M rows, c0..c7 of cardinality 10 ..
1 000 000, synthetic, resident in HBM), every segment in one merged submission:

    SELECT STDDEV_POP(c5) FROM benchTable WHERE c6 > K                   next to SUM(c5) and AVG(c5)
    SELECT c3, STDDEV_POP(c5) FROM benchTable WHERE c6 > K GROUP BY c3   next to SUM(c5) and AVG(c5)

at 10 % selectivity.  STDDEV_POP streams c5 once and sums three limb words per surviving row where SUM sums one value.
Per query: step ms (host clock around the call, which ends in a device synchronisation) and device ms (the scan
launches).  The one-off limb build is the first STDDEV query's step on fresh segments minus the steady step.  Plus the
card's name and power limit, read in the same run.  Prints one JSON object.

    python tests/workloads/run_variance.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_variance.py --dry-run     # no GPU: the queries and table shape it would run
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

COLUMNS = ["c3", "c5", "c6"]


def query_texts(selectivity: float):
    """{shape: {function: text}}"""
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k}"
    out = {}
    for shape, head, tail in (("aggregation only", "SELECT", ""), ("group by c3", "SELECT c3,", " GROUP BY c3 LIMIT 100000")):
        out[shape] = {fn: f"{head} {fn}(c5) {w}{tail}" for fn in ("STDDEV_POP", "SUM", "AVG")}
    return out


def timed(run, steps):
    for _ in range(2):
        run()
    total = dev = 0.0
    for _ in range(steps):
        t = time.perf_counter()
        b = run()
        total += time.perf_counter() - t
        dev += b.device_ms
    return {"step_ms": round(total / steps * 1e3, 4), "device_ms": round(dev / steps, 4)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--dry-run", action="store_true", help="print the plan of the run without a GPU")
    args = ap.parse_args(argv)
    from pinot_b200 import sql
    plan = query_texts(0.10)
    for texts in plan.values():
        assert sql.parse(texts["STDDEV_POP"]).aggregations[0].function == "STDDEVPOP"
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
    out = {"gpu": card, "table": f"{args.segments} x {args.rows} rows", "steps": args.steps, "selectivity": "10 %"}
    try:
        first = sql.parse(plan["aggregation only"]["STDDEV_POP"])
        t = time.perf_counter()
        pm.execute_segments(segs, first, merge=True)   # builds the limb dictionaries of c5, once per segment dictionary
        first_ms = (time.perf_counter() - t) * 1e3
        for shape, texts in plan.items():
            out[shape] = {}
            for fn, text in texts.items():
                q = sql.parse(text, num_groups_limit=2_000_000)
                out[shape][fn] = timed(lambda: pm.execute_segments(segs, q, merge=True)[0], args.steps)
        out["first STDDEV_POP step ms (limb build included)"] = round(first_ms, 4)
        out["limb build ms (first step minus steady step)"] = round(first_ms - out["aggregation only"]["STDDEV_POP"]["step_ms"], 4)
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

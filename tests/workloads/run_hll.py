#!/usr/bin/env python
"""What DISTINCTCOUNTHLL costs next to DISTINCTCOUNT on ONE GPU, on bench.py's table (8 segments x 100 M rows, c0..c7
of cardinality 10 .. 1 000 000, synthetic, resident in HBM), every segment in one merged submission:

    SELECT [c3,] DISTINCTCOUNT(c5)        FROM benchTable WHERE c6 > K [GROUP BY c3]
    SELECT [c3,] DISTINCTCOUNTHLL(c5)     ...
    SELECT [c3,] DISTINCTCOUNTHLL(c5, 12) ...

at 10 % selectivity.  Both functions set the same bits in the scan; DISTINCTCOUNTHLL adds the finalize, which reads
every bitset row once, and its sets are never decoded on the host (DISTINCTCOUNT's are, inside EXTRACT).  Per query:
step ms (host clock around the call, which ends in a device synchronisation), scan ms (the scan launches' CUDA events)
and the host phases of pb200_last_phases (the group-by finalize runs inside EXTRACT, the aggregation-only one before
DEVICE_WAIT).  Plus the card's name and power limit, read in the same run.  Prints one JSON object.

    python tests/workloads/run_hll.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_hll.py --dry-run     # no GPU: the queries and table shape it would run
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
SELECTS = {"DISTINCTCOUNT": "DISTINCTCOUNT(c5)", "DISTINCTCOUNTHLL": "DISTINCTCOUNTHLL(c5)",
           "DISTINCTCOUNTHLL_12": "DISTINCTCOUNTHLL(c5, 12)"}


def query_texts(selectivity: float):
    """{shape: {name: text}}"""
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k}"
    out = {}
    for shape, head, tail in (("aggregation only", "SELECT", ""), ("group by c3", "SELECT c3,", " GROUP BY c3 LIMIT 100000")):
        out[shape] = {name: f"{head} {sel} {w}{tail}" for name, sel in SELECTS.items()}
    return out


def timed(ctx, run, steps):
    for _ in range(2):
        run()
    total = dev = 0.0
    phases = {}
    for _ in range(steps):
        t = time.perf_counter()
        b = run()
        total += time.perf_counter() - t
        dev += b.device_ms
        for k, v in ctx.last_phases().items():
            phases[k] = phases.get(k, 0.0) + v
    out = {"step_ms": round(total / steps * 1e3, 4), "scan_ms": round(dev / steps, 4)}
    out.update({f"{k}_ms": round(v / steps, 4) for k, v in phases.items()})
    return out


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
        assert [a.arg for a in sql.parse(texts["DISTINCTCOUNTHLL_12"]).aggregations] == [12]
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
        for shape, texts in plan.items():
            out[shape] = {}
            for name, text in texts.items():
                q = sql.parse(text, num_groups_limit=2_000_000)
                out[shape][name] = timed(ctx, lambda: pm.execute_segments(segs, q, merge=True)[0], args.steps)
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

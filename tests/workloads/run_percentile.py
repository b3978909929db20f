#!/usr/bin/env python
"""What PERCENTILE queries cost on ONE GPU, on bench.py's table (8 segments x 100 M rows, c0..c7 of cardinality 10 ..
1 000 000, synthetic, resident in HBM), every segment in one merged submission (the synthetic segments share one
dictionary per column, which is what binding them to a domain gives):

    SELECT PERCENTILE(c5, 95) FROM benchTable WHERE c6 > K                                   (2^17 bins)
    SELECT PERCENTILE(c5, 50), PERCENTILE(c5, 95), PERCENTILE(c5, 99) ... (one shared histogram)
    SELECT PERCENTILE(c0, 50) ...                                                            (10 bins: contention)
    SELECT PERCENTILE(c2, 50) ...                                                            (1 000 bins)
    SELECT PERCENTILE(c6, 50) ...                                                            (2^20 bins: finalize)
    SELECT SUM(c5), PERCENTILE(c2, 95) ... GROUP BY c3                                       (10 000 groups x 1 000 bins)
    SELECT SUM(c5), PERCENTILE(c2, 99) ... GROUP BY c3 ORDER BY PERCENTILE(c2, 99) DESC LIMIT 10

at 10 % and 1 % selectivity, each next to the same query with MAX in place of PERCENTILE.  Per query: step ms (host
clock around the call, which ends in a device synchronisation), device ms (the scan launches), finalize ms (the device
wait after the scan was queued minus the scan: the finalize kernels and the read-back behind them), extract ms
(pb200_last_phases "extract"); plus the card's name and power limit, read in the same run.  Prints one JSON object.

    python tests/workloads/run_percentile.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_percentile.py --dry-run     # no GPU: the queries and table shape it would run
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

COLUMNS = ["c0", "c2", "c3", "c5", "c6"]


def query_texts(selectivity: float):
    """{shape: (PERCENTILE text, the same with MAX)}"""
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k}"
    shapes = {"p95(c5)": f"SELECT PERCENTILE(c5, 95) {w}",
              "p50,p95,p99(c5)": f"SELECT PERCENTILE(c5, 50), PERCENTILE(c5, 95), PERCENTILE(c5, 99) {w}",
              "p50(c0)": f"SELECT PERCENTILE(c0, 50) {w}",
              "p50(c2)": f"SELECT PERCENTILE(c2, 50) {w}",
              "p50(c6)": f"SELECT PERCENTILE(c6, 50) {w}",
              "sum(c5), p95(c2) group by c3": f"SELECT SUM(c5), PERCENTILE(c2, 95) {w} GROUP BY c3 LIMIT 100000",
              "... order by p99(c2) desc limit 10":
                  f"SELECT SUM(c5), PERCENTILE(c2, 99) {w} GROUP BY c3 ORDER BY PERCENTILE(c2, 99) DESC LIMIT 10"}
    as_max = lambda t: re.sub(r"PERCENTILE\((c\d), [0-9.]+\)", r"MAX(\1)", t)  # noqa: E731
    return {name: (t, as_max(t)) for name, t in shapes.items()}


def timed(run, steps):
    for _ in range(2):
        run()
    total = dev = wait = extract = 0.0
    for _ in range(steps):
        t = time.perf_counter()
        b, phases = run()
        total += time.perf_counter() - t
        dev += b.device_ms
        wait += phases["device_wait"]
        extract += phases["extract"]
    return {"step_ms": round(total / steps * 1e3, 4), "device_ms": round(dev / steps, 4),
            "finalize_ms": round(max(wait - dev, 0.0) / steps, 4), "extract_ms": round(extract / steps, 4)}


def measure(pm, segs, text, steps):
    from pinot_b200 import sql
    q = sql.parse(text, num_groups_limit=2_000_000)

    def run():
        b = pm.execute_segments(segs, q, merge=True)[0]
        return b, pm.ctx.last_phases()
    return timed(run, steps)


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
        for p, m in texts.values():
            assert any(a.function == "PERCENTILE" for a in sql.parse(p).aggregations)
            assert not any(a.function == "PERCENTILE" for a in sql.parse(m).aggregations)
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
            out[label] = {name: {"percentile": measure(pm, segs, p, args.steps), "max": measure(pm, segs, m, args.steps)}
                          for name, (p, m) in texts.items()}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

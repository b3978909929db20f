#!/usr/bin/env python
"""What an aggregation over a multi-column expression costs on ONE GPU, on bench.py's table (8 segments x 100 M rows,
synthetic, resident in HBM), every segment in one merged submission:

    SELECT SUM(c5 * c6), COUNT(*) FROM benchTable WHERE c6 > K GROUP BY c3     (10 000 groups, 10 % selectivity)
    SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c6 > K GROUP BY c3          (the same without the expression)

Per query: step ms (host clock around the call, which ends in a device synchronisation) and, from a separate
torch.profiler pass of 5 steps, the kernel times by name: the query's scan (scan_kernel<W, true>), the filter-only mask
scan (scan_kernel<W, false>) and the expression pass (expr_kernel); plus the card's name, power limit and SM clocks, read
in the same run.  Prints one JSON object.

    python tests/workloads/run_expr.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_expr.py --dry-run     # no GPU: the queries and table shape it would run
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


def query_texts(selectivity: float = 0.10):
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k} GROUP BY c3 LIMIT 100000"
    return {"expression": f"SELECT SUM(c5 * c6), COUNT(*) {w}", "column": f"SELECT SUM(c5), COUNT(*) {w}"}


def kernel_ms(run, steps=5):
    from torch.profiler import ProfilerActivity, profile
    run()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
    out = {"scan_ms": 0.0, "mask_scan_ms": 0.0, "expr_kernel_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "expr_kernel" in e.key:
            out["expr_kernel_ms"] += us / 1e3 / steps
        elif "scan_kernel" in e.key:
            out["scan_ms" if "true" in e.key else "mask_scan_ms"] += us / 1e3 / steps
    return {k: round(v, 4) for k, v in out.items()}


def measure(pm, segs, text, steps):
    from pinot_b200 import sql
    q = sql.parse(text)

    def run():
        return pm.execute_segments(segs, q, merge=True)[0]
    for _ in range(2):
        run()
    t = time.perf_counter()
    for _ in range(steps):
        run()
    out = {"step_ms": round((time.perf_counter() - t) / steps * 1e3, 4)}
    out.update(kernel_ms(run))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--dry-run", action="store_true", help="print the plan of the run without a GPU")
    args = ap.parse_args(argv)
    texts = query_texts()
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {COLUMNS}", "queries": texts,
                          "measured": "not measured (dry run, no GPU)"}))
        return 0
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    segs = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, bench.column_specs(0, s, COLUMNS)) for s in range(args.segments)]
    out = {"gpu": card, "table": f"{args.segments} x {args.rows} rows", "steps": args.steps}
    try:
        for name, text in texts.items():
            out[name] = dict(query=text, **measure(pm, segs, text, args.steps))
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    out["expression_cost_ms"] = round(out["expression"]["step_ms"] - out["column"]["step_ms"], 4)
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

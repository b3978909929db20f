#!/usr/bin/env python
"""What selection queries cost on ONE GPU, on bench.py's table (8 segments x 100 M rows, synthetic, resident in HBM):

    SELECT c3, c5 FROM benchTable WHERE c6 > K LIMIT 10
    SELECT c3, c5 FROM benchTable WHERE c6 > K ORDER BY c5 DESC LIMIT 10
    SELECT c3, c5 FROM benchTable WHERE c6 > K ORDER BY c5 DESC LIMIT 10000

at 10 % and 1 % selectivity, every segment in one merged submission.  Per query: step ms (host clock around
execute_selection, which ends in the select phase's synchronisation), the scan kernels' CUDA-event time, the select phase
(pb200_last_phases "extract": host clock from the end of the scans to the end of the call, host merge included), the
rows returned and the docs scanned (the selection-only prefix scan scans far fewer than 800 M); plus the card's name and
power limit.  Prints one JSON object.

    python tests/workloads/run_selection.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_selection.py --dry-run     # no GPU: the queries and table shape it would run
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


def query_texts(selectivity: float):
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    base = f"SELECT c3, c5 FROM benchTable WHERE c6 > {k}"
    return {"limit 10": f"{base} LIMIT 10",
            "order by c5 desc limit 10": f"{base} ORDER BY c5 DESC LIMIT 10",
            "order by c5 desc limit 10000": f"{base} ORDER BY c5 DESC LIMIT 10000"}


def measure(pm, segs, q, steps):
    for _ in range(2):
        pm.execute_selection(segs, q, merge=True)
    step = kernel = select = 0.0
    for _ in range(steps):
        t = time.perf_counter()
        block = pm.execute_selection(segs, q, merge=True)
        step += time.perf_counter() - t
        kernel += block.device_ms
        select += pm.ctx.last_phases()["extract"]
    return {"step_ms": round(step / steps * 1e3, 4), "scan_kernel_ms": round(kernel / steps, 4),
            "select_phase_ms": round(select / steps, 4), "rows": block.num_rows,
            "docs_scanned_matched": block.stats.num_docs_scanned}


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
        for text in texts.values():
            sql.parse_selection(text)   # every query parses
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {bench.TOUCHED}", "queries": plan,
                          "measured": "not measured (dry run, no GPU)"}))
        return 0
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    segs = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, bench.column_specs(0, s, bench.TOUCHED)) for s in range(args.segments)]
    out = {"gpu": card, "table": f"{args.segments} x {args.rows} rows", "steps": args.steps}
    try:
        for label, texts in plan.items():
            out[label] = {name: measure(pm, segs, sql.parse_selection(text), args.steps) for name, text in texts.items()}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

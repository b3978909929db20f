#!/usr/bin/env python
"""What a predicate on an expression over two columns costs on ONE GPU, on bench.py's table (8 segments x 100 M rows,
synthetic, resident in HBM), every segment in one merged submission:

    SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c5 > c6 GROUP BY c3        (the doc-mask pass, then the usual scan)
    SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c6 > K GROUP BY c3         (a single-column filter of similar selectivity)

Per query: step ms (host clock around the call, which ends in a device synchronisation) and, from a separate
torch.profiler pass of 5 steps, the kernel times by name: the mask pass (expr_mask_kernel) and the query's scan
(scan_kernel).  For the mask pass, the bytes it must move (the leaf forward indexes, bits / 8 per doc per leaf, plus
num_docs / 8 of mask) over its kernel time, and that time against the HBM bound at the data sheet's 3.35 TB/s; plus the
card's name, power limit and SM clocks, read in the same run.  Prints one JSON object.

    python tests/workloads/run_expr_filter.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_expr_filter.py --dry-run     # no GPU: the queries and table shape it would run
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
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def query_texts(selectivity: float):
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    tail = "GROUP BY c3 LIMIT 100000"
    return {"expression": f"SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c5 > c6 {tail}",
            "column": f"SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c6 > {k} {tail}"}


def kernel_ms(run, steps=5):
    from torch.profiler import ProfilerActivity, profile
    run()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
    out = {"mask_pass_ms": 0.0, "scan_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "expr_mask_kernel" in e.key:
            out["mask_pass_ms"] += us / 1e3 / steps
        elif "scan_kernel" in e.key:
            out["scan_ms"] += us / 1e3 / steps
    return {k: round(v, 4) for k, v in out.items()}


def measure(pm, segs, text, steps):
    from pinot_b200 import sql
    q = sql.parse(text)

    def run():
        return pm.execute_segments(segs, q, merge=True)[0]
    for _ in range(2):
        b = run()
    t = time.perf_counter()
    for _ in range(steps):
        run()
    out = {"step_ms": round((time.perf_counter() - t) / steps * 1e3, 4), "matched": int(b.stats.num_docs_scanned)}
    out.update(kernel_ms(run))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--dry-run", action="store_true", help="print the plan of the run without a GPU")
    args = ap.parse_args(argv)
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {COLUMNS}", "queries": query_texts(0.175),
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
        texts = query_texts(0.175)
        out["expression"] = dict(query=texts["expression"], **measure(pm, segs, texts["expression"], args.steps))
        total = args.rows * args.segments
        texts = query_texts(out["expression"]["matched"] / total)   # the column filter at the measured selectivity
        out["column"] = dict(query=texts["column"], **measure(pm, segs, texts["column"], args.steps))
        bits = sum(segs[0].column_info(c)["bits"] for c in ("c5", "c6"))
        need = total * (bits / 8 + 1 / 8)
        ms = out["expression"]["mask_pass_ms"]
        out["mask_pass"] = {"bytes": int(need), "leaf_bits_per_doc": bits, "hbm_bound_ms": round(need / HBM_BYTES_PER_S * 1e3, 4),
                            "achieved_gb_per_s": round(need / (ms / 1e3) / 1e9, 1) if ms else None,
                            "times_the_bound": round(ms / (need / HBM_BYTES_PER_S * 1e3), 2) if ms else None}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    out["expression_cost_ms"] = round(out["expression"]["step_ms"] - out["column"]["step_ms"], 4)
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

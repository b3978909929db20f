#!/usr/bin/env python
"""What FIRSTWITHTIME / LASTWITHTIME queries cost on ONE GPU, on bench.py's table (8 segments x 100 M rows, c0..c7 of
cardinality 10 .. 1 000 000, synthetic, resident in HBM), every segment in one merged submission (the synthetic segments
share one dictionary per column, which is what binding them to a domain gives):

    SELECT LASTWITHTIME(c5, c7, 'INT') FROM benchTable WHERE c6 > K GROUP BY c3     (10 000 groups)
    the same on the hash table (dense_max = 1: 2^22 slots for numGroupsLimit 2 000 000, one finalize thread each)
    SELECT LASTWITHTIME(c5, c7, 'INT') FROM benchTable WHERE c6 > K                 (aggregation only)

at 10 % and 1 % selectivity, each next to the same query with MAX(c5) in its place.  Per query: step ms (host clock
around the call, which ends in a device synchronisation), device ms (the scan kernel, CUDA events), extract ms
(pb200_last_phases "extract"), and from a separate torch.profiler pass of 5 steps the kernel times by name: the scan and
the finalize (withtime_finalize_kernel); plus the card's name, power limit and SM clocks, read in the same run.  Prints
one JSON object.

    python tests/workloads/run_withtime.py [--steps 10] [--rows 100000000] [--segments 8]
    python tests/workloads/run_withtime.py --dry-run     # no GPU: the queries and table shape it would run
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

COLUMNS = ["c3", "c5", "c6", "c7"]


def query_texts(selectivity: float):
    """{shape: (LASTWITHTIME text, the same with MAX)}"""
    k_id = int(round(bench.CARDS[6] * (1 - selectivity))) - 1     # c6 > value(k_id): the upper `selectivity` of the dictionary
    k = bench.VALUE_BASE[6] + bench.VALUE_STEP[6] * k_id
    w = f"FROM benchTable WHERE c6 > {k}"
    shapes = {"group by c3": f"SELECT LASTWITHTIME(c5, c7, 'INT') {w} GROUP BY c3 LIMIT 100000",
              "group by c3 (hash table)": f"SELECT LASTWITHTIME(c5, c7, 'INT') {w} GROUP BY c3 LIMIT 100000",
              "aggregation only": f"SELECT LASTWITHTIME(c5, c7, 'INT') {w}"}
    as_max = lambda t: re.sub(r"LASTWITHTIME\((c\d), c7, 'INT'\)", r"MAX(\1)", t)  # noqa: E731
    return {name: (t, as_max(t)) for name, t in shapes.items()}


def timed(run, steps):
    for _ in range(2):
        run()
    total = dev = extract = 0.0
    for _ in range(steps):
        t = time.perf_counter()
        b, phases = run()
        total += time.perf_counter() - t
        dev += b.device_ms
        extract += phases["extract"]
    return {"step_ms": round(total / steps * 1e3, 4), "device_ms": round(dev / steps, 4),
            "extract_ms": round(extract / steps, 4)}


def kernel_ms(run, steps=5):
    """Per-step device time of the scan and the finalize kernels, from torch.profiler (CUPTI sees every kernel of the
    process, the library's included).  A separate pass: tracing slows the host."""
    from torch.profiler import ProfilerActivity, profile
    run()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
    out = {"scan_kernel_ms": 0.0, "finalize_kernel_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "scan_kernel" in e.key:
            out["scan_kernel_ms"] += us / 1e3 / steps
        elif "withtime_finalize" in e.key:
            out["finalize_kernel_ms"] += us / 1e3 / steps
    return {k: round(v, 4) for k, v in out.items()}


def measure(pm, segs, name, text, steps):
    from pinot_b200 import sql
    q = sql.parse(text, num_groups_limit=2_000_000)
    hashed = "hash table" in name
    if hashed:
        pm.ctx.set_tuning("dense_max", 1)

    def run():
        b = pm.execute_segments(segs, q, merge=True)[0]
        return b, pm.ctx.last_phases()
    try:
        out = timed(run, steps)
        out.update(kernel_ms(run))
    finally:
        if hashed:
            pm.ctx.set_tuning("dense_max", 1 << 24)
    return out


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
            assert any(a.function == "LASTWITHTIME" for a in sql.parse(p).aggregations)
            assert [a.function for a in sql.parse(m).aggregations] == ["MAX"]
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {COLUMNS}", "queries": plan,
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
        for label, texts in plan.items():
            out[label] = {name: {"lastwithtime": measure(pm, segs, name, p, args.steps), "max": measure(pm, segs, name, m, args.steps)}
                          for name, (p, m) in texts.items()}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""What an aggregation over CASE WHEN costs on ONE GPU, on bench.py's table (8 segments x 100 M rows, synthetic, resident
in HBM), every segment in one merged submission:

    SELECT SUM(CASE WHEN c4 = K THEN c5 ELSE 0 END), COUNT(*) FROM benchTable GROUP BY c3     (10 000 groups)
    SELECT SUM(c5) FILTER (WHERE c4 = K), COUNT(*) FROM benchTable GROUP BY c3                 (the FILTER-clause form)
    SELECT SUM(c5), COUNT(*) FROM benchTable GROUP BY c3                                       (no condition)

bench.py's columns are all INT, so the condition is an INT equality.  One more run puts a STRING condition on a table
of this script's own (--string-rows rows in 2 segments: a 6-value STRING status, an INT value, 1 000 groups):

    SELECT SUM(CASE WHEN status = 'error' THEN bytes ELSE 0 END), COUNT(*) FROM logs GROUP BY host

Per query: step ms (host clock around the call, which ends in a device synchronisation) and, from a separate
torch.profiler pass of 5 steps, the kernel times by name (run_expr.kernel_ms): the scans and the expression pass
(expr_kernel); plus the card's name, power limit and SM clocks, read in the same run.  Prints one JSON object.

    python tests/workloads/run_case.py [--steps 10] [--rows 100000000] [--segments 8] [--string-rows 20000000]
    python tests/workloads/run_case.py --dry-run     # no GPU: the queries and table shape it would run
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import bench  # noqa: E402
from run_expr import measure  # noqa: E402

COLUMNS = ["c3", "c4", "c5"]
STATUSES = [b"ok", b"error", b"warn", b"retry", b"timeout", b"redirect"]


def query_texts():
    k = bench.VALUE_BASE[4] + bench.VALUE_STEP[4] * (bench.CARDS[4] // 3)   # one value of c4: 1 / 65 536 of the rows
    g = "FROM benchTable GROUP BY c3 LIMIT 100000"
    return {"case": f"SELECT SUM(CASE WHEN c4 = {k} THEN c5 ELSE 0 END), COUNT(*) {g}",
            "filter_clause": f"SELECT SUM(c5) FILTER (WHERE c4 = {k}), COUNT(*) {g}",
            "column": f"SELECT SUM(c5), COUNT(*) {g}"}


STRING_QUERY = "SELECT SUM(CASE WHEN status = 'error' THEN bytes ELSE 0 END), COUNT(*) FROM logs GROUP BY host LIMIT 100000"


def string_table(ctx, rows):
    import numpy as np

    from oracle.pinot_oracle import oracle as get_oracle
    from pinot_b200.plan_maker import IndexSegment
    o = get_oracle()
    out = []
    for s in range(2):
        rng = np.random.default_rng(40 + s)
        n = rows // 2
        seg = o.build_segment(f"logs{s}", {"status": np.array(STATUSES)[rng.integers(0, len(STATUSES), size=n)],
                                           "bytes": rng.integers(0, 100_000, size=n).astype(np.int32),
                                           "host": rng.integers(0, 1000, size=n).astype(np.int32)})
        out.append(IndexSegment.from_columns(ctx, seg.name, seg.num_docs, seg.columns))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--string-rows", type=int, default=20_000_000)
    ap.add_argument("--dry-run", action="store_true", help="print the plan of the run without a GPU")
    args = ap.parse_args(argv)
    texts = query_texts()
    if args.dry_run:
        print(json.dumps({"table": f"{args.segments} x {args.rows} rows, columns {COLUMNS}", "queries": texts,
                          "string_table": f"2 x {args.string_rows // 2} rows", "string_query": STRING_QUERY,
                          "measured": "not measured (dry run, no GPU)"}))
        return 0
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    out = {"gpu": card, "table": f"{args.segments} x {args.rows} rows", "steps": args.steps}
    segs = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, bench.column_specs(0, s, COLUMNS)) for s in range(args.segments)]
    try:
        for name, text in texts.items():
            out[name] = dict(query=text, **measure(pm, segs, text, args.steps))
    finally:
        for s in segs:
            s.destroy()
    logs = string_table(ctx, args.string_rows)
    try:
        out["string_case"] = dict(query=STRING_QUERY, table=f"2 x {args.string_rows // 2} rows", **measure(pm, logs, STRING_QUERY, args.steps))
    finally:
        for s in logs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

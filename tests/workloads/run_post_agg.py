#!/usr/bin/env python
"""What ORDER BY an expression over aggregations costs on ONE GPU, against the same order by a plain aggregation: bench's
8 x 100 M-row table, merged, grouped into 10 000 (c3), 100 000 (c2, c1) and 1 M (c6) groups (bench's filter c6 > K for
the first two, which keeps 10 % of the rows; c7 > K, which keeps half of them, for c6), each run with
`ORDER BY AVG(c5) DESC LIMIT 10` and with `ORDER BY SUM(c5) / COUNT(*) DESC LIMIT 10`, alternating, 3 repeats.  Both
arms keep a sum and a count per group, so their scans do the same work; the expression adds one evaluation per row in
one sort pass.  Per run: step ms (host clock around execute_segments, which ends in the extraction's synchronisation),
the library's extract phase (pb200_last_phases), the scan kernel's CUDA-event time and the rows returned; the kept rows
of the two arms must be the same groups in the same order.  Also the card's name and power limit, read in the same run.
Prints one JSON object."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ARMS = {"avg": "AVG(c5)", "expr": "SUM(c5) / COUNT(*)"}


def measure(pm, segs, q, steps):
    for _ in range(3):
        pm.execute_segments(segs, q, merge=True)
    t = time.perf_counter()
    extract = 0.0
    for _ in range(steps):
        block = pm.execute_segments(segs, q, merge=True)[0]
        extract += pm.ctx.last_phases()["extract"]
    step = (time.perf_counter() - t) / steps * 1e3
    keys = [tuple(int(x) for x in row) for row in block.keys[: block.num_groups]]
    return {"step_ms": round(step, 4), "extract_ms": round(extract / steps, 4), "kernel_ms": round(block.device_ms, 4),
            "rows": block.num_groups}, keys


def compare(pm, segs, group_by, where, steps, limit):
    from pinot_b200 import sql
    queries = {arm: sql.parse(f"SELECT {group_by}, {item} FROM benchTable WHERE {where} GROUP BY {group_by} "
                              f"ORDER BY {item} DESC LIMIT 10", num_groups_limit=limit)
               for arm, item in ARMS.items()}
    runs = {arm: [] for arm in ARMS}
    rows = {}
    for _ in range(3):
        for arm, q in queries.items():
            r, keys = measure(pm, segs, q, steps)
            runs[arm].append(r)
            rows.setdefault(arm, keys)
            assert keys == rows[arm], f"{arm}: rows changed between repeats"
    runs["same_rows"] = rows["avg"] == rows["expr"]
    assert runs["same_rows"], f"{group_by}: the two arms kept different rows"
    return runs


def main():
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    out = {"gpu": card}
    segs = [IndexSegment.synthetic(ctx, f"s{s}", 100_000_000, bench.column_specs(0, s)) for s in range(8)]
    c6_filter = bench.groupby_query_text(0.10).split(" WHERE ")[1].split(" GROUP BY")[0]
    c7_half = f"c7 > {bench.VALUE_BASE[7] + bench.VALUE_STEP[7] * (bench.CARDS[7] // 2 - 1)}"
    try:
        out["10 000 groups (c3)"] = compare(pm, segs, "c3", c6_filter, 30, 100_000)
        out["100 000 groups (c2, c1)"] = compare(pm, segs, "c2, c1", c6_filter, 20, 1_000_000)
        out["1 M groups (c6)"] = compare(pm, segs, "c6", c7_half, 10, 2_000_000)
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

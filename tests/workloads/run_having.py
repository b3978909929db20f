#!/usr/bin/env python
"""What HAVING costs on ONE GPU: the bench headline's table (8 x 100 M rows, 10 000 groups), C4 (100 000 groups) and the
1 M-group query, merged, each with `ORDER BY SUM(...) DESC LIMIT 10` and run without HAVING and with `HAVING COUNT(*) > K`,
K chosen from the groups' counts to keep about 1 % and about 50 % of them; the three alternate, 3 repeats.  Per run: step
ms (host clock around execute_segments, which ends in the extraction's synchronisation), the library's extract phase
(pb200_last_phases), the scan kernel's CUDA-event time and the rows returned; plus the card's name and power limit.  Prints
one JSON object."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from run_order_by import measure  # noqa: E402


def compare(pm, segs, text, steps, limit):
    """text: a GROUP BY query without ORDER BY; its first aggregation is the SUM the runs order by."""
    from pinot_b200 import sql
    counted = sql.parse(text.replace("SELECT ", "SELECT COUNT(*), ", 1), num_groups_limit=limit)
    counts = np.asarray(pm.execute_segments(segs, counted, merge=True)[0].longs[0])
    sum_expr = "SUM(" + text.split("SUM(")[1].split(")")[0] + ")"
    order = f" ORDER BY {sum_expr} DESC LIMIT 10"
    queries = {"no_having": sql.parse(text + order, num_groups_limit=limit)}
    for name, q in (("having_1pct", 0.99), ("having_50pct", 0.50)):
        k = int(np.quantile(counts, q))
        queries[f"{name} (COUNT(*) > {k})"] = sql.parse(f"{text} HAVING COUNT(*) > {k}{order}", num_groups_limit=limit)
    runs = {name: [] for name in queries}
    for _ in range(3):
        for name, q in queries.items():
            runs[name].append(measure(pm, segs, q, steps))
    runs["groups"] = int(len(counts))
    return runs


def main():
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    out = {"gpu": card}
    segs = [IndexSegment.synthetic(ctx, f"s{s}", 100_000_000, bench.column_specs(0, s)) for s in range(8)]
    out["headline (10 000 groups)"] = compare(pm, segs, bench.groupby_query_text(0.10).split(" LIMIT")[0], 30, 100_000)
    for s in segs:
        s.destroy()
    cols = [("f", 10_000), ("g1", 1_000), ("g2", 100), ("m1", 100_000), ("m2", 65_536), ("g3", 1_000)]
    segs = [IndexSegment.synthetic(ctx, f"c4s{s}", 50_000_000,
                                   [{"name": n, "cardinality": c, "value_base": 1, "value_step": 3, "seed": 7919 * s + i}
                                    for i, (n, c) in enumerate(cols)]) for s in range(8)]
    out["C4 (100 000 groups)"] = compare(pm, segs, "SELECT SUM(m1), MAX(m2) FROM t WHERE f BETWEEN 3001 AND 5998 GROUP BY g1, g2",
                                         20, 1_000_000)
    out["1 M groups"] = compare(pm, segs, "SELECT SUM(m1) FROM t WHERE f BETWEEN 3001 AND 5998 GROUP BY g1, g3", 10, 2_000_000)
    for s in segs:
        s.destroy()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

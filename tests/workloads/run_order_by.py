#!/usr/bin/env python
"""What ORDER BY ... LIMIT 10 costs on ONE GPU: the bench headline (10 000 groups), C4 (100 000) and the 1 M-group query,
each run with and without `ORDER BY SUM(...) DESC LIMIT 10`, alternating, 3 repeats.  Per run: step ms (host clock around
execute_segments, which ends in the extraction's synchronisation), the library's extract phase (pb200_last_phases), the
scan kernel's CUDA-event time and the rows returned; plus the card's name and power limit.  Prints one JSON object."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def measure(pm, segs, q, steps):
    for _ in range(3):
        pm.execute_segments(segs, q, merge=True)
    t = time.perf_counter()
    extract = 0.0
    for _ in range(steps):
        block = pm.execute_segments(segs, q, merge=True)[0]
        extract += pm.ctx.last_phases()["extract"]
    step = (time.perf_counter() - t) / steps * 1e3
    return {"step_ms": round(step, 4), "extract_ms": round(extract / steps, 4), "kernel_ms": round(block.device_ms, 4),
            "rows": block.num_groups}


def compare(pm, segs, text, order, steps, limit):
    from pinot_b200 import sql
    plain = sql.parse(text, num_groups_limit=limit)
    ordered = sql.parse(text.split(" LIMIT")[0] + order, num_groups_limit=limit)
    runs = {"plain": [], "ordered": []}
    for _ in range(3):
        runs["plain"].append(measure(pm, segs, plain, steps))
        runs["ordered"].append(measure(pm, segs, ordered, steps))
    return runs


def main():
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    out = {"gpu": card}
    segs = [IndexSegment.synthetic(ctx, f"s{s}", 100_000_000, bench.column_specs(0, s)) for s in range(8)]
    text = bench.groupby_query_text(0.10)
    sum_col = text.split("SUM(")[1].split(")")[0]
    out["headline (10 000 groups)"] = compare(pm, segs, text, f" ORDER BY SUM({sum_col}) DESC LIMIT 10", 30, 100_000)
    for s in segs:
        s.destroy()
    cols = [("f", 10_000), ("g1", 1_000), ("g2", 100), ("m1", 100_000), ("m2", 65_536), ("g3", 1_000)]
    segs = [IndexSegment.synthetic(ctx, f"c4s{s}", 50_000_000,
                                   [{"name": n, "cardinality": c, "value_base": 1, "value_step": 3, "seed": 7919 * s + i}
                                    for i, (n, c) in enumerate(cols)]) for s in range(8)]
    out["C4 (100 000 groups)"] = compare(pm, segs, "SELECT SUM(m1), MAX(m2) FROM t WHERE f BETWEEN 3001 AND 5998 GROUP BY g1, g2",
                                         " ORDER BY SUM(m1) DESC LIMIT 10", 20, 1_000_000)
    out["1 M groups"] = compare(pm, segs, "SELECT SUM(m1), COUNT(*) FROM t WHERE f BETWEEN 3001 AND 5998 GROUP BY g1, g3",
                                " ORDER BY SUM(m1) DESC LIMIT 10", 10, 2_000_000)
    for s in segs:
        s.destroy()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

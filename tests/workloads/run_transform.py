#!/usr/bin/env python
"""What a derived column costs (DESIGN.md section 3.8), on bench.py's table: 8 segments x 100 M rows of dictionary-encoded INT
columns c0..c7, queried in one merged submission.  For each expression E of

    datetrunc('SECOND',c7)    floor(divide(c5,'100'))    mod(c6,'10000')

it reports
  * the derived column's cardinality and bits;
  * the derivation: the first query naming E (which derives it on all 8 segments) minus the steady-state step, and the
    derive call alone (pb200h_segment_derive on each segment of a second, identical table, host clock, summed);
  * steady-state ms per step (host clock around `steps` steps, each ending with its results on the host) and scan-kernel
    ms (CUDA events) of SELECT SUM(c5), COUNT(*) WHERE c6 > K GROUP BY E, next to GROUP BY c3 (the bench headline) and
    GROUP BY a stored column of the same cardinality -- so of the same bits -- added to the table for the comparison,
    measured alternately in the same run.

    python tests/workloads/run_transform.py [--segments 8 --rows 100000000 --steps 100 --warmup 10 --selectivity 0.1]

Prints one JSON line per expression and one with the device's name, power limit and SM clock."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

EXPRESSIONS = ["datetrunc('SECOND',c7)", "floor(divide(c5,'100'))", "mod(c6,'10000')"]


def derived_cardinalities():
    """|f(dictionary)| of each expression over bench.py's dictionaries (value_base + value_step * id)."""
    import numpy as np

    from bench import CARDS, VALUE_BASE, VALUE_STEP
    dict_of = lambda c: VALUE_BASE[c] + VALUE_STEP[c] * np.arange(CARDS[c], dtype=np.int64)  # noqa: E731
    return [len(np.unique(dict_of(7) // 1000 * 1000)),
            len(np.unique(np.floor(dict_of(5).astype(np.float64) / 100.0))),
            len(np.unique(np.fmod(dict_of(6).astype(np.float64), 10000.0)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--selectivity", type=float, default=0.10)
    args = ap.parse_args()

    import numpy as np

    from bench import CARDS, VALUE_BASE, VALUE_STEP, bits_of, column_specs
    from pinot_b200 import sql
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment

    cards = derived_cardinalities()
    k_id = int(round(CARDS[6] * (1 - args.selectivity))) - 1
    where = f"WHERE c6 > {VALUE_BASE[6] + VALUE_STEP[6] * k_id}"

    def query(key):
        return sql.parse(f"SELECT SUM(c5), COUNT(*) FROM benchTable {where} GROUP BY {key} LIMIT 100000")

    def specs(s):
        extra = [{"name": f"x{k}", "cardinality": card, "value_base": 0, "value_step": 1, "seed": 77 + 31 * s + k}
                 for k, card in enumerate(cards)]
        return column_specs(0, s) + extra

    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    table = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, specs(s)) for s in range(args.segments)]
    fresh = [IndexSegment.synthetic(ctx, f"f{s}", args.rows, specs(s)) for s in range(args.segments)]
    try:
        def steady(q):
            for _ in range(args.warmup):
                pm.execute_segments(table, q, merge=True)
            kms = []
            t0 = time.perf_counter()
            for _ in range(args.steps):
                b = pm.execute_segments(table, q, merge=True)[0]
                kms.append(b.device_ms)
            return (time.perf_counter() - t0) / args.steps * 1e3, float(np.mean(kms)), b

        headline = query("c3")
        for k, expr in enumerate(EXPRESSIONS):
            q = query(expr)
            t0 = time.perf_counter()
            first = pm.execute_segments(table, q, merge=True)[0]      # derives expr on every segment
            first_ms = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            for s in fresh:
                s.derive(expr)
            derive_ms = (time.perf_counter() - t0) * 1e3
            info_e = table[0].column_info(expr)
            rows = {}
            for name, qq in (("expression", q), ("headline_c3", headline), (f"stored_x{k}", query(f"x{k}")),
                             ("expression_again", q)):
                ms, kms, b = steady(qq)
                rows[name] = {"ms_per_step": round(ms, 4), "kernel_ms": round(kms, 4), "groups": int(b.num_groups)}
            assert first.num_groups == rows["expression"]["groups"]
            print(json.dumps({
                "expression": expr, "cardinality": info_e["cardinality"], "bits": info_e["bits"],
                "stored_same_bits": {"column": f"x{k}", "bits": bits_of(cards[k])},
                "first_query_ms": round(first_ms, 3),
                "derivation_ms_first_minus_steady": round(first_ms - rows["expression"]["ms_per_step"], 3),
                "derive_call_ms_all_segments": round(derive_ms, 3), "segments": args.segments, "rows": args.rows,
                "steady": rows}), flush=True)
        print(json.dumps({"device": info}))
    finally:
        for s in table + fresh:
            s.destroy()
        ctx.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""The bench headline's query shape on the bench table, grouped by any of its columns: SELECT SUM(c5), COUNT(*) WHERE
c6 > K GROUP BY <col>, merged over the segments.  GROUP BY c3 (10 000 groups) is the headline itself (one 8-warp CTA per
SM with a shared-memory table); GROUP BY c2 (1 000 groups) takes two 6-warp CTAs per SM with replicated shared tables.

    python tests/workloads/run_spec_groupby.py --group-by c2 [--segments 8 --rows 100000000 --steps 300 --selectivity 0.1]

Prints one JSON line: wall ms per step (a host clock around `steps` steps that ends in a device synchronisation), the
mean device time of the scan (CUDA events), the number of groups and a digest of the result (sorted keys, sums and
counts), so that two builds can be checked for identical outputs.  PB200_* environment knobs apply (PB200_NO_SPEC=1:
the generic group-by kernel)."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--group-by", default="c2")
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--selectivity", type=float, default=0.10)
    args = ap.parse_args()

    import numpy as np

    from bench import CARDS, VALUE_BASE, VALUE_STEP, column_specs
    from pinot_b200 import sql
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment

    k_id = int(round(CARDS[6] * (1 - args.selectivity))) - 1
    text = (f"SELECT SUM(c5), COUNT(*) FROM benchTable WHERE c6 > {VALUE_BASE[6] + VALUE_STEP[6] * k_id} "
            f"GROUP BY {args.group_by} LIMIT 100000")
    q = sql.parse(text)
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    segs = [IndexSegment.synthetic(ctx, f"s{s}", args.rows, column_specs(0, s)) for s in range(args.segments)]
    try:
        def step():
            b = pm.execute_segments(segs, q, merge=True)[0]
            return b, b.device_ms

        for _ in range(args.warmup):
            block, _ = step()
        kms = []
        t0 = time.perf_counter()
        for _ in range(args.steps):
            block, ms = step()
            kms.append(ms)
        elapsed = time.perf_counter() - t0   # every step ends with its results on the host
        order = np.argsort(block.keys[:, 0])
        digest = hashlib.sha256()
        for a in (block.keys[:, 0][order].astype(np.int64), block.doubles[0][order], block.longs[1][order]):
            digest.update(np.ascontiguousarray(a).tobytes())
        print(json.dumps({"query": text, "ms_per_step": elapsed / args.steps * 1e3, "kernel_ms": float(np.mean(kms)),
                          "steps": args.steps, "groups": int(block.num_groups), "matched": int(block.longs[1].sum()),
                          "digest": digest.hexdigest()[:16],
                          "env": {k: v for k, v in os.environ.items() if k.startswith("PB200_")}}))
    finally:
        for s in segs:
            s.destroy()
        ctx.close()


if __name__ == "__main__":
    main()

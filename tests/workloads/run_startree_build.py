#!/usr/bin/env python
"""Star-tree built on the device (pb200h_startree_build) on C5's segment shape, next to the host builder.

    python tests/workloads/run_startree_build.py --rows 100000000 --host-rows 2000000

C5's columns (d_hi 100 000 values, d_lo 10, metric m 1 000) plus two more dimensions (d_mid 100, d_small 4) make one
4-dimension config: split order d_hi, d_lo, d_mid, d_small; pairs COUNT(*), SUM(m), MAX(m); maxLeafRecords 10 000.

  full size   the segment is generated in HBM and the tree built on the device (phases reported); the three run_c5.py
              queries run through it and through the raw scan, results checked equal.
  host size   the test-side host builder (oracle/startree_builder.py, numpy) cannot finish 100 M rows in reasonable time:
              at --host-rows both builders run on the same data and must agree on star docs and nodes; the queries run
              through the device-built tree, the host-built tree (attached) and the raw scan, results checked equal.

Prints one JSON line with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

QUERIES = ["SELECT SUM(m), COUNT(*), MAX(m) FROM t GROUP BY d_hi",
           "SELECT SUM(m), COUNT(*) FROM t WHERE d_lo = 3 GROUP BY d_hi",
           "SELECT SUM(m), COUNT(*) FROM t WHERE d_hi BETWEEN 1000 AND 1999"]
DIMS = ["d_hi", "d_lo", "d_mid", "d_small"]
PAIRS = [("COUNT", None), ("SUM", "m"), ("MAX", "m")]


def specs(high_card):
    return [{"name": "d_hi", "cardinality": high_card, "value_base": 0, "value_step": 1, "seed": 11},
            {"name": "d_lo", "cardinality": 10, "value_base": 0, "value_step": 1, "seed": 12},
            {"name": "m", "cardinality": 1000, "value_base": 1, "value_step": 1, "seed": 13},
            {"name": "d_mid", "cardinality": 100, "value_base": 0, "value_step": 1, "seed": 14},
            {"name": "d_small", "cardinality": 4, "value_base": 0, "value_step": 1, "seed": 15}]


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split("\n")[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stay valid; the card is then unnamed in the output
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def time_queries(pm, plans, host_seg, steps, warmup):
    """plans: {name: (segment, use_star_tree)} -> per query, ms per query of each plan; results checked equal."""
    from gpu_util import assert_tables_equal, gpu_table
    from pinot_b200 import sql
    out = []
    for text in QUERIES:
        res, tables = {"query": text}, {}
        for name, (seg, use) in plans.items():
            q = sql.parse(text, use_star_tree=use, num_groups_limit=2_000_000)
            for _ in range(warmup):
                b = pm.execute_segments([seg], q, views=True)[0]
            t0 = time.perf_counter()
            for _ in range(steps):
                b = pm.execute_segments([seg], q, views=True)[0]
            ms = (time.perf_counter() - t0) / steps * 1e3
            assert (b.operator_kind == "STAR_TREE") == use, (name, b.operator_kind)
            tables[name] = gpu_table(host_seg, q, b)
            res[name] = {"ms_per_query": round(ms, 3), "docs_scanned": b.stats.num_docs_scanned, "groups": b.num_groups}
        first = next(iter(tables))
        for name in tables:
            assert_tables_equal(q, tables[name], tables[first], f"{name} vs {first}: {text}")
        res["identical"] = True
        out.append(res)
    return out


def host_segment(o, seg, sp, n):
    """The synthetic segment's columns read back as oracle SegmentData (what the host builder takes)."""
    import numpy as np
    from oracle import segment_builder as sb
    docs = np.arange(n, dtype=np.int32)
    cols = []
    for s in sp:
        info = seg.column_info(s["name"])
        fwd = seg.read_index(s["name"], "fwd")
        vals = (s["value_base"] + s["value_step"] * np.arange(s["cardinality"])).astype(np.int32)
        cols.append(sb.ColumnData(s["name"], sb.INT, True, info["bits"], s["cardinality"], False, 4, fwd,
                                  seg.read_index(s["name"], "dict"), None, dict_values=vals,
                                  dict_ids=o.read_dict_ids(fwd, n, info["bits"], docs)))
    return sb.SegmentData(seg.name, n, cols)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--host-rows", type=int, default=2_000_000)
    ap.add_argument("--high-card", type=int, default=100_000)
    ap.add_argument("--max-leaf-records", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    from oracle import segment_builder as sb
    from oracle import startree_builder as stb
    from oracle.pinot_oracle import oracle as get_oracle
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    from startree_canon import tree_nodes

    o = get_oracle()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    sp = specs(args.high_card)
    out = {"workload": "startree_build", **card_info(), "dimensions": DIMS, "pairs": [f"{f}__{c or '*'}" for f, c in PAIRS],
           "max_leaf_records": args.max_leaf_records}

    # ---- full size: device build, queries through it vs the raw scan ------------------------------------------------
    seg = IndexSegment.synthetic(ctx, "c5", args.rows, sp)
    t0 = time.perf_counter()
    info = seg.build_star_tree(DIMS, PAIRS, max_leaf_records=args.max_leaf_records)
    info["wall_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    out["full"] = {"rows": args.rows, "device_build": info}
    # results are decoded through the synthetic dictionaries alone (value = base + step * dictId)
    dict_only = sb.SegmentData("c5", args.rows, [sb.ColumnData(s["name"], sb.INT, True, 0, s["cardinality"], False, 4, None, None,
                                                               None, dict_values=(s["value_base"] + s["value_step"] * np.arange(
                                                                   s["cardinality"])).astype(np.int32)) for s in sp])
    out["full"]["queries"] = time_queries(pm, {"device_tree": (seg, True), "raw_scan": (seg, False)}, dict_only,
                                          args.steps, args.warmup)
    seg.destroy()

    # ---- host size: both builders on the same data -------------------------------------------------------------------
    n = args.host_rows
    seg = IndexSegment.synthetic(ctx, "c5h", n, sp)
    attached = IndexSegment.synthetic(ctx, "c5h", n, sp)
    host = host_segment(o, seg, sp, n)
    t0 = time.perf_counter()
    st = stb.build_star_tree(host, DIMS, PAIRS, max_leaf_records=args.max_leaf_records)
    host_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    info = seg.build_star_tree(DIMS, PAIRS, max_leaf_records=args.max_leaf_records)
    info["wall_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    assert info["num_star_docs"] == st.num_docs and info["num_nodes"] == len(tree_nodes(st.tree)), (info, st.num_docs)
    nd = len(st.dimensions)
    attached.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                              [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
    out["host_size"] = {"rows": n, "device_build": info,
                        "host_build": {"ms": round(host_ms, 1), "num_star_docs": int(st.num_docs),
                                       "num_nodes": int(len(tree_nodes(st.tree)))},
                        "queries": time_queries(pm, {"device_tree": (seg, True), "host_tree": (attached, True),
                                                     "raw_scan": (seg, False)}, host, args.steps, args.warmup)}
    seg.destroy()
    attached.destroy()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

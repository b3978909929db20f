#!/usr/bin/env python
"""What REGEXP_LIKE costs on ONE GPU: 8 segments of 20 M rows (the same rows in each), each with a STRING column of URL-like values (dictionaries
of 10^4, 10^5 and 10^6 entries, 40-90 bytes each) and an INT metric.  Per dictionary size:

  upload_ms      the first pattern query minus the steady-state one: the compact dictionary copies going to the device
  match_ms       the pattern kernel (pattern_match_kernel), CUDA time from torch.profiler in a run of its own
  scan_ms        the scan kernel's CUDA-event time of the pattern query, and of the same query with the matched values
                 given as an IN list (scan_in_ms): the same leaves, so they should be equal
  step_ms        host clock around execute_segments (ends in a device synchronise), pattern query and IN query

plus the card's name and power limit.  Prints one JSON object."""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

ROWS = 20_000_000
SEGMENTS = 8
PATTERN = "^/api/v[12]/users/[0-9]+/orders$"


def url_dictionary(card, rng):
    words = ["api", "v1", "v2", "users", "orders", "items", "static", "img", "search", "login", "cart", "admin"]
    out = set()
    while len(out) < card:
        k = rng.integers(2, 6)
        parts = [words[i] for i in rng.integers(0, len(words), size=k)]
        out.add("/" + "/".join(parts[:2]) + f"/users/{rng.integers(0, 10**9)}/" + "/".join(parts[2:]) + "orders")
    return sorted(v.encode() for v in out)


def string_column(name, values, rng):
    from oracle import segment_builder as sb
    card = len(values)
    width = max(len(v) for v in values)
    dict_values = np.array(values, dtype=f"S{width}")
    ids = rng.integers(0, card, size=ROWS).astype(np.int32)
    ids[:card] = np.arange(card, dtype=np.int32)   # every entry occurs
    bits = sb.num_bits_per_value(card - 1)
    dbytes = np.frombuffer(dict_values.tobytes(), dtype=np.uint8).copy()
    return sb.ColumnData(name, sb.STRING, True, bits, card, False, width, sb.pack_fixed_bits(ids, bits), dbytes, None,
                         dict_values, ids)


def metric_column(rng):
    from oracle import segment_builder as sb
    ids = rng.integers(0, 1000, size=ROWS).astype(np.int32)
    ids[:1000] = np.arange(1000)
    vals = np.arange(1000, dtype=np.int32) * 7
    return sb.ColumnData("m", sb.INT, True, 10, 1000, False, 4, sb.pack_fixed_bits(ids, 10),
                         np.frombuffer(vals.astype(">i4").tobytes(), dtype=np.uint8).copy(), None, vals, ids)


def timed(pm, segs, q, merge=True):
    t = time.perf_counter()
    b = pm.execute_segments(segs, q, merge=merge)[0]
    return (time.perf_counter() - t) * 1e3, b


def main():
    import torch
    from pinot_b200 import sql
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    from pinot_b200.query import Predicate
    card_info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    out = {"gpu": card_info, "rows": ROWS * SEGMENTS, "pattern": PATTERN}
    for card in (10_000, 100_000, 1_000_000):
        rng = np.random.default_rng(card)
        values = url_dictionary(card, rng)
        cols = [string_column("u", values, rng), metric_column(rng)]   # the same rows in every segment
        segs = [IndexSegment.from_columns(ctx, f"u{card}_{s}", ROWS, cols) for s in range(SEGMENTS)]
        q = sql.parse(f"SELECT COUNT(*), SUM(m) FROM t WHERE REGEXP_LIKE(u, '{PATTERN}')")
        matched = [v for v in values if re.search(PATTERN, v.decode())]
        q_in = sql.parse("SELECT COUNT(*), SUM(m) FROM t WHERE u = 'x'")
        q_in.filter = Predicate("IN", "u", matched) if matched else Predicate("EQ", "u", [b"\x01"])
        before = sum(s.device_bytes() for s in segs)
        first, b = timed(pm, segs, q)
        upload_bytes = sum(s.device_bytes() for s in segs) - before
        for _ in range(3):
            timed(pm, segs, q)
            timed(pm, segs, q_in)
        runs = {"pattern": [], "in": []}
        for _ in range(10):
            runs["pattern"].append(timed(pm, segs, q))
            runs["in"].append(timed(pm, segs, q_in))
        steady = float(np.median([t for t, _ in runs["pattern"]]))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                pm.execute_segments(segs, q, merge=True)
        match = [e.device_time for e in prof.events() if "pattern_match_kernel" in e.name]
        res_p, res_i = runs["pattern"][-1][1], runs["in"][-1][1]
        assert int(res_p.longs[0][0]) == int(res_i.longs[0][0]) and float(res_p.doubles[1][0]) == float(res_i.doubles[1][0])
        out[f"dictionary {card}"] = {
            "matched_values": len(matched), "matched_rows": int(res_p.longs[0][0]),
            "first_query_ms": round(first, 3), "steady_step_ms": round(steady, 3),
            "upload_ms": round(first - steady, 3), "upload_bytes": int(upload_bytes),
            "match_ms": round(float(np.median(match)) / 1e3, 4) if match else None,
            "scan_ms": round(float(np.median([b.device_ms for _, b in runs["pattern"]])), 4),
            "scan_in_ms": round(float(np.median([b.device_ms for _, b in runs["in"]])), 4),
            "step_ms": round(steady, 3),
            "step_in_ms": round(float(np.median([t for t, _ in runs["in"]])), 3),
        }
        for s in segs:
            s.destroy()
    ctx.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

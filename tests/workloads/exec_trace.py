#!/usr/bin/env python
"""The device work of each executor path, as a list that two builds of the library can be compared by.

    python tests/workloads/exec_trace.py --out trace.json [--lib path/to/libpinot_b200.so]
    python tests/workloads/exec_trace.py --compare a.json b.json

Loads the library at --lib (default: the tree's), builds three synthetic segments of 4 M rows (bench.py's columns), runs
every shape once to warm up, then runs each shape once more under torch.profiler with CUDA activities.  Per shape it
writes the ordered device activities (kernel name and grid, memcpy kind and bytes, memset bytes) and a hash of every
result array, group-by rows taken in key order.  The shapes cover each path of pb200_execute (aggregation only with
DISTINCTCOUNT / PERCENTILE / VAR; the dense, shared-memory, hash and specialised GROUP BY tables; a forced count-carrier
retry; merged, per-segment and deferred results; ORDER BY ... LIMIT), selections (a prefix pass with a rescan, a merged
ORDER BY) and a DISTINCT whose prefix pass is rescanned.  Runtime API calls (synchronisations) are not in the list: the library links cudart
statically, so the profiler may not see them.  --compare exits 1 and names the first difference of every shape that
differs."""
import argparse
import ctypes as C
import dataclasses
import hashlib
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

ROWS = 4_000_000
SEGMENTS = 3
RARE = 1 + 2 * 999_990  # c6 > RARE: the top 9 of c6's 1 M values, about 9 matches per million rows (rescans)
HEADLINE = "SELECT SUM(c5), COUNT(*) FROM t WHERE c6 > 500000 GROUP BY c3 LIMIT 100000"
DEFAULTS = {"spec": 1, "smem_groups": 1, "dense_max": 1 << 24, "pack_shift": 0}


def shapes():
    """(name, kind, query text, merge, tuning knobs)"""
    aggs = "SELECT DISTINCTCOUNT(c2), PERCENTILE(c5, 90), VAR_POP(c3) FROM t WHERE c6 > 500000"   # 6 with VAR's limb sums
    return [
        ("aggregation merged", "agg", aggs, True, {}),
        ("aggregation per segment", "agg", aggs, False, {}),
        ("aggregation sum min max", "agg", "SELECT SUM(c5), COUNT(*), MIN(c3), MAX(c6) FROM t WHERE c6 > 500000", True, {}),
        ("group by spec", "agg", HEADLINE, True, {}),
        ("group by shared memory", "agg", HEADLINE, True, {"spec": 0}),
        ("group by dense", "agg", HEADLINE, True, {"smem_groups": 0}),
        ("group by hash", "agg", HEADLINE, True, {"dense_max": 1000}),
        ("group by carrier retry", "agg", HEADLINE, True, {"pack_shift": 60}),
        ("group by per segment", "agg",
         "SELECT DISTINCTCOUNT(c1), PERCENTILE(c2, 50), VAR_SAMP(c1) FROM t GROUP BY c0 LIMIT 100000", False, {}),
        ("group by deferred", "deferred", HEADLINE, True, {}),
        ("group by order by limit", "agg",
         "SELECT SUM(c5), COUNT(*) FROM t WHERE c6 > 500000 GROUP BY c3 ORDER BY SUM(c5) DESC LIMIT 10", True, {}),
        ("selection prefix rescan", "selection", f"SELECT c3, c5 FROM t WHERE c6 > {RARE} LIMIT 100", False, {}),
        ("selection merged order by", "selection", "SELECT c3, c5 FROM t WHERE c6 > 1000000 ORDER BY c5 DESC LIMIT 100", True, {}),
        ("distinct prefix rescan", "distinct", f"SELECT DISTINCT c3 FROM t WHERE c6 > {RARE} LIMIT 100", False, {}),
    ]


def key_order(block):
    """A group-by block with its rows in key order: a hash table's rows come out in slot order, and which slot a key
    takes depends on the order in which the scan's threads insert keys."""
    keys = getattr(block, "keys", None)
    if not isinstance(keys, np.ndarray) or keys.ndim != 2 or len(keys) < 2:
        return block
    perm = np.lexsort(keys.T[::-1])
    rank = np.empty_like(perm)
    rank[perm] = np.arange(len(perm))
    cols = lambda xs: [x[perm] if isinstance(x, np.ndarray) and len(x) == len(perm) else x for x in xs]
    rows = lambda d: {(a, int(rank[r])): v for (a, r), v in d.items()}
    return dataclasses.replace(block, keys=keys[perm], doubles=cols(block.doubles), longs=cols(block.longs),
                               dict_ids=cols(block.dict_ids), distinct=rows(block.distinct),
                               histograms=rows(block.histograms), moments=rows(block.moments))


def digest(x, h):
    if isinstance(x, np.ndarray):
        h.update(str(x.dtype).encode() + str(x.shape).encode() + np.ascontiguousarray(x).tobytes())
    elif dataclasses.is_dataclass(x):
        x = key_order(x)
        for f in dataclasses.fields(x):
            if f.name not in ("device_ms", "handle"):
                h.update(f.name.encode())
                digest(getattr(x, f.name), h)
    elif isinstance(x, dict):
        for k in sorted(x, key=repr):
            h.update(repr(k).encode())
            digest(x[k], h)
    elif isinstance(x, (list, tuple)):
        for v in x:
            digest(v, h)
    else:
        h.update(repr(x).encode())


def run_deferred(pm, segs, q):
    """merge_segments 2 (the groups stay on the device), then pb200_result_finalize"""
    from pinot_b200 import _lib
    from pinot_b200.plan_maker import _marshal_query, _read_result
    ctx, L = pm.ctx, pm.ctx.lib
    hq, _keep = _marshal_query(q, 2, reduce_world=1)
    n = len(segs)
    sh = (C.c_void_p * n)(*[s.handle for s in segs])
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * n)()
    _lib.check(L.pb200h_execute(ctx.handle, C.byref(hq), sh, n, res, kinds))
    _lib.check(L.pb200_result_finalize(ctx.handle, res[0]))
    return [_read_result(ctx, C.c_void_p(res[0]), q, kinds[0], False)]


def run(pm, segs, shape):
    from pinot_b200 import sql
    _, kind, text, merge, knobs = shape
    for k, v in knobs.items():
        pm.ctx.set_tuning(k, v)
    try:
        if kind == "selection":
            return pm.execute_selection(segs, sql.parse_selection(text), merge=merge)
        if kind == "distinct":
            return pm.execute_distinct(segs, sql.parse_distinct(text), merge=merge)
        if kind == "deferred":
            return run_deferred(pm, segs, sql.parse(text))
        return pm.execute_segments(segs, sql.parse(text), merge=merge)
    finally:
        for k in knobs:
            pm.ctx.set_tuning(k, DEFAULTS[k])


def device_activities(trace_path):
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    out = []
    for e in sorted((e for e in events if e.get("ph") == "X"), key=lambda e: (e["ts"], e.get("tid", 0))):
        cat, args = e.get("cat", ""), e.get("args", {})
        name = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", e["name"])
        if cat == "kernel":
            out.append(f"kernel {name} grid {args.get('grid')} block {args.get('block')}")
        elif cat == "gpu_memcpy":
            out.append(f"{name} {args.get('bytes')} B")
        elif cat == "gpu_memset":
            out.append(f"memset {args.get('bytes')} B")
    return out


def trace(lib_path, out_path):
    from pinot_b200 import _lib
    if lib_path:
        _lib.LIB_PATH = os.path.abspath(lib_path)
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment
    torch.cuda.init()
    ctx = B200Context(0)
    pm = B200PlanMaker(ctx)
    segs = [IndexSegment.synthetic(ctx, f"s{s}", ROWS, bench.column_specs(0, s)) for s in range(SEGMENTS)]
    result = {"library": _lib.LIB_PATH, "shapes": {}}
    try:
        for shape in shapes():
            run(pm, segs, shape)
        with tempfile.TemporaryDirectory() as tmp:
            for shape in shapes():
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    blocks = run(pm, segs, shape)
                    torch.cuda.synchronize()
                path = os.path.join(tmp, "trace.json")
                prof.export_chrome_trace(path)
                h = hashlib.sha256()
                digest(blocks, h)
                result["shapes"][shape[0]] = {"activities": device_activities(path), "results": h.hexdigest()}
    finally:
        for s in segs:
            s.destroy()
        ctx.close()
    with open(out_path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({name: len(v["activities"]) for name, v in result["shapes"].items()}))


def compare(a_path, b_path):
    with open(a_path) as f:
        a = json.load(f)["shapes"]
    with open(b_path) as f:
        b = json.load(f)["shapes"]
    bad = 0
    for name in sorted(set(a) | set(b)):
        x, y = a.get(name), b.get(name)
        if x == y:
            print(f"same       {name}: {len(x['activities'])} device activities")
            continue
        bad += 1
        if x is None or y is None:
            print(f"DIFFERENT  {name}: only in {'the second' if x is None else 'the first'} trace")
            continue
        if x["results"] != y["results"]:
            print(f"DIFFERENT  {name}: result hashes differ")
        for i, (p, q) in enumerate(zip(x["activities"], y["activities"])):
            if p != q:
                print(f"DIFFERENT  {name}: activity {i}: {p!r} vs {q!r}")
                break
        else:
            if len(x["activities"]) != len(y["activities"]):
                print(f"DIFFERENT  {name}: {len(x['activities'])} vs {len(y['activities'])} device activities")
    return 1 if bad else 0


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--lib", default=None, help="library to load (default: pinot_b200/libpinot_b200.so)")
    ap.add_argument("--out", default=None, help="JSON file for the trace")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare two traces")
    args = ap.parse_args(argv)
    if args.compare:
        return compare(*args.compare)
    if not args.out:
        ap.error("--out is required")
    trace(args.lib, args.out)
    return 0


if __name__ == "__main__":
    sys.exit(main())

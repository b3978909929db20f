"""Differential check of the scan planner between two builds of the library, without a GPU.

    python tests/host_probe/plan_diff.py --base <git revision> [--shapes 20000] [--seed 20261016]

Builds <base> in a temporary git worktree and the working tree in place, compiles host_probe.cpp (this tree's) against
each, and plans one seeded sweep of shapes with both in separate processes: plan_scan on every shape, plan_selection and
plan_distinct on the same segments, with and without a prefix pass.  probe_plan_dump writes every field of each plan (or
the refusal's status and message), so any difference in a decision, a layout or an error message is a mismatch.  Reports
the shapes planned and refused per planner and every mismatch; exits 1 on any mismatch."""
import argparse
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from pinot_b200 import _lib  # noqa: E402  (ctypes layouts only: the library itself is never loaded here)
from test_scan_plan_cpu import (AVG, COUNT, DISTINCTCOUNT, H100, MAX, MIN, SUM, Q_DEFER_FINALIZE, Q_MERGE,  # noqa: E402
                                Q_NO_COUNT_CARRIER, Q_PER_SEGMENT_FILTER, F, ProbeCol, col)

PERCENTILE, VARPOP, VARSAMP, STDDEVPOP, STDDEVSAMP = range(6, 11)
KINDS = ("scan", "selection", "distinct")
DOC_MASK_MAX_DOCS = 2_000_000          # shapes with a DOC_MASK leaf keep their segments this small
MASK_WORDS = np.zeros(DOC_MASK_MAX_DOCS // 32 + 8, dtype=np.int32)
DUMP_BUFFER = C.create_string_buffer(1 << 24)
KNOBS = (("warps", [6, 8]), ("ctas_per_sm", [1, 2]), ("stages", [0, 2, 3]), ("smem_copies", [0, 1, 2, 4, 32, 3]),
         ("dense_max", [1 << 24, 1 << 16]), ("defer", [0, 1]), ("gb_defer", [0, 1]), ("pack_count", [0, 1]),
         ("table_stride", [0, 1, 4]), ("smem_groups", [0, 1]), ("grid", [0, 0, 77]), ("always_count", [0, 1]),
         ("spec", [0, 1]), ("pack_shift", [0, 40]), ("smem_groups_max", [1 << 24, 5000]), ("skip", [0, 1]),
         ("sparse_max", [4, 0]), ("sparse_max_agg", [-1, 3]))


def _column(rng):
    r = rng.random()
    if r < 0.08:
        c = col(0, raw=True)
    elif r < 0.14:
        c = col(int(rng.integers(1, 500)), stored=_lib.STRING)
    else:
        bits = int(rng.integers(1, 32)) if rng.random() < 0.3 else int(rng.integers(1, 17))
        card = int(rng.integers(1 << (bits - 1), (1 << bits) + 1)) if bits > 1 else int(rng.integers(1, 3))
        card = min(card, (1 << 31) - 1)
        step = int(rng.choice([1, 3, 1000, 1 << 20]))
        base = int(rng.integers(-(1 << 31), (1 << 31) - step * (card - 1))) if step * (card - 1) < (1 << 32) - 1 else -(1 << 31)
        stored = _lib.INT if rng.random() < 0.8 else int(rng.choice([_lib.LONG, _lib.FLOAT, _lib.DOUBLE]))
        c = col(card, base, step if step * (card - 1) < (1 << 32) else 1, stored=stored, shared=rng.random() < 0.3,
                inv=card <= 1 << 16 and rng.random() < 0.3, device_dict=rng.random() < 0.95)
    c["eligible"] = int(rng.choice([1] * 18 + [0, -1])) if c["native"] else -1   # mostly built: VAR plans reach every stage
    return c


def _leaf(rng, cols, k, docs):
    c, r = cols[k], rng.random()
    card = max(c["card"], 1)
    if c["kind"] == _lib.FWD_RAW_FIXEDBYTE and r < 0.6:
        return dict(op=F["RAW_RANGE"], column=k, raw=(float(rng.integers(-1000, 0)), float(rng.integers(0, 1000)), int(rng.integers(0, 16))))
    if r < 0.35:
        lo = int(rng.integers(0, card))
        return dict(op=F["SCAN_RANGE"], column=k, lo=lo, hi=lo + int(rng.integers(0, card)))
    if r < 0.55 and c["bits"] <= 20:
        ids = sorted({int(x) for x in rng.integers(0, card, size=int(rng.integers(0, 4)))})
        return dict(op=F["SCAN_IN"] if rng.random() < 0.5 else F["SCAN_NOT_IN"], column=k, ids=ids)
    if r < 0.7 and c["inv"]:
        return dict(op=F["INV_IN"] if rng.random() < 0.5 else F["INV_NOT_IN"], column=k,
                    ids=[int(x) for x in rng.integers(0, card, size=int(rng.integers(1, 3)))])
    if r < 0.78 and max(docs) <= DOC_MASK_MAX_DOCS:
        need = (max(docs) + 31) // 32
        return dict(op=F["DOC_MASK"], column=0, mask=need - (1 if rng.random() < 0.05 else 0), reserved=int(rng.random() < 0.3))
    if r < 0.86:
        return dict(op=F["DOC_RANGES"], ids=[0, 100] if rng.random() < 0.9 else [5])
    return dict(op=int(rng.choice([F["MATCH_ALL"], F["EMPTY"]])))


def _tree(rng, leaves):
    filt = list(leaves)
    if len(leaves) > 1:
        if rng.random() < 0.5:
            filt.append(dict(op=F["AND"], children=len(leaves)))
        else:   # nested: (l0 OR l1) AND NOT(rest...)
            filt = [leaves[0], leaves[1], dict(op=F["OR"], children=2)] + leaves[2:]
            filt.append(dict(op=F["AND"], children=1 + len(leaves) - 2))
            if rng.random() < 0.5:
                filt.append(dict(op=F["NOT"]))
    return filt


def shape(rng):
    """One input: per-segment columns, docs, query parts, knobs, and the selection / DISTINCT columns."""
    nseg = int(rng.choice([1, 1, 2, 3, 8, 16, 17, 33, 40]))
    ncols = int(rng.integers(1, 13))
    cols = [_column(rng) for _ in range(ncols)]
    seg_cols = [list(cols) for _ in range(nseg)]
    if nseg > 1 and rng.random() < 0.15:    # a column stored differently in some segments
        k = int(rng.integers(0, ncols))
        for s in rng.choice(nseg, size=int(rng.integers(1, nseg)), replace=False):
            seg_cols[int(s)][k] = _column(rng)
    big = rng.random() < 0.05
    docs = [int(rng.integers(1, (1 << 31) - 1 if big else 20_000_000)) for _ in range(nseg)]
    dict_cols = [k for k, c in enumerate(cols) if c["kind"] == _lib.FWD_DICT_FIXEDBIT]
    ngb = int(rng.choice([0, 0, 1, 1, 1, 2, 3]))
    group_by = [int(x) for x in rng.choice(dict_cols, size=min(ngb, len(dict_cols)), replace=False)] if dict_cols else []
    aggs, args = [], []
    for _ in range(int(rng.integers(1, 7))):
        fn = int(rng.choice([COUNT, COUNT, SUM, SUM, SUM, MIN, MAX, AVG, AVG, DISTINCTCOUNT, PERCENTILE] if rng.random() < 0.9 else
                            [VARPOP, VARSAMP, STDDEVPOP, STDDEVSAMP]))
        strings = [k for k, c in enumerate(cols) if c["stored"] == _lib.STRING]
        k = int(rng.choice(strings)) if fn in (MIN, MAX) and strings and rng.random() < 0.3 else int(rng.integers(0, ncols))
        aggs.append((fn, -1 if fn == COUNT else k))
        args.append(float(rng.choice([0.0, 50.0, 99.5, 100.0, -1.0, 101.0])) if rng.random() < 0.1 else float(rng.uniform(0, 100)))
    flags = (Q_MERGE if rng.random() < 0.4 else 0) | (Q_NO_COUNT_CARRIER if rng.random() < 0.05 else 0)
    if flags & Q_MERGE and rng.random() < 0.3:
        flags |= Q_DEFER_FINALIZE
    nleaves = int(rng.integers(0, 5))
    leaf_cols = [int(rng.integers(0, ncols)) for _ in range(nleaves)]
    tree = _tree(rng, [_leaf(rng, cols, k, docs) for k in leaf_cols])
    trees = [tree]
    if nseg > 1 and rng.random() < 0.25:    # one tree per segment, the same shape (rarely not)
        flags |= Q_PER_SEGMENT_FILTER
        trees = [tree] + [_tree(rng, [_leaf(rng, seg_cols[s], k, docs) for k in leaf_cols]) if rng.random() < 0.95 else
                          _tree(rng, [_leaf(rng, seg_cols[s], k, docs) for k in leaf_cols[::-1] + [0]]) for s in range(1, nseg)]
    knobs = {n: int(rng.choice(v)) for n, v in KNOBS if rng.random() < 0.15} if rng.random() < 0.5 else {}
    sel_cols = [int(x) for x in rng.integers(-1 if rng.random() < 0.03 else 0, ncols, size=int(rng.integers(0, 5)))]
    dist_cols = [int(x) for x in rng.choice(ncols, size=int(rng.integers(1, min(ncols, 9) + 1)), replace=False)]
    order = [(int(rng.integers(0, ncols)), int(rng.random() < 0.5)) for _ in range(int(rng.choice([0, 0, 1, 2])))]
    return dict(seg_cols=seg_cols, docs=docs, trees=trees, aggs=aggs, args=args if rng.random() < 0.9 else None,
                group_by=group_by, flags=flags, limit=int(rng.choice([100, 100_000, 5_000_000])),
                reduce_world=int(rng.choice([0, 1, 2, 8])), merged_docs_bound=int(rng.choice([0, 0, 1 << 33, (1 << 31) - 1])),
                knobs=knobs, carrier=bool(rng.random() < 0.9), sel_cols=sel_cols, dist_cols=dist_cols, order=order,
                sel_limit=int(rng.choice([0, 10, 1000, 1 << 20, 2_000_000])), merge=bool(rng.random() < 0.5),
                prefix=bool(rng.random() < 0.5))


def _query(sh, keep):
    nodes = [n for t in sh["trees"] for n in t]
    fn = (_lib.FilterNode * max(len(nodes), 1))()
    for i, n in enumerate(nodes):
        if "mask" in n:
            ids, num = MASK_WORDS.ctypes.data_as(C.POINTER(C.c_int32)), n["mask"]
        else:
            arr = (C.c_int32 * max(len(n.get("ids", [])), 1))(*n.get("ids", []))
            keep.append(arr)
            ids, num = C.cast(arr, C.POINTER(C.c_int32)), len(n.get("ids", []))
        raw = n.get("raw", (0.0, 0.0, 0))
        fn[i] = _lib.FilterNode(n["op"], n.get("column", 0), n.get("children", 0), n.get("lo", 0), n.get("hi", 0), num, ids,
                                raw[0], raw[1], raw[2], n.get("reserved", 0))
    gb = (C.c_int32 * max(len(sh["group_by"]), 1))(*sh["group_by"])
    ag = (_lib.Agg * max(len(sh["aggs"]), 1))(*[_lib.Agg(f, c) for f, c in sh["aggs"]])
    q = _lib.Query(len(sh["trees"][0]), len(sh["group_by"]), len(sh["aggs"]), 100_000, 10_000, sh["flags"], fn, gb, ag,
                   sh["reduce_world"], 0, sh["merged_docs_bound"])
    keep += [fn, gb, ag]
    return q


def _selection(columns, order, limit, keep):
    cs = (C.c_int32 * max(len(columns), 1))(*columns)
    keep.append(cs)
    sel = _lib.Selection(len(columns), C.cast(cs, C.POINTER(C.c_int32)), len(order))
    for i, (c, d) in enumerate(order):
        sel.order[i] = _lib.SelectOrder(c, d)
    sel.limit = limit
    return sel


def dumps(probe, sh):
    """The three planners' dumps of one shape (bytes)."""
    keep = []
    ncols = len(sh["seg_cols"][0])
    cols = (ProbeCol * (len(sh["seg_cols"]) * ncols))()
    for s, cs in enumerate(sh["seg_cols"]):
        for k, c in enumerate(cs):
            cols[s * ncols + k] = ProbeCol(c["kind"], c["stored"], c["bits"], c["card"], int(c["native"]), int(c["shared"]),
                                           int(c["inv"]), c["eligible"], c["hash"], C.cast(c["cbuf"], C.c_void_p) if c["cbuf"] else None,
                                           len(c["host"]) if c["cbuf"] else 0)
    names = (C.c_char_p * max(len(sh["knobs"]), 1))(*[k.encode() for k in sh["knobs"]])
    values = (C.c_int64 * max(len(sh["knobs"]), 1))(*sh["knobs"].values())
    docs = (C.c_int32 * len(sh["docs"]))(*sh["docs"])
    q = _query(sh, keep)
    args = (C.c_double * len(sh["args"]))(*sh["args"]) if sh["args"] else None
    sel = _selection(sh["sel_cols"], sh["order"], sh["sel_limit"], keep)
    dist = _selection(sh["dist_cols"], sh["order"], sh["sel_limit"], keep)
    out = DUMP_BUFFER
    res = []
    for kind, s in ((0, None), (1, sel), (2, dist)):
        n = probe.probe_plan_dump(kind, H100[0], H100[1], names, values, len(sh["knobs"]), C.byref(q), args,
                                  C.byref(s) if s else None, cols, ncols, docs, len(sh["docs"]), int(sh["carrier"]),
                                  int(sh["merge"]), int(sh["prefix"]), out, len(out))
        assert 0 <= n < len(out), n
        res.append(out.raw[:n])
    return res


def worker(probe_path, lib_dir, shapes, seed, only, report):
    probe = C.CDLL(probe_path)
    probe.probe_plan_dump.restype = C.c_int64
    with open("/proc/self/maps") as f:     # this process must plan with exactly the build it was given
        libs = {line.split()[-1] for line in f if line.rstrip().endswith("libpinot_b200.so")}
    assert libs == {os.path.join(lib_dir, "libpinot_b200.so")}, libs
    rng = np.random.default_rng(seed)
    with open(report, "w") as out:
        for i in range(shapes):
            sh = shape(rng)
            if only is not None and i not in only:
                continue
            for kind, d in zip(KINDS, dumps(probe, sh)):
                if only is None:
                    out.write(f"{i} {kind} {int(d.startswith(b'refused'))} {hashlib.sha1(d).hexdigest()}\n")
                else:
                    out.write(f"=== {i} {kind}\n{d.decode(errors='replace')}")


def _build(tree, probe_out):
    subprocess.run([sys.executable, "-m", "pinot_b200.build"], cwd=tree, check=True, stdout=subprocess.DEVNULL)
    libdir = os.path.join(tree, "pinot_b200")
    src = os.path.join(tree, "tests", "host_probe", "host_probe.cpp")   # this tree's probe, beside the base's headers
    if tree != ROOT:
        shutil.copyfile(os.path.join(HERE, "host_probe.cpp"), src)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", probe_out, src, f"-L{libdir}",
                    "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return libdir


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", required=True, help="git revision to compare the working tree with (e.g. HEAD~1)")
    ap.add_argument("--shapes", type=int, default=20_000)
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--worker", nargs=2, help=argparse.SUPPRESS)
    ap.add_argument("--only", help=argparse.SUPPRESS)
    ap.add_argument("--report", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        only = None if a.only is None else {int(x) for x in a.only.split(",")}
        return worker(a.worker[0], a.worker[1], a.shapes, a.seed, only, a.report)

    tmp = tempfile.mkdtemp(prefix="plan_diff_")
    base = os.path.join(tmp, "base")
    rev = subprocess.run(["git", "rev-parse", a.base], cwd=ROOT, check=True, capture_output=True, text=True).stdout.strip()
    subprocess.run(["git", "worktree", "add", "--detach", base, rev], cwd=ROOT, check=True, capture_output=True)
    try:
        builds = {"base": (_build(base, os.path.join(tmp, "base_probe.so")), os.path.join(tmp, "base_probe.so")),
                  "branch": (_build(ROOT, os.path.join(tmp, "branch_probe.so")), os.path.join(tmp, "branch_probe.so"))}

        def run(only=None):
            procs, reports = [], {}
            for name, (libdir, probe) in builds.items():
                reports[name] = os.path.join(tmp, f"{name}.txt")
                cmd = [sys.executable, __file__, "--base", rev, "--worker", probe, libdir, "--shapes", str(a.shapes),
                       "--seed", str(a.seed), "--report", reports[name]] + (["--only", ",".join(map(str, only))] if only else [])
                procs.append(subprocess.Popen(cmd))
            assert all(p.wait() == 0 for p in procs)
            return {n: open(r).read() for n, r in reports.items()}

        rep = run()
        lines = {n: r.splitlines() for n, r in rep.items()}
        assert len(lines["base"]) == len(lines["branch"]) == 3 * a.shapes
        bad = [b.split()[:2] for b, c in zip(lines["base"], lines["branch"]) if b != c]
        print(f"base {rev} vs working tree, {a.shapes} shapes, seed {a.seed}")
        for kind in KINDS:
            rows = [x.split() for x in lines["branch"] if x.split()[1] == kind]
            refused = sum(int(r[2]) for r in rows)
            print(f"  {kind:9s}: {len(rows) - refused} planned, {refused} refused")
        print(f"  mismatches: {len(bad)}")
        if bad:
            full = run(sorted({int(i) for i, _ in bad[:5]}))
            for i, kind in bad[:5]:
                b, c = (full[n].split(f"=== {i} {kind}\n")[1].split("\n=== ")[0].splitlines() for n in ("base", "branch"))
                diff = [(x, y) for x, y in zip(b, c) if x != y] or [("(length)", f"{len(b)} vs {len(c)} lines")]
                print(f"  shape {i} {kind}: first difference\n    base:   {diff[0][0][:300]}\n    branch: {diff[0][1][:300]}")
        return 1 if bad else 0
    finally:
        subprocess.run(["git", "worktree", "remove", "--force", base], cwd=ROOT, capture_output=True)
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    sys.exit(main())

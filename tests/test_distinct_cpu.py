"""CPU tests of DISTINCT queries: the parser (sql.parse_distinct), the planner (pb200::plan_distinct / distinct_rescan
through tests/distinct_probe/distinct_probe.cpp: key layout, table offsets, refusals, prefix planning and the prefix-final
rule on constructed first-occurrence tables), the reference's rules and the Python by-value merge of per-segment
blocks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from distinct_ref import expected, merge_by_value
from pinot_b200 import _lib, sql
from pinot_b200.plan_maker import DistinctResultsBlock, ExecutionStatistics, merge_distinct_blocks
from pinot_b200.query import Predicate

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H100 = (132, 232_448)
SEG, COL = 40, 8
EMPTY = -1   # kDistinctEmpty (~0) as the probe's int64 field holds it
FIELDS = ([(n, 1) for n in ("nres", "table_entries", "prefix", "num_order", "num_rescan")]
          + [("order_key", COL), ("order_desc", COL)]
          + [(n, SEG) for n in ("table_off", "table_size", "scan_docs", "bound", "rescan")]
          + [("cards", SEG * COL), ("mult", SEG * COL)])


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32),
                ("dict_native", C.c_int32), ("dict_hash", C.c_int32)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "distinct_probe", "distinct_probe.cpp")
    out = os.path.join(HERE, "distinct_probe", "libdistinct_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.dist_probe_plan_size.restype = C.c_int64
    assert lib.dist_probe_plan_size() == C.sizeof(ProbePlan)
    lib.dist_probe_plan_distinct.restype = C.c_int32
    lib.dist_probe_plan_distinct.argtypes = [C.c_int32, C.c_int32, C.POINTER(_lib.Query), C.POINTER(_lib.Selection),
                                             C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                             C.c_int32, C.POINTER(C.c_uint64), C.POINTER(ProbePlan)]
    return lib


D, S, R = _lib.FWD_DICT_FIXEDBIT, _lib.STRING, _lib.FWD_RAW_FIXEDBYTE
# columns: 0 INT card 10, 1 STRING card 100, 2 LONG card 1000, 3 raw INT streamed, 4 INT card 4096, 5 INT card 4097,
#          6 INT card 2^20, 7 INT card 2^24
COLS = [(D, _lib.INT, 4, 10, 1, 1), (D, S, 7, 100, 0, 2), (D, _lib.LONG, 10, 1000, 1, 3), (R, _lib.INT, 32, 0, 0, 0),
        (D, _lib.INT, 12, 4096, 1, 5), (D, _lib.INT, 13, 4097, 1, 6), (D, _lib.INT, 20, 1 << 20, 1, 7),
        (D, _lib.INT, 24, 1 << 24, 1, 8)]


def run(probe, num_docs, columns, limit, merge=False, prefix=True, order=(), tables=None, cols=None):
    n = len(num_docs)
    pc = (ProbeCol * (n * len(COLS)))()
    for s in range(n):
        for k, c in enumerate(cols[s] if cols is not None else COLS):
            pc[s * len(COLS) + k] = ProbeCol(*c)
    fn = (_lib.FilterNode * 1)()
    fn[0] = _lib.FilterNode(5, 0, 0, 1, 5, 0, None, 0.0, 0.0, 0, 0)   # SCAN_RANGE on column 0
    q = _lib.Query(1, 0, 0, 0, 0, 0, fn, None, None, 0, 0, 0)
    cc = (C.c_int32 * max(1, len(columns)))(*columns)
    sel = _lib.Selection(len(columns), cc, len(order))
    for k, (col, desc) in enumerate(order):
        sel.order[k] = _lib.SelectOrder(col, int(desc))
    sel.limit = limit
    nd = (C.c_int32 * n)(*num_docs)
    t = None if tables is None else (C.c_uint64 * max(1, len(tables)))(*[int(x) for x in tables])
    out = ProbePlan()
    rc = probe.dist_probe_plan_distinct(*H100, C.byref(q), C.byref(sel), pc, len(COLS), nd, n, int(merge), int(prefix), t,
                                        C.byref(out))
    return rc, out


def test_key_layout_and_tables(probe):
    rc, p = run(probe, [100, 200, 300], [0, 1, 2], 10)
    assert rc == 0 and p.nres == 3
    assert [p.cards[k] for k in range(3)] == [10, 100, 1000] and [p.mult[k] for k in range(3)] == [1, 10, 1000]
    assert list(p.table_size[:3]) == [10 ** 6] * 3 and list(p.table_off[:3]) == [0, 10 ** 6, 2 * 10 ** 6]
    assert p.table_entries == 3 * 10 ** 6
    rc, p = run(probe, [100, 200, 300], [2, 0], 10, merge=True)
    assert rc == 0 and p.nres == 1 and p.table_size[0] == 10_000 and p.table_entries == 10_000
    assert [p.mult[k] for k in range(2)] == [1, 1000]
    # order items map onto key columns; a repeated column orders nothing and is dropped
    rc, p = run(probe, [100], [0, 1, 2], 10, order=[(2, True), (0, False), (2, False)])
    assert rc == 0 and p.num_order == 2 and list(p.order_key[:2]) == [2, 0] and list(p.order_desc[:2]) == [1, 0]


def test_refusals(probe):
    assert run(probe, [100], [3], 10)[0] == _lib.E_UNSUPPORTED                     # streamed raw column: no dictIds
    assert run(probe, [100], [4, 4], 10)[0] == 0                                   # 4096 x 4096 = 2^24 fits
    assert run(probe, [100], [7], 10)[0] == 0
    assert run(probe, [100], [4, 5], 10)[0] == _lib.E_UNSUPPORTED                  # 4096 x 4097
    assert run(probe, [100], [7, 0], 10)[0] == _lib.E_UNSUPPORTED
    assert run(probe, [100] * 8, [7], 10)[0] == 0                                  # 8 x 2^24 = 2^27 entries
    assert run(probe, [100] * 9, [7], 10)[0] == _lib.E_UNSUPPORTED                 # above 2^27 entries in one call
    assert run(probe, [100] * 9, [7], 10, merge=True)[0] == 0                      # merged: one table
    assert run(probe, [100], [0] * 7, 1)[0] == 0                                   # 10^7 keys
    assert run(probe, [100], [0] * 9, 1)[0] == _lib.E_UNSUPPORTED                  # more than 8 columns
    assert run(probe, [100], [0], _lib.MAX_SELECT_LIMIT + 1)[0] == _lib.E_UNSUPPORTED
    assert run(probe, [100], [0, 1], 10, order=[(2, False)])[0] == _lib.E_INVALID   # order item outside the columns
    assert run(probe, [100], [], 10)[0] == _lib.E_INVALID
    assert run(probe, [1] * 65_536, [0], 1)[0] == _lib.E_UNSUPPORTED
    # merged over different dictionaries: refused; per segment fine
    other = [COLS, [c if k != 1 else c[:5] + (99,) for k, c in enumerate(COLS)]]
    assert run(probe, [100, 100], [0, 1], 10, merge=True, cols=other)[0] == _lib.E_UNSUPPORTED
    assert run(probe, [100, 100], [0, 1], 10, merge=False, cols=other)[0] == 0
    assert run(probe, [100, 100], [0], 10, merge=True, cols=other)[0] == 0         # column 0 has one dictionary


def test_prefix_planning(probe):
    big, small = 3_000_000, 500_000
    rc, p = run(probe, [big, small, big], [0], 10)
    assert rc == 0 and p.prefix == 1
    pre = p.scan_docs[0]
    assert pre >= 1 << 20 and pre < big and list(p.scan_docs[:3]) == [pre, small, pre]
    assert list(p.bound[:3]) == [pre, EMPTY, (2 << 32) | pre]                     # per segment: its own cut
    rc, p = run(probe, [small, big, big], [0], 10, merge=True)
    assert rc == 0 and p.bound[0] == (1 << 32) | pre                              # merged: the earliest truncated segment
    rc, p = run(probe, [big], [0], 10, order=[(0, True)])
    assert rc == 0 and p.prefix == 0 and p.scan_docs[0] == big and p.bound[0] == EMPTY


def _tables(probe, docs, merge, keys_per_seg, columns=(0,)):
    """First-occurrence tables of the constructed keys: keys_per_seg[s] = [(key, doc)] of segment s."""
    rc, p = run(probe, docs, list(columns), 1, merge=merge)
    assert rc == 0
    t = np.full(p.table_entries, (1 << 64) - 1, dtype=np.uint64)
    for s, kd in enumerate(keys_per_seg):
        off = p.table_off[0 if merge else s]
        for key, doc in kd:
            v = (s << 32) | doc
            t[off + key] = min(int(t[off + key]), v)
    return t


def test_prefix_final_rule(probe):
    big, small = 3_000_000, 500_000
    _, p = run(probe, [big], [0], 1)
    pre = p.scan_docs[0]
    # one segment: 3 keys first occurring below the prefix end, one exactly at it (not below)
    t = _tables(probe, [big], False, [[(1, 0), (2, 5), (3, pre - 1), (4, pre)]])
    for limit, rescan in ((2, 0), (3, 0), (4, 1), (5, 1)):
        rc, p = run(probe, [big], [0], limit, tables=t)
        assert rc == 0 and p.num_rescan == rescan, limit
    # merged, the truncated segment first / middle / last: entries of earlier (fully scanned) segments count, entries
    # of later segments do not
    for layout, cut in (([big, small, small], 0), ([small, big, small], 1), ([small, small, big], 2)):
        keys = [[(1, 3)], [(2, 3)], [(3, 3)]]
        keys[cut] = [(5, 7), (6, pre + 1)]
        t = _tables(probe, layout, True, keys)
        below = cut + 1   # keys of the segments before the cut + the cut segment's key below its prefix end
        for limit in (below - 1, below, below + 1):
            if limit < 0:
                continue
            rc, p = run(probe, layout, [0], limit, merge=True, tables=t)
            assert rc == 0 and p.num_rescan == (1 if limit > below else 0), (layout, limit)
            if p.num_rescan:
                assert p.rescan[0] == cut
        # per segment: each truncated segment decides alone
        t = _tables(probe, layout, False, keys)
        rc, p = run(probe, layout, [0], 2, merge=False, tables=t)
        assert rc == 0 and p.num_rescan == 1 and p.rescan[0] == cut             # 1 key below its prefix end < 2
        rc, p = run(probe, layout, [0], 1, merge=False, tables=t)
        assert rc == 0 and p.num_rescan == 0
    # two truncated segments merged: both are rescanned when the result is not final
    t = _tables(probe, [big, big], True, [[(1, 0)], [(2, 0)]])
    rc, p = run(probe, [big, big], [0], 2, merge=True, tables=t)
    assert rc == 0 and p.num_rescan == 2 and list(p.rescan[:2]) == [0, 1]


def test_prefix_rule_is_exact():
    """Brute force: whenever the rule says final, the first `limit` tuples over the prefix-scanned docs equal those over
    all docs (merged, random positions of the cut)."""
    rng = np.random.default_rng(4)
    for case in range(300):
        nseg = int(rng.integers(1, 4))
        docs = [int(rng.integers(1, 40)) for _ in range(nseg)]
        pre = [int(rng.integers(1, d + 1)) for d in docs]           # scanned prefix (== docs: whole segment)
        keys = [rng.integers(0, int(rng.integers(1, 12)), size=d) for d in docs]
        limit = int(rng.integers(0, 8))

        def first(scanned):
            seen = {}
            for s in range(nseg):
                for d in range(scanned[s]):
                    seen.setdefault(int(keys[s][d]), (s, d))
            return sorted(seen.items(), key=lambda kv: kv[1])
        cut = next((s for s in range(nseg) if pre[s] < docs[s]), None)
        part = first(pre)
        if cut is None:
            continue
        below = sum(1 for _, occ in part if occ < (cut, pre[cut]))
        if below >= limit:
            assert part[:limit] == first(docs)[:limit], case


def test_parser():
    q = sql.parse_distinct("SELECT DISTINCT a, b FROM t WHERE c > 3 AND NOT d IN (1, 2) ORDER BY b DESC, a LIMIT 5")
    assert q.columns == ["a", "b"] and q.limit == 5 and q.order_by == [("b", False), ("a", True)] and q.table == "t"
    assert q.filter.type == "AND"
    q = sql.parse_distinct("select distinct a from t")
    assert q.columns == ["a"] and q.limit == 10 and q.filter is None and q.order_by == []
    for bad in ("SELECT DISTINCT * FROM t", "SELECT DISTINCT SUM(a) FROM t", "SELECT DISTINCT a FROM t GROUP BY a",
                "SELECT DISTINCT a FROM t ORDER BY b", "SELECT DISTINCT a FROM t LIMIT -1", "SELECT DISTINCT FROM t",
                "SELECT DISTINCT a FROM t extra", "SELECT DISTINCT lower(a) FROM t"):
        with pytest.raises(sql.SqlError):
            sql.parse_distinct(bad)
    assert sql.is_distinct("SELECT DISTINCT a FROM t") and not sql.is_distinct("SELECT a FROM t")
    assert not sql.is_distinct("SELECT COUNT(*) FROM t")
    # the other parsers stay as they are
    with pytest.raises(sql.SqlError):
        sql.parse("SELECT DISTINCT a FROM t")


def _block(r, names):
    return DistinctResultsBlock(names, r["columns"], r["doc_ids"].astype(np.int32), r["segment_index"].astype(np.int32),
                                ExecutionStatistics(r["matched"], 0, 0, 0))


def test_by_value_merge(oracle):
    rng = np.random.default_rng(8)
    for case in range(12):
        segs = []
        for i in range(int(rng.integers(1, 5))):
            n = int(rng.integers(1, 120))
            segs.append(oracle.build_segment(f"dm{case}_{i}", {
                "a": rng.integers(0, 5, size=n).astype(np.int32),
                "s": np.array([b"x", b"yy", b"z", b"ab"])[rng.integers(0, 4, size=n)],
                "f": (rng.integers(-4, 4, size=n) / 2.0).astype(np.float32)}))
        flt = Predicate("RANGE", "a", [], 1, None, True, True)
        cols = ["s", "a", "f"][: int(rng.integers(1, 4))]
        order = [[], [(cols[0], True)], [(cols[-1], False), (cols[0], True)]][case % 3]
        limit = int(rng.integers(0, 12))
        per = expected(oracle, segs, flt, cols, limit, False, order)
        merged = expected(oracle, segs, flt, cols, limit, True, order)[0]
        ref = merge_by_value(per, cols, order, limit)
        got = merge_distinct_blocks([_block(r, cols) for r in per], order, limit)
        for w in (ref, merged):
            assert list(got.segment_index) == list(w["segment_index"]) and list(got.doc_ids) == list(w["doc_ids"]), case
            for g, e in zip(got.columns, w["columns"]):
                assert list(g) == list(e), case
        assert got.stats.num_docs_scanned == merged["matched"]


def test_reference_rules(oracle):
    """distinct_ref against a plain Python walk over (segment, doc): first occurrences, ORDER BY with ties."""
    rng = np.random.default_rng(6)
    segs = [oracle.build_segment(f"dr{i}", {"a": rng.integers(0, 4, size=n).astype(np.int32),
                                            "b": rng.integers(-2, 2, size=n).astype(np.int64) * 10 ** 12})
            for i, n in enumerate((60, 9, 45))]
    from exact_ref import column_values
    for merge in (False, True):
        for order in ([], [("b", False)], [("a", True), ("b", False)]):
            got = expected(oracle, segs, None, ["a", "b"], 100, merge, order)
            groups = [list(range(3))] if merge else [[s] for s in range(3)]
            for g, w in zip(groups, got):
                seen = {}
                for s in g:
                    a = column_values(oracle, segs[s], "a", np.arange(segs[s].num_docs))
                    b = column_values(oracle, segs[s], "b", np.arange(segs[s].num_docs))
                    for d in range(segs[s].num_docs):
                        seen.setdefault((int(a[d]), int(b[d])), (s, d))
                rows = sorted(seen.items(), key=lambda kv: kv[1])
                for col, asc in reversed(order):
                    k = ["a", "b"].index(col)
                    rows.sort(key=lambda kv: kv[0][k], reverse=not asc)
                assert list(zip(w["segment_index"], w["doc_ids"])) == [occ for _, occ in rows], (merge, order)

"""CPU tests of selection queries: the parser (sql.parse_selection), the planner (pb200::plan_selection through
tests/selection_probe/selection_probe.cpp: mask layout, prefix and rescan decision, refusals) and the reference
(selection_ref) on a small segment."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pinot_b200 import _lib, sql
from pinot_b200.query import Predicate
from selection_ref import expected

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H100 = (132, 232_448)
SEL_DICT_I32, SEL_DICT_I64, SEL_DICT_F32, SEL_DICT_F64, SEL_DICT_ID, SEL_RAW_I32, SEL_RAW_F32 = range(7)
SEG, COL, CHUNK = 40, 8, 4
FIELDS = ([(n, 1) for n in ("tile_rows", "prefix", "mask_words", "num_chunks", "limit", "num_rescan")]
          + [("kinds", COL), ("chunk_word_off", CHUNK), ("chunk_total_tiles", CHUNK)]
          + [(n, SEG) for n in ("mask_word_off", "scan_docs", "num_tiles", "first_tile", "in_filter", "rescan")])


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32),
                ("dict_native", C.c_int32), ("reserved", C.c_int32)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "selection_probe", "selection_probe.cpp")
    out = os.path.join(HERE, "selection_probe", "libselection_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.sel_probe_plan_size.restype = C.c_int64
    assert lib.sel_probe_plan_size() == C.sizeof(ProbePlan)
    lib.sel_probe_plan_selection.restype = C.c_int32
    lib.sel_probe_plan_selection.argtypes = [C.c_int32, C.c_int32, C.POINTER(_lib.Query), C.POINTER(_lib.Selection),
                                             C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                             C.POINTER(C.c_int64), C.POINTER(ProbePlan)]
    return lib


# columns: 0 INT dict (card 1000), 1 LONG dict, 2 FLOAT dict, 3 DOUBLE dict, 4 STRING, 5 raw INT, 6 raw FLOAT, 7 INT without device dict
COLS = [(_lib.FWD_DICT_FIXEDBIT, _lib.INT, 10, 1000, 1), (_lib.FWD_DICT_FIXEDBIT, _lib.LONG, 4, 9, 1),
        (_lib.FWD_DICT_FIXEDBIT, _lib.FLOAT, 3, 5, 1), (_lib.FWD_DICT_FIXEDBIT, _lib.DOUBLE, 3, 5, 1),
        (_lib.FWD_DICT_FIXEDBIT, _lib.STRING, 2, 3, 0), (_lib.FWD_RAW_FIXEDBYTE, _lib.INT, 32, 0, 0),
        (_lib.FWD_RAW_FIXEDBYTE, _lib.FLOAT, 32, 0, 0), (_lib.FWD_DICT_FIXEDBIT, _lib.INT, 10, 1000, 0)]


def run(probe, num_docs, columns, limit, prefix=True, matches=None, leaf=True, order=0, cols=COLS):
    n = len(num_docs)
    pc = (ProbeCol * (n * len(cols)))()
    for s in range(n):
        for k, c in enumerate(cols):
            pc[s * len(cols) + k] = ProbeCol(*c, 0)
    fn = (_lib.FilterNode * 1)()
    fn[0] = _lib.FilterNode(5, 0, 0, 10, 500, 0, None, 0.0, 0.0, 0, 0)   # SCAN_RANGE on column 0
    q = _lib.Query(1 if leaf else 0, 0, 0, 0, 0, 0, fn, None, None, 0, 0, 0)
    cc = (C.c_int32 * max(1, len(columns)))(*columns)
    sel = _lib.Selection(len(columns), cc, order)
    sel.limit = limit
    nd = (C.c_int32 * n)(*num_docs)
    m = (C.c_int64 * n)(*matches) if matches is not None else None
    out = ProbePlan()
    rc = probe.sel_probe_plan_selection(*H100, C.byref(q), C.byref(sel), pc, len(cols), nd, n, int(prefix), m, C.byref(out))
    return rc, out


def test_mask_layout_per_segment(probe):
    docs = [1, 31, 32, 1025, 49_157, 196_609]
    rc, p = run(probe, docs, [0, 1, 2, 3, 4, 5, 6], 10)
    assert rc == 0
    assert list(p.kinds[:7]) == [SEL_DICT_I32, SEL_DICT_I64, SEL_DICT_F32, SEL_DICT_F64, SEL_DICT_ID, SEL_RAW_I32, SEL_RAW_F32]
    t = p.tile_rows
    tiles = [(d + t - 1) // t for d in docs]
    assert p.prefix == 0 and list(p.num_tiles[:6]) == tiles and list(p.scan_docs[:6]) == docs
    # doc d of segment s: bit d % 32 of word mask_word_off[s] + d // 32; segments back to back in tile order
    assert list(p.mask_word_off[:6]) == [sum(tiles[:s]) * t // 32 for s in range(6)]
    assert p.mask_words == sum(tiles) * t // 32
    assert p.num_chunks == 1 and p.chunk_word_off[0] == 0 and p.chunk_total_tiles[0] == sum(tiles)
    assert list(p.in_filter[:6]) == docs   # one scan leaf


def test_two_launch_chunks(probe):
    docs = [5000 + 100 * i for i in range(17)]
    rc, p = run(probe, docs, [0], 3)
    assert rc == 0 and p.num_chunks == 2
    assert p.chunk_word_off[0] == 0 and p.chunk_word_off[1] == p.mask_word_off[16]
    assert p.first_tile[16] == 0 and p.first_tile[15] == sum(p.num_tiles[:15])
    assert p.chunk_total_tiles[0] + p.chunk_total_tiles[1] == p.mask_words * 32 // p.tile_rows


def test_prefix_and_rescan(probe):
    big, small = 3_000_000, 500_000
    rc, p = run(probe, [big, small, big], [0], 10, matches=[10, 3, 9])
    assert rc == 0 and p.prefix == 1
    t = p.tile_rows
    pre = -(-(1 << 20) // t)
    assert list(p.num_tiles[:3]) == [pre, -(-small // t), pre]
    assert list(p.scan_docs[:3]) == [pre * t, small, pre * t] and pre * t >= 1 << 20
    assert list(p.in_filter[:3]) == [pre * t, small, pre * t]
    # segment 2's prefix held 9 < 10 matches: scanned again in full; segment 1 was scanned whole, segment 0 has enough
    assert p.num_rescan == 1 and p.rescan[0] == 2
    # a LIMIT beyond half the default prefix lengthens the prefix
    rc, p = run(probe, [big], [0], 800_000, matches=[0])
    assert rc == 0 and p.scan_docs[0] >= 1_600_000 and p.num_rescan == 1
    rc, p = run(probe, [big], [0], 10, prefix=False, matches=[0])
    assert rc == 0 and p.prefix == 0 and p.scan_docs[0] == big and p.num_rescan == 0


def test_refusals(probe):
    assert run(probe, [100], [0], _lib.MAX_SELECT_LIMIT + 1)[0] == _lib.E_UNSUPPORTED
    assert run(probe, [100], [0], _lib.MAX_SELECT_LIMIT)[0] == 0
    assert run(probe, [100], [0], -1)[0] == _lib.E_INVALID
    assert run(probe, [100], [9], 10)[0] == _lib.E_INVALID                 # no such column
    assert run(probe, [100], [7], 10)[0] == _lib.E_UNSUPPORTED             # no device dictionary
    assert run(probe, [100], [0], 10, order=9)[0] == _lib.E_INVALID         # more than 8 order items
    assert run(probe, [70_000] * 4, [0], 10)[0] == 0
    assert run(probe, [100], [], 0)[0] == 0                                # LIMIT 0, no column: statistics only


def test_parser():
    q = sql.parse_selection("SELECT a, b FROM t WHERE c > 3 AND NOT d IN (1, 2) LIMIT 5")
    assert q.columns == ["a", "b"] and q.limit == 5 and q.order_by == [] and q.table == "t"
    assert q.filter.type == "AND"
    q = sql.parse_selection("SELECT * FROM t")
    assert q.columns is None and q.limit == 10 and q.filter is None
    q = sql.parse_selection("SELECT ts FROM t WHERE x BETWEEN 1 AND 2 ORDER BY ts DESC, y, z ASC LIMIT 0")
    assert q.order_by == [("ts", False), ("y", True), ("z", True)] and q.limit == 0
    q = sql.parse_selection("SELECT a FROM t WHERE a IN (3, 3, 4) OR a = 5")   # optimize_filter merges EQ / IN
    assert isinstance(q.filter, Predicate) and q.filter.type == "IN"
    for bad in ("SELECT SUM(a) FROM t", "SELECT a FROM t GROUP BY a", "SELECT a FROM t LIMIT -1", "SELECT a FROM t LIMIT 2.5",
                "SELECT a FROM t extra", "SELECT FROM t"):
        with pytest.raises(sql.SqlError):
            sql.parse_selection(bad)
    assert sql.is_selection("SELECT a, b FROM t") and sql.is_selection("SELECT * FROM t WHERE a = 1")
    assert not sql.is_selection("SELECT COUNT(*) FROM t") and not sql.is_selection("SELECT a, MAX(b) FROM t GROUP BY a")
    with pytest.raises(sql.SqlError):   # the aggregation parser keeps refusing selections
        sql.parse("SELECT a FROM t")


def test_reference_rules(oracle):
    rng = np.random.default_rng(3)
    segs = [oracle.build_segment(f"sr{i}", {"a": rng.integers(0, 10, size=n).astype(np.int32),
                                            "s": np.array([b"x", b"yy", b"z"])[rng.integers(0, 3, size=n)]})
            for i, n in enumerate((50, 7, 40))]
    flt = Predicate("RANGE", "a", [], 5, None, True, True)
    per = expected(oracle, segs, flt, ["a", "s"], 4, merge=False)
    for s, r in enumerate(per):
        a = np.asarray(sb_values(oracle, segs[s], "a"))
        st = np.asarray(sb_values(oracle, segs[s], "s"))
        docs = np.flatnonzero(a >= 5)
        assert list(r["doc_ids"]) == list(docs[:4]) and set(r["segment_index"]) <= {s}
        assert list(r["columns"][0]) == list(a[docs[:4]])
        assert list(r["columns"][1]) == [v.decode() for v in st[docs[:4]]]
    merged = expected(oracle, segs, flt, ["a"], 9, merge=True)[0]
    take = []
    for s, r in enumerate(expected(oracle, segs, flt, ["a"], 9, merge=False)):
        take += [(s, d) for d in r["doc_ids"]]
    assert list(zip(merged["segment_index"], merged["doc_ids"])) == take[:9]
    assert merged["matched"] == sum(r["matched"] for r in per)


def test_order_by_plans_every_doc(probe):
    big = 3_000_000
    rc, p = run(probe, [big, 40], [0, 4], 10, order=2, matches=[0, 0])
    assert rc == 0 and p.prefix == 0 and p.scan_docs[0] == big and p.scan_docs[1] == 40 and p.num_rescan == 0


def test_segment_cap(probe):
    rc, _ = run(probe, [1] * 65_536, [0], 1, cols=COLS[:1])
    assert rc == _lib.E_UNSUPPORTED
    rc, _ = run(probe, [1] * 65_535, [0], 1, cols=COLS[:1])
    assert rc == 0


def test_order_by_reference(oracle):
    """The ORDER BY rule of selection_ref: value order per item, DESC reversed, ties by doc id (merged: segment, doc id),
    checked against a plain Python sort of the same rows; and the merged top equals the merge of the per-segment tops."""
    rng = np.random.default_rng(5)
    segs = []
    for i, n in enumerate((300, 1, 250)):
        segs.append(oracle.build_segment(f"so{i}", {
            "a": rng.integers(0, 4, size=n).astype(np.int32),                                     # low cardinality
            "b": rng.integers(-3, 3, size=n).astype(np.int64) * (10 ** 12),
            "s": np.array([b"x", b"yy", b"y", b"ab"])[rng.integers(0, 4, size=n)],
            "f": (rng.integers(-8, 8, size=n) / 2.0).astype(np.float32)}))
    flt = Predicate("RANGE", "b", [], -2 * 10 ** 12, None, True, True)
    for order_by in ([("a", True)], [("a", False), ("s", True)], [("s", False), ("f", True), ("b", False)]):
        for merge in (False, True):
            got = expected(oracle, segs, flt, ["b", "a"], 7, merge, order_by)
            rows = []
            for s, seg in enumerate(segs):
                b = np.asarray(sb_values(oracle, seg, "b"))
                for d in np.flatnonzero(b >= -2 * 10 ** 12):
                    vals = [sb_values(oracle, seg, c)[d] for c, _ in order_by]
                    rows.append((s, int(d), vals))
            groups = [rows] if merge else [[r for r in rows if r[0] == s] for s in range(len(segs))]
            for g, want in zip(groups, got):
                import functools

                def cmp(x, y):
                    for k, (_, asc) in enumerate(order_by):
                        if x[2][k] != y[2][k]:
                            c = -1 if x[2][k] < y[2][k] else 1
                            return c if asc else -c
                    return -1 if (x[0], x[1]) < (y[0], y[1]) else 1
                top = sorted(g, key=functools.cmp_to_key(cmp))[:7]
                assert list(zip(want["segment_index"], want["doc_ids"])) == [(s, d) for s, d, _ in top], (order_by, merge)
    per = expected(oracle, segs, flt, ["a"], 7, False, [("s", True)])
    merged = expected(oracle, segs, flt, ["a"], 7, True, [("s", True)])[0]
    union = sorted(((sb_values(oracle, segs[s], "s")[d], s, d) for r in per for s, d in zip(r["segment_index"], r["doc_ids"])))
    assert [(s, d) for _, s, d in union[:7]] == list(zip(merged["segment_index"], merged["doc_ids"]))


def sb_values(oracle, seg, column):
    from exact_ref import column_values
    return column_values(oracle, seg, column, np.arange(seg.num_docs))

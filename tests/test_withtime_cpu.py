"""CPU tests of FIRSTWITHTIME / LASTWITHTIME(v, t, 'T'): the parser (canonical text, case variants, ORDER BY and HAVING
resolution, refusals), the planner (pb200::plan_scan through tests/withtime_probe/withtime_probe.cpp: the time column's
slot, the key code, the doc bases, no shared-memory table and no specialised kernel, plans without the new functions
unchanged, every refusal with its code), the per-row reference on an oracle-built segment, the CLI's by-value merge
with ties across segments, and the multi-GPU refusal."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from withtime_ref import withtime
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import ExecutionStatistics, ResultsBlock
from pinot_b200.query import Aggregation, Predicate, QueryContext, withtime_pick

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H100 = (132, 232_448)
FIRST, LAST = 11, 12
SUM, COUNT, MIN, MAX, P = 1, 0, 2, 3, 6


# ---- parser --------------------------------------------------------------------------------------------------------
def test_parse_and_canonical_text():
    q = sql.parse("SELECT LastWithTime(v, ts, 'int'), FIRSTWITHTIME(s, DATETRUNC('hour', ts), 'String'), "
                  "lastwithtime(b, t, 'BOOLEAN'), COUNT(*) FROM t GROUP BY g")
    a = q.aggregations
    assert [(x.function, x.column, x.time_column, x.value_type) for x in a[:3]] == [
        ("LASTWITHTIME", "v", "ts", "INT"), ("FIRSTWITHTIME", "s", "datetrunc('HOUR',ts)", "STRING"),
        ("LASTWITHTIME", "b", "t", "BOOLEAN")]
    assert str(a[0]) == "lastwithtime(v,ts,'INT')"
    assert str(a[1]) == "firstwithtime(s,datetrunc('HOUR',ts),'STRING')"
    assert sql.having_name(a[0]) == "lastwithtime(v,ts,'INT')"
    assert not sql.is_selection("SELECT LASTWITHTIME(v, ts, 'INT') FROM t")


def test_order_by_and_having_resolution():
    q = sql.parse("SELECT COUNT(*), lastwithtime(v, ts, 'LONG') FROM t GROUP BY g HAVING LASTWITHTIME(v, ts, 'long') > 5 "
                  "AND firstwithtime(v, ts, 'LONG') < 100 ORDER BY LASTWITHTIME(v, ts, 'Long') DESC, COUNT(*) LIMIT 3")
    assert sql.resolve_order_by(q) == [("AGG", 1, False), ("AGG", 0, True)]
    assert q.aggregations[2].hidden and q.aggregations[2].function == "FIRSTWITHTIME"
    assert sql.resolve_having(q) == [("RANGE", 1, 5.0, None, False, True), ("RANGE", 2, None, 100.0, True, False), ("AND", 2)]


@pytest.mark.parametrize("text", [
    "SELECT LASTWITHTIME(v, ts) FROM t",                      # missing type
    "SELECT LASTWITHTIME(v, ts, INT) FROM t",                 # not a literal
    "SELECT LASTWITHTIME(v, ts, 4) FROM t",                   # not a string literal
    "SELECT LASTWITHTIME(v, ts, 'CHAR') FROM t",              # not a type
    "SELECT LASTWITHTIME(v) FROM t",                          # argument count
    "SELECT LASTWITHTIME(v, ts, 'INT', 'INT') FROM t",
    "SELECT FIRSTWITHTIME(*) FROM t",
    "SELECT LASTWITHTIME(s, ts, 'STRING') FROM t GROUP BY g ORDER BY LASTWITHTIME(s, ts, 'STRING')",
    "SELECT LASTWITHTIME(s, ts, 'STRING') FROM t GROUP BY g HAVING LASTWITHTIME(s, ts, 'STRING') > 1",
])
def test_parse_refusals(text):
    with pytest.raises(sql.SqlError):
        q = sql.parse(text)
        sql.resolve_order_by(q)
        sql.resolve_having(q)


# ---- planner probe -------------------------------------------------------------------------------------------------
class ProbeCol(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("fwd_kind", "stored_type", "bits", "cardinality", "dict_native", "dict_hash")]


class ProbePlan(C.Structure):
    _fields_ = ([(n, C.c_int64) for n in ("nres", "group_by", "hashed", "groups", "smem_groups", "spec", "num_slots",
                                          "num_agg_codes", "warps", "ctas_per_sm", "smem_bytes")]
                + [("slot_col", C.c_int64 * 12)]
                + [(n, C.c_int64 * 6) for n in ("code_agg", "code_fn", "code_vk", "code_slot_words", "wt_time", "val_kind")]
                + [("doc_base", (C.c_int64 * 6) * 20)])


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "withtime_probe", "withtime_probe.cpp")
    out = os.path.join(HERE, "withtime_probe", "libwithtime_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.wt_probe_plan_size.restype = C.c_int64
    assert lib.wt_probe_plan_size() == C.sizeof(ProbePlan)
    lib.wt_probe_segdesc_size.restype = C.c_int64
    lib.wt_probe_smem_header_size.restype = C.c_int64
    lib.wt_probe_key.restype = C.c_uint64
    lib.wt_probe_key.argtypes = [C.c_uint32, C.c_uint32]
    lib.wt_probe_plan_scan.restype = C.c_int32
    lib.wt_probe_plan_scan.argtypes = [C.c_int32, C.c_int32, C.POINTER(_lib.Query), C.POINTER(_lib.AggArg),
                                       C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int64,
                                       C.POINTER(ProbePlan), C.c_void_p]
    return lib


D, R = _lib.FWD_DICT_FIXEDBIT, _lib.FWD_RAW_FIXEDBYTE
# 0 INT card 10 (group key), 1 LONG card 1000 (time), 2 DOUBLE card 2^20, 3 STRING card 100, 4 raw INT streamed,
# 5 INT card 5000 (time), 6 FLOAT card 3, 7 LONG card 2^20 with another dictionary
COLS = [(D, _lib.INT, 4, 10, 1, 1), (D, _lib.LONG, 10, 1000, 1, 2), (D, _lib.DOUBLE, 20, 1 << 20, 1, 3), (D, _lib.STRING, 7, 100, 0, 4),
        (R, _lib.INT, 32, 0, 0, 0), (D, _lib.INT, 13, 5000, 1, 6), (D, _lib.FLOAT, 2, 3, 1, 7), (D, _lib.LONG, 20, 1 << 20, 1, 8)]


def plan(probe, aggs, args, group_by=(), num_docs=(100_000,), merge=False, cols=None, dense_max=0, flags=0, reduce_world=0):
    """aggs: (function, column); args: (p, time column, type) per aggregation, or None."""
    n = len(num_docs)
    pc = (ProbeCol * (n * len(COLS)))()
    for s in range(n):
        for k, c in enumerate(cols[s] if cols is not None else COLS):
            pc[s * len(COLS) + k] = ProbeCol(*c)
    ag = (_lib.Agg * len(aggs))(*[_lib.Agg(f, c) for f, c in aggs])
    gb = (C.c_int32 * max(1, len(group_by)))(*group_by)
    q = _lib.Query(0, len(group_by), len(aggs), 100_000, 10_000, flags | (2 if merge else 0), None, gb, ag, reduce_world, 0, 0)
    a = None if args is None else (_lib.AggArg * len(args))(*[_lib.AggArg(*x) for x in args])
    out = ProbePlan()
    seg0 = C.create_string_buffer(probe.wt_probe_segdesc_size())
    rc = probe.wt_probe_plan_scan(H100[0], H100[1], C.byref(q), a, pc, len(COLS), (C.c_int32 * n)(*num_docs), n, dense_max,
                                  C.byref(out), seg0)
    return rc, out, seg0.raw


def test_key_layout(probe):
    assert probe.wt_probe_key(7, 3) == (7 << 32) | 3
    assert probe.wt_probe_key(0xFFFFFFFF, 0xFFFFFFFF) == (1 << 64) - 1
    # the descriptors keep their layout (the parent's sizes: a byte-identical SegDesc and shared-memory header)
    assert probe.wt_probe_segdesc_size() == 1248 and probe.wt_probe_smem_header_size() == 1680


@pytest.mark.parametrize("group_by", [(), (0,)])
def test_slots_codes_and_doc_bases(probe, group_by):
    aggs = [(COUNT, -1), (LAST, 2), (FIRST, 3), (SUM, 0)]
    args = [(0, -1, 0), (0, 1, _lib.DOUBLE), (0, 5, _lib.STRING), (0, -1, 0)]
    rc, o, _ = plan(probe, aggs, args, group_by, num_docs=(100_000, 70_000, 5), merge=True)
    assert rc == 0
    slots = list(o.slot_col[:o.num_slots])
    assert 2 not in slots and 3 not in slots          # the data columns are not streamed
    assert 1 in slots and 5 in slots                  # the time columns are
    assert list(o.wt_time[:4]) == [-1, 1, 5, -1]
    assert o.val_kind[1] == 4 and o.val_kind[2] == 1  # VAL_DICT_F64 / VAL_DICT_I32 of the data column
    codes = {o.code_agg[k]: (o.code_fn[k], o.code_vk[k]) for k in range(o.num_agg_codes)}
    assert codes[1] == (7, 0) and codes[2] == (7, 1)  # kFnWithTime, WT_MAX for LAST and WT_MIN for FIRST
    for a in (1, 2):
        assert [o.doc_base[s][a] for s in range(3)] == [0, 100_000, 170_000]
    assert o.smem_groups == 0 and o.spec == 0         # never the CTA-private table, never the specialised kernel


def test_shared_table_and_spec_only_without_withtime(probe):
    # COUNT + INT SUM over a 10-key group: the shared table and the specialised kernel ...
    rc, o, _ = plan(probe, [(COUNT, -1), (SUM, 0)], None, (0,))
    assert rc == 0 and o.smem_groups > 0 and o.spec == 1
    # ... which a FIRST/LASTWITHTIME in the same query turns off
    rc, o, _ = plan(probe, [(COUNT, -1), (SUM, 0), (LAST, 0)], [(0, -1, 0), (0, -1, 0), (0, 1, _lib.INT)], (0,))
    assert rc == 0 and o.smem_groups == 0 and o.spec == 0


@pytest.mark.parametrize("aggs,group_by", [([(COUNT, -1), (SUM, 0)], (0,)), ([(MAX, 1), (SUM, 5), (P, 2)], ()),
                                           ([(MIN, 2), (COUNT, -1)], (5,))])
def test_plans_without_withtime_unchanged(probe, aggs, group_by):
    """pb200_execute_agg_args without the new functions plans exactly what pb200_execute_args plans."""
    pargs = [(50.0, -1, 0) if f == P else (0.0, -1, 0) for f, _ in aggs]
    rc0, o0, s0 = plan(probe, aggs, None if P not in [f for f, _ in aggs] else [tuple(x) for x in pargs], group_by)
    rc1, o1, s1 = plan(probe, aggs, pargs, group_by)
    assert rc0 == rc1 == 0 and bytes(o0) == bytes(o1) and s0 == s1


def test_refusals(probe):
    E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
    ok = [(0, 1, _lib.INT)]
    assert plan(probe, [(LAST, 0)], ok)[0] == 0
    assert plan(probe, [(LAST, 0)], None)[0] == E_INVALID                          # the older entry points
    assert plan(probe, [(LAST, 0)], [(0, 99, _lib.INT)])[0] == E_INVALID           # time column out of range
    assert plan(probe, [(LAST, 0)], [(0, 2, _lib.INT)])[0] == E_UNSUPPORTED        # DOUBLE time
    assert plan(probe, [(LAST, 0)], [(0, 3, _lib.INT)])[0] == E_UNSUPPORTED        # STRING time
    assert plan(probe, [(LAST, 0)], [(0, 4, _lib.INT)])[0] == E_UNSUPPORTED        # raw time, no dictIds
    assert plan(probe, [(LAST, 4)], [(0, 1, _lib.INT)])[0] == E_UNSUPPORTED        # data streamed as raw 32-bit values
    assert plan(probe, [(LAST, 0)], [(0, 1, _lib.LONG)])[0] == E_UNSUPPORTED       # type literal mismatch
    assert plan(probe, [(FIRST, 6)], [(0, 1, _lib.DOUBLE)])[0] == E_UNSUPPORTED    # FLOAT named DOUBLE: never cast
    big = ((1 << 31) - 1, (1 << 31) - 1, 2)
    assert plan(probe, [(LAST, 0)], ok, num_docs=big)[0] == E_UNSUPPORTED          # 2^32 docs in the call
    assert plan(probe, [(LAST, 0)], ok, num_docs=((1 << 31) - 1, (1 << 31) - 1, 1))[0] == 0
    assert plan(probe, [(LAST, 0)], ok, (0,), merge=True, flags=4)[0] == E_UNSUPPORTED   # PB200_Q_DEFER_FINALIZE
    assert plan(probe, [(LAST, 0)], ok, (0,), merge=True, reduce_world=2)[0] == E_UNSUPPORTED
    other = [COLS, COLS[:7] + [(D, _lib.LONG, 20, 1 << 20, 1, 9)]]
    assert plan(probe, [(LAST, 7)], ok, num_docs=(10, 10), merge=True, cols=other)[0] == E_UNSUPPORTED   # v: two dictionaries
    other = [COLS, [COLS[0], (D, _lib.LONG, 10, 1000, 1, 9)] + COLS[2:]]
    assert plan(probe, [(LAST, 0)], ok, num_docs=(10, 10), merge=True, cols=other)[0] == E_UNSUPPORTED   # t: two dictionaries
    assert plan(probe, [(LAST, 0)], ok, num_docs=(10, 10), merge=True)[0] == 0


# ---- reference, merge, distributed ---------------------------------------------------------------------------------
def test_reference_tie_rule(oracle):
    cols = {"t": np.array([5, 7, 7, 3, 7, 3], dtype=np.int32), "v": np.array([1, 2, 3, 4, 5, 6], dtype=np.int32),
            "g": np.array([0, 0, 1, 1, 1, 0], dtype=np.int32)}
    seg = oracle.build_segment("wt_ref", cols)
    assert withtime(oracle, [seg], None, [], "LASTWITHTIME", "v", "t") == {(): (7, 5)}
    assert withtime(oracle, [seg], None, [], "FIRSTWITHTIME", "v", "t") == {(): (3, 4)}
    assert withtime(oracle, [seg, seg], None, ["g"], "LASTWITHTIME", "v", "t") == {(0,): (7, 2), (1,): (7, 5)}
    assert withtime(oracle, [seg], Predicate("EQ", "v", [99]), [], "LASTWITHTIME", "v", "t") == {(): None}


def test_pick_ties():
    assert withtime_pick("LASTWITHTIME", (5, "a"), (5, "b")) == (5, "b")
    assert withtime_pick("FIRSTWITHTIME", (5, "a"), (5, "b")) == (5, "a")
    assert withtime_pick("LASTWITHTIME", (6, "a"), (5, "b")) == (6, "a")
    assert withtime_pick("FIRSTWITHTIME", (6, "a"), (5, "b")) == (5, "b")
    assert withtime_pick("LASTWITHTIME", None, (1, "b")) == (1, "b") and withtime_pick("FIRSTWITHTIME", (1, "a"), None) == (1, "a")


class _Seg:
    def __init__(self, values):
        self.values = values

    def dictionary_value(self, column, dict_id):
        return self.values[column][dict_id]


def _block(keys, doubles, longs, ids):
    stats = ExecutionStatistics(0, 0, 0, 0)
    g = len(keys) if keys is not None else -1
    k = np.array(keys, dtype=np.int32).reshape(max(g, 0), -1) if keys is not None else np.zeros((0, 0), np.int32)
    return ResultsBlock(g, "ARRAY", False, stats, k, [np.array(x, np.float64) for x in doubles],
                        [np.array(x, np.int64) for x in longs], [np.array(x, np.int32) for x in ids], {})


def test_cli_merge_by_value_with_ties_across_segments():
    q = QueryContext(aggregations=[Aggregation("LASTWITHTIME", "s", time_column="t", value_type="STRING"),
                                   Aggregation("FIRSTWITHTIME", "s", time_column="t", value_type="STRING")],
                     group_by=["g"], limit=10)
    s0 = _Seg({"g": ["x", "y"], "s": [b"a", b"b", b"c"]})
    s1 = _Seg({"g": ["y", "x"], "s": [b"c", b"d"]})
    # segment 0: x -> (t 10, 'a') / (t 1, 'b'), y -> (t 3, 'c') both; segment 1: x -> (t 10, 'd') / (t 1, 'c'), y empty
    b0 = _block([[0], [1]], [[0, 2], [1, 2]], [[10, 3], [1, 3]], [[0, 2], [1, 2]])
    b1 = _block([[1], [0]], [[1, 0], [0, 0]], [[10, 0], [1, 0]], [[1, -1], [0, -1]])
    rows = cli.final_rows(q, cli.merge_blocks(q, [s0, s1], [b0, b1]))
    # x: LAST tie at 10 -> the later segment's 'd'; FIRST tie at 1 -> the earlier segment's 'b'
    assert rows == [["x", b"d", b"b"], ["y", b"c", b"c"]]
    q1 = QueryContext(aggregations=[Aggregation("LASTWITHTIME", "s", time_column="t", value_type="STRING")], limit=10)
    empty = _block(None, [[float("-inf")]], [[0]], [[-1]])
    assert cli.final_rows(q1, cli.merge_blocks(q1, [s0], [empty])) == [[float("-inf")]]


def test_distributed_refuses_withtime():
    from pinot_b200 import distributed
    q = QueryContext(aggregations=[Aggregation("LASTWITHTIME", "v", time_column="t", value_type="INT")], limit=10)

    class _Dist:
        def get_world_size(self):
            return 2

    with pytest.raises(_lib.UnsupportedQueryError):
        distributed.execute_and_combine(object(), [], q, _Dist())


def test_cli_having_next_to_a_string_withtime():
    """HAVING on another function of a query whose select list holds a STRING FIRST/LASTWITHTIME (the README's 'latest
    status per device' query with a HAVING): the string value is carried, never compared."""
    q = sql.parse("SELECT device, LASTWITHTIME(status, ts, 'STRING'), COUNT(*) FROM t GROUP BY device HAVING COUNT(*) > 10")
    table = {("d1",): [(5, b"up"), 11], ("d2",): [(7, b"down"), 3], ("d3",): [None, 20]}
    assert cli.final_rows(q, table) == [["d1", b"up", 11], ["d3", float("-inf"), 20]]
    # through the by-value merge of blocks as well
    s0 = _Seg({"device": ["d1", "d2"], "status": [b"down", b"up"]})
    b0 = _block([[0], [1]], [[1, 0], [11, 3]], [[5, 7], [11, 3]], [[1, 0], [-1, -1]])
    assert cli.final_rows(q, cli.merge_blocks(q, [s0], [b0])) == [["d1", b"up", 11]]


def test_results_block_decodes_string_values():
    q = QueryContext(aggregations=[Aggregation("LASTWITHTIME", "s", time_column="t", value_type="STRING"),
                                   Aggregation("FIRSTWITHTIME", "l", time_column="t", value_type="LONG"), Aggregation("COUNT")],
                     limit=10)
    seg = _Seg({"s": [b"a", b"b"], "l": [1, (1 << 53) + 1]})
    b = _block(None, [[1.0], [float(1 << 53)], [4.0]], [[9], [2], [4]], [[1], [1], [-1]])
    assert b.get_results(q, seg) == [b"b", (1 << 53) + 1, 4]
    assert b.withtime(0, 0, seg, "s") == (9, b"b")
    assert b.get_results(q) == [1.0, float(1 << 53), 4]   # without the segment: the double column (STRING: the dictId)
    empty = _block(None, [[float("-inf")], [float("-inf")], [0.0]], [[0], [0], [0]], [[-1], [-1], [-1]])
    assert empty.get_results(q, seg) == [float("-inf"), float("-inf"), 0]

"""CPU tests of DISTINCTSUM / DISTINCTAVG and COUNT / SUM / AVG(DISTINCT col): the parser (every spelling, the canonical
text, ORDER BY and HAVING naming, refusals), the eligibility rule and the finalize arithmetic
(pinot_b200/csrc/pb200_distinct_sum.h, the code the device runs, through tests/distinct_sum_probe) against Fractions, the
planner's bitset sharing and refusals (pb200::plan_scan through the same probe), and the CLI's by-value merge."""
import ctypes as C
import math
import os
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import ExecutionStatistics, ResultsBlock
from pinot_b200.query import distinct_final

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DSUM, DAVG, DCOUNT, SUM, COUNT = 13, 14, 5, 1, 0
AGG = 8


# ---- parser --------------------------------------------------------------------------------------------------------
def test_parse_every_spelling():
    q = sql.parse("SELECT COUNT(DISTINCT a), count(distinct a), DISTINCTCOUNT(a), SUM(DISTINCT b), DistinctSum(b), "
                  "AVG(DISTINCT c), distinctavg(c) FROM t")
    assert [(x.function, x.column) for x in q.aggregations] == [
        ("DISTINCTCOUNT", "a"), ("DISTINCTCOUNT", "a"), ("DISTINCTCOUNT", "a"), ("DISTINCTSUM", "b"), ("DISTINCTSUM", "b"),
        ("DISTINCTAVG", "c"), ("DISTINCTAVG", "c")]
    assert [str(x) for x in q.aggregations[::3]] == ["distinctcount(a)", "distinctsum(b)", "distinctavg(c)"]
    q = sql.parse("SELECT SUM(DISTINCT DATETRUNC('HOUR', ts)) FROM t")
    assert q.aggregations[0].function == "DISTINCTSUM" and q.aggregations[0].column.startswith("datetrunc(")


def test_order_by_and_having_naming():
    q = sql.parse("SELECT g, COUNT(DISTINCT m), SUM(DISTINCT m), AVG(DISTINCT m) FROM t GROUP BY g "
                  "HAVING distinctsum(m) > 2 AND AVG(DISTINCT m) < 9 ORDER BY distinctcount(m), SUM(DISTINCT m) DESC, "
                  "DISTINCTAVG(m) LIMIT 3")
    assert sql.resolve_order_by(q) == [("AGG", 0, True), ("AGG", 1, False), ("AGG", 2, True)]
    assert [a.hidden for a in q.aggregations] == [False, False, False]
    leaves = [n for n in sql.resolve_having(q) if n[0] == "RANGE"]
    assert [n[1] for n in leaves] == [1, 2]
    q = sql.parse("SELECT g, DISTINCTCOUNT(m) FROM t GROUP BY g ORDER BY COUNT(DISTINCT m) DESC")
    assert sql.resolve_order_by(q) == [("AGG", 0, False)]
    q = sql.parse("SELECT g, COUNT(*) FROM t GROUP BY g HAVING SUM(DISTINCT m) >= 1")   # named only in HAVING: hidden
    assert q.aggregations[1].function == "DISTINCTSUM" and q.aggregations[1].hidden


@pytest.mark.parametrize("text", ["SELECT MIN(DISTINCT a) FROM t", "SELECT MAX(DISTINCT a) FROM t",
                                  "SELECT COUNT(DISTINCT *) FROM t", "SELECT COUNT(DISTINCT a, b) FROM t",
                                  "SELECT SUM(DISTINCT) FROM t", "SELECT DISTINCTSUM(*) FROM t",
                                  "SELECT g, SUM(DISTINCT m) FROM t GROUP BY g ORDER BY MAX(DISTINCT m)"])
def test_parse_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


# ---- probe ---------------------------------------------------------------------------------------------------------
FIELDS = [(n, 1) for n in ("group_by", "num_agg_codes")] + [(n, AGG) for n in ("ds_rep", "code_fn", "code_agg", "slot",
                                                                                   "dwords", "distinct_words")]


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32), ("raw", C.c_int32),
                ("dict_hash", C.c_int32), ("dict", C.c_void_p)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "distinct_sum_probe", "distinct_sum_probe.cpp")
    out = os.path.join(HERE, "distinct_sum_probe", "libdistinct_sum_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.ds_probe_plan_size.restype = C.c_int64
    assert lib.ds_probe_plan_size() == C.sizeof(ProbePlan)
    lib.ds_probe_grid.restype = C.c_int32
    lib.ds_probe_grid.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
    lib.ds_probe_final_doubles.restype = C.c_double
    lib.ds_probe_final_doubles.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_int32]
    lib.ds_probe_final_state.restype = C.c_double
    lib.ds_probe_final_state.argtypes = [C.c_int32, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int32]
    lib.ds_probe_plan_scan.restype = C.c_int32
    lib.ds_probe_plan_scan.argtypes = [C.POINTER(_lib.Query), C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32),
                                       C.c_int32, C.POINTER(ProbePlan)]
    return lib


DTYPES = {_lib.INT: np.int32, _lib.LONG: np.int64, _lib.FLOAT: np.float32, _lib.DOUBLE: np.float64}


def grid(probe, stored_type, values):
    arr = np.ascontiguousarray(np.sort(np.asarray(values, dtype=DTYPES[stored_type])))
    e = C.c_int32()
    return e.value if probe.ds_probe_grid(stored_type, arr.ctypes.data, len(arr), C.byref(e)) else None


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def reference(fn, values):
    """Fraction reference of the semantics (DESIGN.md section 3.14), independent of the library."""
    vals = [float(v) for v in values]
    nan = any(v != v for v in vals)
    if nan or (math.inf in vals and -math.inf in vals):
        return math.nan
    if math.inf in vals:
        return math.inf
    if -math.inf in vals:
        return -math.inf
    if not vals:
        return 0.0 if fn == DSUM else -math.inf
    s = sum((Fraction(v) for v in vals), Fraction(0))
    if fn == DAVG:
        s /= len(vals)
    try:
        return float(s)
    except OverflowError:
        return math.inf if s > 0 else -math.inf


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or bits(a) == bits(b)


def final_doubles(probe, fn, values, e):
    arr = np.ascontiguousarray(np.asarray(values, dtype=np.float64))
    return probe.ds_probe_final_doubles(fn, arr.ctypes.data, len(arr), e)


def final_sum(probe, fn, total, n, e=0, flags=0):
    u = total & ((1 << 128) - 1)
    return probe.ds_probe_final_state(fn, u & ((1 << 64) - 1), u >> 64, n, flags, e)


# ---- eligibility ---------------------------------------------------------------------------------------------------
def test_grid_integers_always(probe):
    assert grid(probe, _lib.INT, [-(1 << 31), 0, (1 << 31) - 1]) == 0
    assert grid(probe, _lib.LONG, [-(1 << 63), (1 << 63) - 1]) == 0


def test_grid_dyadic_floats(probe):
    assert grid(probe, _lib.DOUBLE, [-1.5, 0.25, 1000.125, 3.0]) == -3
    assert grid(probe, _lib.DOUBLE, [1024.0, 2048.0, 3 * 4096.0]) == 10
    assert grid(probe, _lib.FLOAT, [-0.5, 0.25, 7.75]) == -2
    assert grid(probe, _lib.DOUBLE, [math.nan, -math.inf, -0.0, 0.0, 2.5, math.inf]) == -1   # specials never constrain e
    assert grid(probe, _lib.DOUBLE, [0.0, -0.0]) == 0
    assert grid(probe, _lib.DOUBLE, [5e-324, 1.0]) is None                                     # 2^1074 steps: |j| too large
    assert grid(probe, _lib.DOUBLE, [5e-324, 2.0 ** -1020]) == -1074                          # |j| = 2^54: fits


@pytest.mark.parametrize("values", [[0.01 * i for i in range(1, 10001)], [0.1 * i for i in range(1, 100001)],
                                    [1.0, 2.0 ** -63], [2.0 ** 70, 1.0], [1e300, 1.0]])
def test_grid_refusals(probe, values):
    assert grid(probe, _lib.DOUBLE, values) is None


# ---- finalize arithmetic -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", [DSUM, DAVG])
@pytest.mark.parametrize("values", [
    [1.0, 2.0, -7.5], [-0.5, -0.25], [0.125] * 0, [-0.0], [0.0, -0.0], [3.0, -3.0],
    [1.0, math.inf], [-math.inf, 5.0], [math.inf, -math.inf], [math.nan, 1.0], [math.nan, math.inf],
    [2.0 ** 52 + 1, 0.5], [1.0, 2.0 ** -52, 2.0 ** -53]])
def test_final_doubles(probe, fn, values):
    finite = [v for v in values if math.isfinite(v) and v != 0.0]
    e = min((Fraction(v).denominator.bit_length() - 1) * -1 for v in finite) if finite else 0
    assert same(final_doubles(probe, fn, values, e), reference(fn, values)), (values, e)


@pytest.mark.parametrize("fn", [DSUM, DAVG])
def test_int_extremes(probe, fn):
    vals = [-(1 << 31), -1, 0, 1, (1 << 31) - 1]
    assert same(final_sum(probe, fn, sum(vals), len(vals)), reference(fn, vals))


@pytest.mark.parametrize("fn", [DSUM, DAVG])
@pytest.mark.parametrize("n", [(1 << 32) - 1, 1 << 32, 3_000_000_000])
@pytest.mark.parametrize("sign", [1, -1])
def test_long_extremes_many_members(probe, fn, n, sign):
    # n members near +-2^63 (a LONG dictionary with a billion-scale set): the sum spans ~95 bits
    total = sign * ((1 << 63) - 12345) * n + sign * (n * (n - 1) // 2) % (1 << 20)
    want = Fraction(total) / (n if fn == DAVG else 1)
    assert bits(final_sum(probe, fn, total, n)) == bits(float(want))


def test_ties_to_even(probe):
    for total, want in [((1 << 53) + 1, 2.0 ** 53), ((1 << 53) + 3, 2.0 ** 53 + 4), (-((1 << 54) + 2), -(2.0 ** 54)),
                        (-((1 << 54) + 6), -(2.0 ** 54 + 8))]:
        assert bits(final_sum(probe, DSUM, total, 2)) == bits(want)
    # DISTINCTAVG: (2^54 + 2) / 2 = 2^53 + 1 -> 2^53 (tie, even);  (2^54 + 6) / 2 = 2^53 + 3 -> 2^53 + 4
    assert bits(final_sum(probe, DAVG, (1 << 54) + 2, 2)) == bits(2.0 ** 53)
    assert bits(final_sum(probe, DAVG, (1 << 54) + 6, 2)) == bits(2.0 ** 53 + 4)
    # a remainder breaks the tie: (2^53 + 1) * 3 + 1 over 3
    assert bits(final_sum(probe, DAVG, ((1 << 53) + 1) * 3 + 1, 3)) == bits(2.0 ** 53 + 2)


@pytest.mark.parametrize("total, n, e", [(1, 1, -1074), (3, 1, -1075), (1, 1, -1076), (5, 2, -1075), (3, 3, -1075),
                                         ((1 << 53) - 1, 1, -1074 - 52), ((1 << 52) + 1, 2, -1074), (-7, 4, -1074),
                                         (1, 7, -1060), ((1 << 60) + 12345, 3, -1130)])
@pytest.mark.parametrize("fn", [DSUM, DAVG])
def test_subnormal_results(probe, total, n, e, fn):
    want = Fraction(total) * Fraction(2) ** e / (n if fn == DAVG else 1)
    assert bits(final_sum(probe, fn, total, n, e)) == bits(float(want))   # float(Fraction): rounded once


@pytest.mark.parametrize("fn", [DSUM, DAVG])
def test_overflow_results(probe, fn):
    big = (1 << 63) - 1
    assert final_sum(probe, fn, big * 4, 4, 1000) == math.inf
    assert final_sum(probe, fn, -big * 4, 4, 1000) == -math.inf
    # just below the overflow threshold: (2^53 - 1) 2^971 = DBL_MAX; + half an ulp rounds up to inf, less stays
    top = ((1 << 53) - 1) << 10
    assert final_sum(probe, DSUM, top, 1, 961) == 1.7976931348623157e308
    assert final_sum(probe, DSUM, top + (1 << 9), 1, 961) == math.inf
    assert final_sum(probe, DSUM, top + (1 << 9) - 1, 1, 961) == 1.7976931348623157e308


def test_special_flags_and_empty(probe):
    NAN, POS, NEG = 1, 2, 4
    assert math.isnan(final_sum(probe, DSUM, 5, 2, flags=NAN))
    assert math.isnan(final_sum(probe, DAVG, 5, 3, flags=POS | NEG))
    assert final_sum(probe, DAVG, -5, 3, flags=POS) == math.inf
    assert final_sum(probe, DSUM, 5, 3, flags=NEG) == -math.inf
    assert bits(final_sum(probe, DSUM, 0, 0)) == bits(0.0)
    assert final_sum(probe, DAVG, 0, 0) == -math.inf
    assert bits(final_doubles(probe, DSUM, [-0.0], 0)) == bits(0.0)   # {-0.0}: 0.0 + -0.0 = 0.0
    assert bits(final_doubles(probe, DAVG, [-0.0], 0)) == bits(0.0)


def test_python_final_matches_reference():
    for fn, name in ((DSUM, "DISTINCTSUM"), (DAVG, "DISTINCTAVG")):
        for vals in ([], [-0.0], [1.0, 2.5], [math.nan], [math.inf, 1.0], [-math.inf, math.inf], [1e308, 1e308, 0.5],
                     [5e-324, 0.5 * 2 ** -1073]):
            assert same(distinct_final(name, vals), reference(fn, vals))
    assert distinct_final("DISTINCTCOUNT", [1.0, 2.0]) == 2


# ---- planner -------------------------------------------------------------------------------------------------------
def plan(probe, aggs, cols, group_by=(), nseg=1, flags=0, docs=1 << 20):
    a = (_lib.Agg * len(aggs))(*[_lib.Agg(f, c) for f, c in aggs])
    gb = (C.c_int32 * max(len(group_by), 1))(*group_by)
    q = _lib.Query(num_group_by=len(group_by), num_aggs=len(aggs), num_groups_limit=100000,
                   max_initial_result_holder_capacity=10000, flags=flags, group_by_columns=gb, aggs=a)
    pc = (ProbeCol * (len(cols) * nseg))(*[ProbeCol(*c) for _ in range(nseg) for c in cols])
    nd = (C.c_int32 * nseg)(*([docs] * nseg))
    out = ProbePlan()
    rc = probe.ds_probe_plan_scan(C.byref(q), pc, len(cols), nd, nseg, C.byref(out))
    return rc, out


_KEEP = []


def dcol(stored, values, bits=8, dict_hash=1):
    arr = np.ascontiguousarray(np.sort(np.asarray(values, dtype=DTYPES[stored])))
    _KEEP.append(arr)
    return (stored, bits, len(arr), 0, dict_hash, arr.ctypes.data)


def test_plan_sharing_and_owner_codes(probe):
    cols = [dcol(_lib.INT, range(200)), dcol(_lib.DOUBLE, [0.5 * i for i in range(100)]), dcol(_lib.INT, range(10), 4)]
    # DISTINCTCOUNT first: the new functions read its bitset and add no code
    rc, p = plan(probe, [(DCOUNT, 0), (DSUM, 0), (DAVG, 0), (SUM, 1)], cols)
    assert rc == 0
    assert list(p.ds_rep[:4]) == [-1, 0, 0, -1] and list(p.slot[1:3]) == [-1, -1]
    assert set(zip(p.code_fn[:p.num_agg_codes], p.code_agg[:p.num_agg_codes])) == {(DCOUNT, 0), (SUM, 3)}
    assert p.distinct_words[0] > 0 and list(p.distinct_words[1:3]) == [0, 0]
    # the first new function owns the set and carries the DISTINCTCOUNT code; a later DISTINCTCOUNT keeps its own bitset
    rc, p = plan(probe, [(DAVG, 1), (DSUM, 1), (DCOUNT, 1), (DSUM, 0)], cols, group_by=[2])
    assert rc == 0 and p.group_by
    assert list(p.ds_rep[:4]) == [0, 0, -1, 3]
    assert set(zip(p.code_fn[:p.num_agg_codes], p.code_agg[:p.num_agg_codes])) == {(DCOUNT, 0), (DCOUNT, 2), (DCOUNT, 3)}
    assert p.dwords[0] == 4 and p.dwords[1] == 0 and p.dwords[2] == 4 and p.dwords[3] == 7


@pytest.mark.parametrize("col, why", [
    ((_lib.STRING, 8, 100, 0, 1, None), "STRING"),
    ((_lib.INT, 32, 0, 1, 1, None), "raw"),
    (None, "grid"),
])
def test_plan_refusals(probe, col, why):
    if col is None:
        col = dcol(_lib.DOUBLE, [0.01 * i for i in range(1, 10001)], 14)
    for fn in (DSUM, DAVG):
        rc, _ = plan(probe, [(fn, 0)], [col])
        assert rc == _lib.E_UNSUPPORTED, why


def test_plan_bitset_budget(probe):
    cols = [dcol(_lib.INT, range(1 << 16), 16), dcol(_lib.INT, range(1 << 15), 15)]
    # dense: 2^15 groups x 2^10 words fits the 2^28-word budget; hashed (2^31 keys): 2^18 slots x 2^11 words does not
    assert plan(probe, [(DSUM, 1)], cols, group_by=[1])[0] == 0
    assert plan(probe, [(DSUM, 0)], cols, group_by=[0, 1])[0] == _lib.E_UNSUPPORTED


def test_plan_merge_needs_one_dictionary(probe):
    same_a, same_b = dcol(_lib.INT, range(100), dict_hash=7), dcol(_lib.INT, range(100), dict_hash=7)
    other = dcol(_lib.INT, range(1, 101), dict_hash=8)
    for fn in (DSUM, DAVG):
        for group_by in ((), (1,)):
            cols = lambda c: [c, dcol(_lib.INT, range(10), 4, dict_hash=3)]
            aggs = (_lib.Agg * 1)(_lib.Agg(fn, 0))
            gb = (C.c_int32 * 1)(*(group_by or (0,)))
            q = _lib.Query(num_group_by=len(group_by), num_aggs=1, num_groups_limit=100000,
                           max_initial_result_holder_capacity=10000, flags=2, group_by_columns=gb, aggs=aggs)
            nd = (C.c_int32 * 2)(1000, 1000)
            for second, want in ((same_b, 0), (other, _lib.E_UNSUPPORTED)):
                pc = (ProbeCol * 4)(*[ProbeCol(*c) for c in cols(same_a) + cols(second)])
                assert probe.ds_probe_plan_scan(C.byref(q), pc, 2, nd, 2, C.byref(ProbePlan())) == want, (fn, group_by)


def test_plan_two_distinctcounts_keep_their_own_bitsets(probe):
    """Queries without the new functions plan as before: two DISTINCTCOUNTs of one column each set their own bitset
    (the full differential check against a parent build is tests/host_probe/plan_diff.py)."""
    cols = [dcol(_lib.INT, range(200)), dcol(_lib.INT, range(10), 4)]
    for group_by in ((), (1,)):
        rc, p = plan(probe, [(DCOUNT, 0), (DCOUNT, 0), (SUM, 0)], cols, group_by=group_by)
        assert rc == 0 and list(p.ds_rep[:3]) == [-1, -1, -1] and list(p.slot[:2]) == [p.slot[0]] * 2 and p.slot[0] >= 0
        assert set(zip(p.code_fn[:p.num_agg_codes], p.code_agg[:p.num_agg_codes])) == {(DCOUNT, 0), (DCOUNT, 1), (SUM, 2)}
        words = p.dwords if group_by else p.distinct_words
        assert words[0] == words[1] > 0


# ---- CLI merge -----------------------------------------------------------------------------------------------------
class _Seg:
    def __init__(self, dicts):
        self.dicts = dicts

    def dictionary_value(self, column, d):
        return self.dicts[column][d]


def _block(groups, keys, doubles, longs, distinct):
    stats = ExecutionStatistics(0, 0, 0, 0)
    n = len(keys)
    return ResultsBlock(groups, "ARRAY", False, stats, np.asarray(keys, dtype=np.int32).reshape(n, -1), doubles, longs,
                        [np.full(max(n, 1), -1, dtype=np.int32)] * len(doubles), distinct, 0.0, "GROUP_BY")


def test_cli_merges_value_sets_by_value():
    q = sql.parse("SELECT g, COUNT(DISTINCT m), SUM(DISTINCT m), AVG(DISTINCT m) FROM t GROUP BY g "
                  "ORDER BY SUM(DISTINCT m) DESC LIMIT 10")
    # two segments with different dictionaries; group 'x' sees {0.5, 2.0} and {2.0, -0.0, 1e308}
    s1 = _Seg({"g": ["x", "y"], "m": [0.5, 2.0, 7.0]})
    s2 = _Seg({"g": ["x"], "m": [-0.0, 2.0, 1e308]})
    z = np.zeros(2)
    b1 = _block(2, [[0], [1]], [z, z, z], [z.astype(np.int64)] * 3,
                {(0, 0): [0, 1], (1, 0): [0, 1], (2, 0): [0, 1], (0, 1): [2], (1, 1): [2], (2, 1): [2]})
    b2 = _block(1, [[0]], [z[:1]] * 3, [z[:1].astype(np.int64)] * 3, {(0, 0): [0, 1, 2], (1, 0): [0, 1, 2], (2, 0): [0, 1, 2]})
    rows = cli.final_rows(q, cli.merge_blocks(q, [s1, s2], [b1, b2]))
    want_x = [0.5, 2.0, -0.0, 1e308]
    assert rows[0][0] == "x" and rows[0][1] == 4
    assert bits(rows[0][2]) == bits(float(sum(Fraction(v) for v in want_x)))
    assert bits(rows[0][3]) == bits(float(sum(Fraction(v) for v in want_x) / 4))
    assert rows[1] == ["y", 1, 7.0, 7.0]


# ---- ABI -----------------------------------------------------------------------------------------------------------
def test_abi_codes_match_the_header():
    import re
    text = open(os.path.join(ROOT, "include", "pinot_b200.h")).read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"PB200_AGG_([A-Z]+) = (\d+)", text)}
    assert codes["DISTINCTSUM"] == 13 and codes["DISTINCTAVG"] == 14
    assert {k: _lib.AGG_CODES[k] for k in codes} == codes
    assert re.search(r"#define PB200_ABI_VERSION 3\b", text)


# ---- LONG members beyond 2^53: the host merges sum Python integers, never doubles -----------------------------------
BIG = 1 << 53
LONG_SETS = {"x": [BIG + 1, BIG + 5], "y": [-(BIG + 3), 7, BIG + 9, (1 << 62) + 1], "z": [(1 << 63) - 1, (1 << 63) - 3]}


def _exact(fn, vals):
    s = sum(Fraction(v) for v in set(vals))
    return float(s / len(set(vals)) if fn == "DISTINCTAVG" else s)


def test_python_final_long_beyond_2_53():
    assert distinct_final("DISTINCTSUM", [BIG + 1, BIG + 5]) == 18014398509481992.0
    assert distinct_final("DISTINCTAVG", [np.int64(BIG + 1), np.int64(BIG + 5)]) == 9007199254740996.0
    for vals in LONG_SETS.values():
        for fn in ("DISTINCTSUM", "DISTINCTAVG"):
            assert bits(distinct_final(fn, vals)) == bits(_exact(fn, vals))


def test_cli_merges_long_sets_exactly():
    q = sql.parse("SELECT g, SUM(DISTINCT l), AVG(DISTINCT l) FROM t GROUP BY g ORDER BY SUM(DISTINCT l) DESC LIMIT 2")
    keys = sorted(LONG_SETS)
    # each group's set split over two segments with different dictionaries (one member in both)
    segs, blocks = [], []
    for part in (0, 1):
        members = {k: v[part::2] + v[:1] for k, v in LONG_SETS.items()}
        dictionary = sorted({x for v in members.values() for x in v})
        segs.append(_Seg({"g": keys, "l": dictionary}))
        z = np.zeros(len(keys))
        dist = {(a, gi): [dictionary.index(x) for x in members[k]] for a in (0, 1) for gi, k in enumerate(keys)}
        blocks.append(_block(len(keys), [[i] for i in range(len(keys))], [z, z], [z.astype(np.int64)] * 2, dist))
    rows = cli.final_rows(q, cli.merge_blocks(q, segs, blocks))
    want = sorted(keys, key=lambda k: -_exact("DISTINCTSUM", LONG_SETS[k]))[:2]
    assert [r[0] for r in rows] == want
    for r in rows:
        assert bits(r[1]) == bits(_exact("DISTINCTSUM", LONG_SETS[r[0]]))
        assert bits(r[2]) == bits(_exact("DISTINCTAVG", LONG_SETS[r[0]]))


# ---- the cross-GPU host route (distributed._combine_with_sets) under gloo --------------------------------------------
class _SetSegment:
    """A rank's segment after global_domain: one table-wide dictionary per column, rows as domain ids."""

    def __init__(self, domain, rows):
        self.domain, self.rows = domain, rows

    def dictionary_value(self, column, d):
        return self.domain[column][d]


class _SetPlanMaker:
    """Stands in for the device: the merged block of a rank's segments, sets of domain ids per group."""
    ctx = None

    def execute_segments(self, segments, query, merge=True, ordered=False):
        gb = query.group_by
        groups = {}
        for seg in segments:
            for row in seg.rows:
                key = tuple(row[c] for c in gb)
                groups.setdefault(key, {a: set() for a in range(len(query.aggregations))})
                for a, agg in enumerate(query.aggregations):
                    groups[key][a].add(row[agg.column])
        keys = sorted(groups)
        n = len(keys) if gb else 1
        if not gb and not keys:
            keys, groups = [()], {(): {a: set() for a in range(len(query.aggregations))}}
        z = np.zeros(max(n, 1))
        distinct = {(a, g): sorted(groups[k][a]) for g, k in enumerate(keys) for a in range(len(query.aggregations))}
        stats = ExecutionStatistics(sum(len(s.rows) for s in segments), 0, 0, sum(len(s.rows) for s in segments))
        return [ResultsBlock(n if gb else -1, "ARRAY", False, stats,
                             np.asarray(keys, dtype=np.int32).reshape(len(keys), len(gb)) if gb else np.zeros((0, 0), dtype=np.int32),
                             [z.copy() for _ in query.aggregations], [z.astype(np.int64) for _ in query.aggregations],
                             [np.full(max(n, 1), -1, dtype=np.int32) for _ in query.aggregations], distinct, 0.0, "GROUP_BY")]


DIST_QUERIES = ["SELECT g, SUM(DISTINCT l), AVG(DISTINCT l), COUNT(DISTINCT l) FROM t GROUP BY g "
                "ORDER BY SUM(DISTINCT l) DESC LIMIT 3",
                "SELECT DISTINCTSUM(l), DISTINCTAVG(l) FROM t"]


def _rank_rows(rank, values, G=6):
    rng = np.random.default_rng(70 + rank)
    return [{"g": int(rng.integers(0, G)), "l": int(rng.integers(0, len(values)))} for _ in range(300)]


def _dist_values():
    rng = np.random.default_rng(5)
    return sorted({int(x) for x in rng.integers(-(1 << 62), 1 << 62, size=60)} | {BIG + 1, BIG + 5})


def _sets_worker(rank, world, port, out_dir):
    import pickle
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pinot_b200.distributed import execute_and_combine
    domain = {"g": list(range(6)), "l": _dist_values()}
    segs = [_SetSegment(domain, _rank_rows(rank, domain["l"]))]
    out = {}
    for text in DIST_QUERIES:
        got = execute_and_combine(_SetPlanMaker(), segs, sql.parse(text), dist, dst=0)
        if rank == 0:
            rows = 1 if got.num_groups < 0 else got.num_groups
            out[text] = [(tuple(int(x) for x in got.keys[g]) if got.num_groups >= 0 else (),
                          [float(got.doubles[a][g]) for a in range(len(got.doubles))]) for g in range(rows)]
    if rank == 0:
        pickle.dump(out, open(os.path.join(out_dir, "sets.pkl"), "wb"))
    dist.destroy_process_group()


def test_distributed_set_route_world_size_2(tmp_path):
    """execute_and_combine over gloo: the per-rank id sets are unioned on the root and finalized exactly (LONG members
    beyond 2^53), ORDER BY DISTINCTSUM DESC LIMIT 3 trims on those exact values."""
    import pickle
    import torch.multiprocessing as mp
    world, port = 2, 33500 + (os.getpid() % 1500)
    mp.spawn(_sets_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    got = pickle.load(open(tmp_path / "sets.pkl", "rb"))
    values = _dist_values()
    rows = [r for k in range(world) for r in _rank_rows(k, values)]
    per_group = {}
    for r in rows:
        per_group.setdefault(r["g"], set()).add(values[r["l"]])
    # rows come back ordered and trimmed like the dense route (max(5 LIMIT, minServerGroupTrimSize)): here every group
    ranked = sorted(per_group, key=lambda g: (-_exact("DISTINCTSUM", per_group[g]), g))
    want = [((g,), [_exact("DISTINCTSUM", per_group[g]), _exact("DISTINCTAVG", per_group[g]), float(len(per_group[g]))])
            for g in ranked]
    assert [(k, [bits(x) for x in v]) for k, v in got[DIST_QUERIES[0]]] == [(k, [bits(x) for x in v]) for k, v in want]
    every = {values[r["l"]] for r in rows}
    assert [bits(x) for x in got[DIST_QUERIES[1]][0][1]] == [bits(_exact("DISTINCTSUM", every)), bits(_exact("DISTINCTAVG", every))]

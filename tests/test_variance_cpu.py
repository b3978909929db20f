"""CPU tests of VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP: the parser (every spelling, ORDER BY resolution,
refusals), the eligibility rule and the finalize arithmetic (pinot_b200/csrc/pb200_moments.h, the code the device runs,
through tests/moments_probe/moments_probe.cpp) against Fractions, the planner's expansion into limb sums (pb200::plan_scan
through the same probe) with every refusal, and the CLI's by-value merge of per-segment moments."""
import ctypes as C
import math
import os
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import variance_ref as vr
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import ExecutionStatistics, ResultsBlock
from pinot_b200.query import Aggregation, Moments, QueryContext, merge_moments, moments_final

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H100 = (132, 232_448)
AGG = 6
VARPOP, VARSAMP, STDDEVPOP, STDDEVSAMP = 7, 8, 9, 10
SUM, COUNT, AVG = 1, 0, 4


# ---- parser --------------------------------------------------------------------------------------------------------
def test_parse_every_spelling():
    q = sql.parse("SELECT VAR_POP(a), varpop(a), VAR_SAMP(b), VarSamp(b), STDDEV_POP(c), stddevpop(c), "
                  "stddev_samp(d), STDDEVSAMP(d) FROM t GROUP BY g")
    assert [(x.function, x.column) for x in q.aggregations] == [
        ("VARPOP", "a"), ("VARPOP", "a"), ("VARSAMP", "b"), ("VARSAMP", "b"), ("STDDEVPOP", "c"), ("STDDEVPOP", "c"),
        ("STDDEVSAMP", "d"), ("STDDEVSAMP", "d")]
    assert str(q.aggregations[0]) == "varpop(a)"
    assert not sql.is_selection("SELECT STDDEV_POP(a) FROM t")
    q = sql.parse("SELECT VAR_POP(DATETRUNC('HOUR', ts)) FROM t")
    assert q.aggregations[0].function == "VARPOP" and q.aggregations[0].column.startswith("datetrunc(")


def test_order_by_resolution():
    q = sql.parse("SELECT g, STDDEV_SAMP(m), VAR_POP(m) FROM t GROUP BY g ORDER BY STDDEV_SAMP(m) DESC LIMIT 10")
    assert sql.resolve_order_by(q) == [("AGG", 0, False)]
    q = sql.parse("SELECT g, STDDEVSAMP(m), VARPOP(m) FROM t GROUP BY g ORDER BY var_pop(m), stddev_samp(m) DESC")
    assert sql.resolve_order_by(q) == [("AGG", 1, True), ("AGG", 0, False)]
    with pytest.raises(sql.SqlError):   # not in the SELECT list
        sql.parse("SELECT g, VAR_POP(m) FROM t GROUP BY g ORDER BY VAR_SAMP(m)")


@pytest.mark.parametrize("text", ["SELECT VAR_POP(*) FROM t", "SELECT VAR_POP(a, 1) FROM t", "SELECT STDDEV(a) FROM t",
                                  "SELECT VARIANCE(a) FROM t", "SELECT COVAR_POP(a, b) FROM t", "SELECT VAR_POP() FROM t"])
def test_parse_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


# ---- probe ---------------------------------------------------------------------------------------------------------
FIELDS = ([(n, 1) for n in ("num_aggs", "num_user_aggs", "spec", "smem_groups", "need_count", "carrier_agg", "projected",
                            "num_slots")]
          + [(n, AGG) for n in ("mom_first", "limb", "fn", "val_kind", "slot", "dict_off")])


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32),
                ("dict_native", C.c_int32), ("dict_hash", C.c_int32), ("eligible", C.c_int32)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "moments_probe", "moments_probe.cpp")
    out = os.path.join(HERE, "moments_probe", "libmoments_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.mom_probe_plan_size.restype = C.c_int64
    assert lib.mom_probe_plan_size() == C.sizeof(ProbePlan)
    lib.mom_probe_grid.restype = C.c_int32
    lib.mom_probe_grid.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int32), C.POINTER(C.c_uint32)]
    lib.mom_probe_final.restype = C.c_double
    lib.mom_probe_final.argtypes = [C.c_int32, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                    C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.mom_probe_plan_scan.restype = C.c_int32
    lib.mom_probe_plan_scan.argtypes = [C.c_int32, C.c_int32, C.POINTER(_lib.Query), C.POINTER(ProbeCol), C.c_int32,
                                        C.POINTER(C.c_int32), C.c_int32, C.POINTER(ProbePlan)]
    return lib


def grid(probe, stored_type, values):
    dtype = {_lib.INT: np.int32, _lib.LONG: np.int64, _lib.FLOAT: np.float32, _lib.DOUBLE: np.float64}[stored_type]
    arr = np.ascontiguousarray(np.sort(np.asarray(values, dtype=dtype)))
    cm, cx, e, k = C.c_int64(), C.c_int32(), C.c_int32(), C.c_uint32()
    ok = probe.mom_probe_grid(stored_type, arr.ctypes.data, len(arr), C.byref(cm), C.byref(cx), C.byref(e), C.byref(k))
    return (cm.value, cx.value, e.value, k.value) if ok else None


def _exact_value(c_mant, c_exp, e, k):
    return Fraction(c_mant) * Fraction(2) ** c_exp + k * Fraction(2) ** e


# ---- eligibility ---------------------------------------------------------------------------------------------------
def test_eligibility_int_extremes(probe):
    g = grid(probe, _lib.INT, [-(1 << 31), -5, 0, 17, (1 << 31) - 1])
    assert g == (-(1 << 31), 0, 0, (1 << 32) - 1)


@pytest.mark.parametrize("offset", [-(1 << 62), 0, 1 << 62])
def test_eligibility_long_range(probe, offset):
    assert grid(probe, _lib.LONG, [offset, offset + 1, offset + (1 << 32) - 1]) == (offset, 0, 0, (1 << 32) - 1)
    assert grid(probe, _lib.LONG, [offset, offset + 1, offset + (1 << 32)]) is None


def test_eligibility_dyadic_doubles(probe):
    vals = [-1.5, -1.375, 0.25, 1000.125, 3.0]
    cm, cx, e, k = grid(probe, _lib.DOUBLE, vals)
    assert e == -3 and _exact_value(cm, cx, 0, 0) == Fraction(-1.5)
    for v in vals:   # every value is c + k 2^e with an integral k < 2^32
        kk = (Fraction(v) - Fraction(-1.5)) / Fraction(2) ** e
        assert kk.denominator == 1 and 0 <= kk < 2 ** 32
    assert grid(probe, _lib.DOUBLE, [1024.0, 2048.0, 4096.0 * 1024]) == (1, 10, 10, 4095)   # a grid coarser than 1
    assert grid(probe, _lib.FLOAT, [-0.5, 0.25, 7.75]) is not None
    assert grid(probe, _lib.DOUBLE, [0.1, 0.2, 0.3]) is None               # 0.1-steps
    assert grid(probe, _lib.DOUBLE, [0.0, 1.0, math.inf]) is None
    assert grid(probe, _lib.DOUBLE, [-math.inf, 0.0]) is None
    assert grid(probe, _lib.DOUBLE, [0.0, 2.0 ** 32]) == (0, 0, 32, 1)     # k = 1 on a 2^32 grid
    assert grid(probe, _lib.DOUBLE, [0.0, 1.0, 2.0 ** 32]) is None         # 2^32 steps of 1
    assert grid(probe, _lib.DOUBLE, [7.5]) == (15, -1, 0, 0)               # one value


# ---- finalize arithmetic -------------------------------------------------------------------------------------------
def _device_sums(ks):
    """The three limb sums as the scan leaves them: each limb word W read as W - 2^31."""
    sk = sum(k - (1 << 31) for k in ks)
    sh = sum(((k * k) >> 32) - (1 << 31) for k in ks)
    sl = sum(((k * k) & 0xFFFFFFFF) - (1 << 31) for k in ks)
    return sk, sh, sl


def _final(probe, fn, n, sk, sh, sl, e):
    s1, lo, hi = C.c_uint64(), C.c_uint64(), C.c_uint64()
    v = probe.mom_probe_final(fn, n, sk, sh, sl, e, C.byref(s1), C.byref(lo), C.byref(hi))
    return v, s1.value, (hi.value << 64) | lo.value


NAMES = {VARPOP: "VARPOP", VARSAMP: "VARSAMP", STDDEVPOP: "STDDEVPOP", STDDEVSAMP: "STDDEVSAMP"}


@pytest.mark.parametrize("ks", [[], [5], [0, (1 << 32) - 1], [3, 3, 3], [1, 2, 3, 4, 1000], list(range(0, 1 << 32, 1 << 27))])
@pytest.mark.parametrize("e", [0, -3, 10])
def test_finalize_against_fractions(probe, ks, e):
    sk, sh, sl = _device_sums(ks)
    for fn, name in NAMES.items():
        v, s1, s2 = _final(probe, fn, len(ks), sk, sh, sl, e)
        assert s1 == sum(ks) and s2 == sum(k * k for k in ks)
        sums = (len(ks), Fraction(sum(ks)) * Fraction(2) ** e, Fraction(sum(k * k for k in ks)) * Fraction(2) ** (2 * e))
        want = vr.final(name, sums)
        assert struct.pack("<d", v) == struct.pack("<d", want), (name, ks, e, v, want)


def test_finalize_128_bit_bounds(probe):
    """n = 2^32 - 1 rows of k = 2^32 - 1 (zero variance), and the same with one row at 0: the largest moments a result
    can hold."""
    n, k = (1 << 32) - 1, (1 << 32) - 1
    hi, lo = (k * k) >> 32, (k * k) & 0xFFFFFFFF
    bias = n << 31
    sk, sh, sl = n * k - bias, n * hi - bias, n * lo - bias
    assert all(-(1 << 63) <= x < (1 << 63) for x in (sk, sh, sl))
    for fn, name in NAMES.items():
        v, s1, s2 = _final(probe, fn, n, sk, sh, sl, 0)
        assert v == 0.0 and s1 == n * k and s2 == n * k * k
    # n - 1 rows at 2^32 - 1 and one at 0
    sk2, sh2, sl2 = (n - 1) * k - bias, (n - 1) * hi - bias, (n - 1) * lo - bias
    for fn, name in NAMES.items():
        v, s1, s2 = _final(probe, fn, n, sk2, sh2, sl2, 0)
        sums = (n, Fraction((n - 1) * k), Fraction((n - 1) * k * k))
        assert v == vr.final(name, sums), name


def test_finalize_empty_and_single(probe):
    for fn in NAMES:
        assert _final(probe, fn, 0, 0, 0, 0, 0)[0] == -math.inf
    sk, sh, sl = _device_sums([42])
    assert [_final(probe, fn, 1, sk, sh, sl, 0)[0] for fn in NAMES] == [0.0, -math.inf, 0.0, -math.inf]


# ---- planner -------------------------------------------------------------------------------------------------------
D, R, S = _lib.FWD_DICT_FIXEDBIT, _lib.FWD_RAW_FIXEDBYTE, _lib.STRING
# columns: 0 INT card 10 (group key), 1 INT card 1000, 2 DOUBLE card 2^12, 3 STRING card 100, 4 raw INT streamed,
#          5 DOUBLE off the grid, 6 LONG card 300 (limbs not prepared), 7 INT card 5000
COLS = [(D, _lib.INT, 4, 10, 1, 1, 1), (D, _lib.INT, 10, 1000, 1, 2, 1), (D, _lib.DOUBLE, 12, 4096, 1, 3, 1),
        (D, S, 7, 100, 0, 4, -1), (R, _lib.INT, 32, 0, 0, 0, -1), (D, _lib.DOUBLE, 8, 200, 1, 5, 0),
        (D, _lib.LONG, 9, 300, 1, 6, -1), (D, _lib.INT, 13, 5000, 1, 7, 1)]


def plan(probe, aggs, group_by=(), num_docs=(100_000,), merge=False, cols=None, flags=0):
    n = len(num_docs)
    pc = (ProbeCol * (n * len(COLS)))()
    for s in range(n):
        for k, c in enumerate(cols[s] if cols is not None else COLS):
            pc[s * len(COLS) + k] = ProbeCol(*c)
    ag = (_lib.Agg * len(aggs))(*[_lib.Agg(f, c) for f, c in aggs])
    gb = (C.c_int32 * max(1, len(group_by)))(*group_by)
    q = _lib.Query(0, len(group_by), len(aggs), 100_000, 10_000, flags | (2 if merge else 0), None, gb, ag, 0, 0, 0)
    out = ProbePlan()
    rc = probe.mom_probe_plan_scan(H100[0], H100[1], C.byref(q), pc, len(COLS), (C.c_int32 * n)(*num_docs), n, C.byref(out))
    return rc, out


def test_expansion_and_sharing(probe):
    rc, o = plan(probe, [(VARPOP, 1), (COUNT, -1), (STDDEVSAMP, 1)])
    assert rc == 0 and o.num_user_aggs == 3 and o.num_aggs == 6
    assert list(o.mom_first)[:3] == [3, -1, 3]           # one triple for both functions of column 1
    assert list(o.limb) == [-1, -1, -1, 0, 1, 2]
    assert list(o.fn)[:6] == [VARPOP, COUNT, STDDEVSAMP, SUM, SUM, SUM]
    assert list(o.slot)[:3] == [-1, -1, -1] and o.slot[3] == o.slot[4] == o.slot[5] >= 0
    assert o.num_slots == 1 and o.projected == 1          # the column is streamed (and counted) once
    assert list(o.dict_off)[3:6] == [0, 1000, 2000]      # K, H, L of the column's limb dictionaries
    assert all(o.val_kind[a] == 1 for a in (3, 4, 5))   # VAL_DICT_I32: limb words are biased INT values
    rc, o = plan(probe, [(VARSAMP, 2), (STDDEVPOP, 2), (VARPOP, 2)])   # three functions of one column: 3 + 3
    assert rc == 0 and o.num_aggs == 6 and list(o.mom_first)[:3] == [3, 3, 3]


def test_no_limb_carrier_and_no_spec_route(probe):
    # GROUP BY with an INT SUM: the user's SUM may carry the count, a limb sum never does
    rc, o = plan(probe, [(SUM, 1), (VARPOP, 2)], group_by=[0])
    assert rc == 0 and o.carrier_agg in (-1, 0)
    rc, o = plan(probe, [(VARPOP, 1)], group_by=[0])
    assert rc == 0 and o.carrier_agg == -1 and o.need_count == 1
    assert o.smem_groups > 0 and o.spec == 0             # the shared-memory table, but not the specialised kernel
    rc, o = plan(probe, [(COUNT, -1), (SUM, 1)], group_by=[0])
    assert rc == 0 and o.spec == 1                       # the same shape without moments does take it


def test_refusals(probe):
    E_INV, E_UNS = _lib.E_INVALID, _lib.E_UNSUPPORTED
    assert plan(probe, [(VARPOP, 3)])[0] == E_UNS                         # STRING
    assert plan(probe, [(VARPOP, 4)])[0] == E_UNS                         # raw INT streamed as 32-bit values
    assert plan(probe, [(VARPOP, 5)])[0] == E_UNS                         # off a 2^32-step grid
    assert plan(probe, [(VARPOP, 6)])[0] == E_INV                         # limb dictionaries not prepared
    assert plan(probe, [(VARPOP, 1), (VARPOP, 2)])[0] == E_UNS            # 2 + 6 internal sums > kMaxAggs
    assert plan(probe, [(VARPOP, 1), (COUNT, -1), (SUM, 2), (AVG, 7)])[0] == E_UNS   # 4 + 3 > 6
    assert plan(probe, [(VARPOP, 1), (COUNT, -1), (SUM, 2)])[0] == 0
    assert plan(probe, [(VARPOP, 99)])[0] == E_INV                        # column out of range
    assert plan(probe, [(VARPOP, 1)], group_by=[0], num_docs=(1000, 1000), merge=True, flags=4)[0] == E_UNS  # deferred
    big = (2_000_000_000, 2_000_000_000, 500_000_000)
    assert plan(probe, [(VARPOP, 1)], num_docs=big, merge=True)[0] == E_UNS   # 2^32 docs in one result
    assert plan(probe, [(VARPOP, 1)], num_docs=big)[0] == 0
    other = [list(COLS), [c if k != 1 else (D, _lib.INT, 10, 1000, 1, 99, 1) for k, c in enumerate(COLS)]]
    assert plan(probe, [(VARPOP, 1)], num_docs=(1000, 1000), merge=True, cols=other)[0] == E_UNS   # two dictionaries
    assert plan(probe, [(VARPOP, 1)], num_docs=(1000, 1000), cols=other)[0] == 0
    assert plan(probe, [(6, -1)])[0] == E_INV                             # the unknown-function refusal is unchanged


# ---- the CLI's by-value merge --------------------------------------------------------------------------------------
def _block(rows, moments, keys=None):
    return ResultsBlock(-1 if keys is None else len(keys), "NONE", False, ExecutionStatistics(0, 0, 0, 0),
                        np.zeros((0, 0), dtype=np.int32) if keys is None else np.asarray(keys, dtype=np.int32).reshape(-1, 1),
                        [np.zeros(rows)], [np.zeros(rows, dtype=np.int64)], [np.full(rows, -1, dtype=np.int32)],
                        moments=moments)


class _Seg:
    def dictionary_value(self, column, d):
        return d


def _moments_of(values, c_mant, c_exp, e):
    c = Fraction(c_mant) * Fraction(2) ** c_exp
    ks = [(Fraction(v) - c) / Fraction(2) ** e for v in values]
    assert all(k.denominator == 1 and 0 <= k < 2 ** 32 for k in ks)
    return Moments(len(values), c_mant, c_exp, e, int(sum(ks)), int(sum(k * k for k in ks)))


def test_cli_merges_moments_of_different_grids():
    a = [-1.5, 2.25, 7.0, 7.0]                     # c = -1.5 = -3 * 2^-1, grid 2^-2
    b = [1 << 40, (1 << 40) + 1024]                # c = 2^40, grid 2^10
    c = []                                          # a segment without a matched row
    parts = [_moments_of(a, -3, -1, -2), _moments_of(b, 1, 40, 10), Moments(0, 0, 0, 0, 0, 0)]
    for fn in vr.FUNCTIONS:
        q = QueryContext(aggregations=[Aggregation(fn, "x")])
        blocks = [_block(1, {(0, 0): m}) for m in parts]
        rows = cli.final_rows(q, cli.merge_blocks(q, [_Seg()] * 3, blocks))
        assert rows == [[vr.final(fn, vr.exact_sums(np.asarray(a + b + c, dtype=np.float64)))]]
        assert rows[0][0] == moments_final(fn, merge_moments(parts))

"""CPU tests of single-column transforms: the SQL front end's canonical text and refusals, the host layer's expression
compiler and normaliser, and the __host__ __device__ evaluator the derivation kernel runs (both through
tests/transform_probe/transform_probe.cpp) against the independent reference tests/transform_ref.py, on seeded random
values plus the edges: the INT / LONG ends, +-2^53 and the values just past them, negative instants, the 1900 / 2000 /
2100 leap rules, ISO week 1 / 53 boundaries, quarter starts, x / 0, 0 / 0 and -0.0."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import transform_ref as ref
from pinot_b200 import _lib, sql

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
B53 = 1 << 53
TYPES = {"INT": _lib.INT, "LONG": _lib.LONG, "FLOAT": _lib.FLOAT, "DOUBLE": _lib.DOUBLE}
KINDS = {_lib.INT: "INT", _lib.LONG: "LONG", _lib.DOUBLE: "DOUBLE"}


# ---- SQL front end -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("text,canonical", [
    ("DATETRUNC('DAY', ts)", "datetrunc('DAY',ts)"),
    ("date_trunc('hour', ts, 'milliseconds', 'UTC', 'seconds')", "datetrunc('HOUR',ts,'MILLISECONDS','UTC','SECONDS')"),
    ("ts / 1000", "divide(ts,'1000')"),
    ("ts / 1000.0", "divide(ts,'1000')"),
    ("DIVIDE(ts, '1e3')", "divide(ts,'1000')"),
    ("x * 2.5 + 1", "plus(times(x,'2.5'),'1')"),
    ("x - 1", "minus(x,'1')"),
    ("x -1", "minus(x,'1')"),
    ("3 - x % 7", "minus('3',mod(x,'7'))"),
    ("(x + 1) * 2", "times(plus(x,'1'),'2')"),
    ("FLOOR(x / 100)", "floor(divide(x,'100'))"),
    ("DOW(ts)", "dayofweek(ts)"),
    ("WEEK_OF_YEAR(ts)", "week(ts)"),
    ("TIMECONVERT(ts, 'milliseconds', 'HOURS')", "timeconvert(ts,'MILLISECONDS','HOURS')"),
    ("ToEpochSecondsBucket(ts, 10)", "toepochsecondsbucket(ts,'10')"),
    ("year(datetrunc('MONTH', ts))", "year(datetrunc('MONTH',ts))"),
])
def test_sql_canonical_text(text, canonical):
    q = sql.parse(f"SELECT {text}, COUNT(*), SUM({text}) FROM t WHERE {text} > 3 GROUP BY {text} ORDER BY {text} DESC")
    assert q.group_by == [canonical]
    assert q.aggregations[1].column == canonical
    assert q.filter.column == canonical
    assert sql.resolve_order_by(q) == [("GROUP_BY", 0, False)]
    assert sql.parse_selection(f"SELECT {text} FROM t ORDER BY {text} LIMIT 3").columns == [canonical]
    assert sql.parse_distinct(f"SELECT DISTINCT {text} FROM t ORDER BY {text} LIMIT 3").order_by == [(canonical, True)]


def test_sql_order_by_aggregation_of_expression():
    q = sql.parse("SELECT g, SUM(x / 2), MAX(YEAR(ts)) FROM t GROUP BY g ORDER BY MAX(year(ts)) DESC, SUM(x/2)")
    assert sql.resolve_order_by(q) == [("AGG", 1, False), ("AGG", 0, True)]


@pytest.mark.parametrize("text", [
    "SELECT MODE(a), COUNT(*) FROM t GROUP BY MODE(a)",            # not a transform
    "SELECT COUNT(*) FROM t GROUP BY 5",                           # a literal is no column
    "SELECT x + 1, COUNT(*) FROM t GROUP BY x",                    # select item not a GROUP BY expression
    "SELECT SUM(x +) FROM t",
    "SELECT DISTINCT SUM(x) FROM t",
])
def test_sql_refusals(text):
    with pytest.raises(sql.SqlError):
        if sql.is_distinct(text):
            sql.parse_distinct(text)
        else:
            sql.parse(text)


# ---- probe ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "transform_probe", "transform_probe.cpp")
    out = os.path.join(HERE, "transform_probe", "libtransform_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    deps = [src, _lib.LIB_PATH, os.path.join(ROOT, "pinot_b200", "csrc", "pb200_transform.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.tp_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_int32]
    p64, pd, p32 = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_int32)
    lib.tp_eval.argtypes = [C.c_char_p, C.c_int32, C.c_int32, p64, pd, p32, p64, pd, C.POINTER(C.c_uint64), p32]
    return lib


def compile_text(probe, text):
    buf = C.create_string_buffer(1024)
    n = probe.tp_compile(text.encode(), buf, 1024)
    return n, buf.value.decode()


@pytest.mark.parametrize("a,b", [
    ("datetrunc('DAY',ts)", "DATE_TRUNC( 'day' , ts )"),
    ("datetrunc('DAY',ts)", "DateTrunc('Day', ts)"),
    ("divide(ts,'1000')", "div(ts, 1000.0)"),
    ("divide(ts,'1000')", "DIVIDE(ts,'1e3')"),
    ("plus(x,'0.5')", "add(x,'.5')"),
    ("dayofweek(ts)", "dow(ts)"),
    ("dayofyear(ts)", "DOY(ts)"),
    ("week(ts)", "weekOfYear(ts)"),
    ("day(ts)", "day_of_month(ts)"),
    ("timeconvert(ts,'MILLISECONDS','HOURS')", "timeConvert(ts, 'milliseconds', 'hours')"),
    ("datetrunc('WEEK',ts,'SECONDS','UTC','DAYS')", "datetrunc('week', ts, 'seconds', 'utc', 'days')"),
])
def test_two_spellings_one_key(probe, a, b):
    ra, ca = compile_text(probe, a)
    rb, cb = compile_text(probe, b)
    assert ra > 0 and rb > 0
    assert ca == cb == a


@pytest.mark.parametrize("text,code", [
    ("plus(a,b)", _lib.E_UNSUPPORTED),                         # two columns
    ("plus(a,a)", _lib.E_UNSUPPORTED),
    ("upper(s)", _lib.E_UNSUPPORTED),                          # unknown function
    ("datetrunc('DAY',ts,'MILLISECONDS','America/Denver')", _lib.E_UNSUPPORTED),
    ("datetrunc('FORTNIGHT',ts)", _lib.E_UNSUPPORTED),
    ("timeconvert(ts,'MILLISECONDS')", _lib.E_UNSUPPORTED),    # argument count
    ("year(ts,'UTC')", _lib.E_UNSUPPORTED),
    ("plus(x,'abc')", _lib.E_UNSUPPORTED),                     # non-numeric literal
    ("plus(x,'0x10')", _lib.E_UNSUPPORTED),                    # literals are decimal: no hex, NaN or infinity
    ("plus(x,'nan')", _lib.E_UNSUPPORTED),
    ("times(x,'Infinity')", _lib.E_UNSUPPORTED),
    ("plus(x,'1e')", _lib.E_UNSUPPORTED),
    ("plus(x,'1'", _lib.E_INVALID),                            # malformed
    ("plus(x,,'1')", _lib.E_INVALID),
    ("x", _lib.E_INVALID),                                     # no expression
    ("plus(x,'1') y", _lib.E_INVALID),
])
def test_compile_refusals(probe, text, code):
    assert compile_text(probe, text)[0] == code


def test_operation_limit(probe):
    e = "x"
    for _ in range(16):
        e = f"plus({e},'1')"
    vals = np.zeros(1, dtype=np.int64)
    assert _eval(probe, e, "LONG", vals)[0] == "DOUBLE"
    assert _eval_rc(probe, f"abs({e})", "LONG", vals) == _lib.E_UNSUPPORTED


def test_type_rules(probe):
    one = np.zeros(1)
    for text in ("year(x)", "datetrunc('DAY',x)", "timeconvert(x,'SECONDS','DAYS')", "toepochseconds(x)", "year(plus(x,'1'))"):
        assert _eval_rc(probe, text, "DOUBLE", one) == _lib.E_UNSUPPORTED
        assert _eval_rc(probe, text, "FLOAT", one) == _lib.E_UNSUPPORTED
    assert _eval_rc(probe, "toepochsecondsbucket(x,'0')", "LONG", np.zeros(1, dtype=np.int64)) == _lib.E_UNSUPPORTED
    assert _eval_rc(probe, "toepochsecondsbucket(x,'2.5')", "LONG", np.zeros(1, dtype=np.int64)) == _lib.E_UNSUPPORTED
    # an integral bucket is the same program however it is spelled
    assert _eval(probe, "toepochsecondsbucket(x,'10.0')", "LONG", np.array([123_456], dtype=np.int64))[1].tolist() == [12]
    assert _eval(probe, "toepochsecondsbucket(x,'1e1')", "LONG", np.array([123_456], dtype=np.int64))[1].tolist() == [12]
    assert _eval_rc(probe, "year(x)", "STRING", np.zeros(1, dtype=np.int64)) == _lib.E_UNSUPPORTED


# ---- evaluator against the reference --------------------------------------------------------------------------------
def _eval_rc(probe, text, source_type, values):
    n = len(values)
    si = np.ascontiguousarray(values, dtype=np.int64) if source_type in ("INT", "LONG", "STRING") else None
    sd = np.ascontiguousarray(values, dtype=np.float64) if source_type in ("FLOAT", "DOUBLE") else None
    kind = C.c_int32()
    oi, od = np.zeros(n, np.int64), np.zeros(n, np.float64)
    key, ok = np.zeros(n, np.uint64), np.zeros(n, np.int32)
    st = TYPES.get(source_type, _lib.STRING)
    rc = probe.tp_eval(text.encode(), st, n, si.ctypes.data_as(C.POINTER(C.c_int64)) if si is not None else None,
                       sd.ctypes.data_as(C.POINTER(C.c_double)) if sd is not None else None, C.byref(kind),
                       oi.ctypes.data_as(C.POINTER(C.c_int64)), od.ctypes.data_as(C.POINTER(C.c_double)),
                       key.ctypes.data_as(C.POINTER(C.c_uint64)), ok.ctypes.data_as(C.POINTER(C.c_int32)))
    _eval_rc.last = (kind.value, oi, od, key, ok)
    return rc


def _eval(probe, text, source_type, values):
    rc = _eval_rc(probe, text, source_type, values)
    assert rc == 0, (text, rc)
    kind, oi, od, key, ok = _eval_rc.last
    return KINDS[kind], oi, od, key, ok


def _edges_ms():
    days = [(1900, 2, 28), (1900, 3, 1), (2000, 2, 29), (2000, 3, 1), (2100, 2, 28), (2100, 3, 1), (1969, 12, 31),
            (1970, 1, 1), (2004, 12, 31), (2005, 1, 1), (2005, 1, 2), (2005, 1, 3), (2008, 12, 29), (2009, 12, 31),
            (2010, 1, 3), (2010, 1, 4), (2015, 12, 31), (2016, 1, 1), (2020, 12, 31), (2021, 1, 3), (2026, 4, 1),
            (2026, 3, 31), (2026, 7, 1), (2026, 10, 1), (1600, 1, 1), (-1, 12, 31), (1, 1, 1)]
    out = []
    for y, m, d in days:
        base = int(np.datetime64(f"{y:05d}-{m:02d}-{d:02d}" if y >= 0 else f"-{-y:05d}-{m:02d}-{d:02d}", "ms").astype(np.int64))
        out += [base, base - 1, base + 86_399_999, base + 43_200_123]
    return out + [-1, 0, 1, -86_400_000, B53, -B53, B53 - 1, 1_767_225_600_000]


def _seeded(seed, n, lo, hi):
    return np.random.default_rng(seed).integers(lo, hi, size=n, dtype=np.int64).tolist()


TIME_EXPRS = ["datetrunc('MILLISECOND',x)", "datetrunc('SECOND',x)", "datetrunc('MINUTE',x)", "datetrunc('HOUR',x)",
              "datetrunc('DAY',x)", "datetrunc('WEEK',x)", "datetrunc('MONTH',x)", "datetrunc('QUARTER',x)",
              "datetrunc('YEAR',x)", "datetrunc('DAY',x,'SECONDS')", "datetrunc('HOUR',x,'MILLISECONDS','UTC','HOURS')",
              "datetrunc('WEEK',x,'DAYS','UTC','MILLISECONDS')",
              *[f"{f}(x)" for f in ref.CALENDAR],
              "timeconvert(x,'MILLISECONDS','SECONDS')", "timeconvert(x,'SECONDS','MILLISECONDS')",
              "timeconvert(x,'DAYS','NANOSECONDS')", "timeconvert(x,'NANOSECONDS','DAYS')", "timeconvert(x,'HOURS','MINUTES')",
              "toepochseconds(x)", "toepochminutes(x)", "toepochhours(x)", "toepochdays(x)",
              "toepochsecondsbucket(x,'10')", "toepochminutesbucket(x,'15')", "toepochhoursbucket(x,'6')", "toepochdaysbucket(x,'7')",
              "toepochsecondsrounded(x,'10')", "toepochhoursrounded(x,'3')", "toepochdaysrounded(x,'7')", "toepochminutesrounded(x,'5')",
              "year(datetrunc('QUARTER',x))", "dayofweek(timeconvert(x,'SECONDS','MILLISECONDS'))"]
ARITH_EXPRS = ["plus(x,'1')", "minus(x,'0.1')", "minus('3',x)", "times(x,'-3')", "times(x,'0.1')", "divide(x,'1000')",
               "divide('1',x)", "divide(x,'0')", "divide(x,'-0.0')", "mod(x,'10000')", "mod('7',x)", "mod(x,'-3.5')",
               "floor(x)", "ceil(x)", "abs(x)", "floor(divide(x,'100'))", "ceil(times(x,'-0.5'))",
               "plus(times(x,'0.1'),'0.7')", "abs(minus(mod(x,'7'),'3'))", "divide(divide(x,'3'),'7')"]


def _check(probe, text, source_type, values):
    kind, oi, od, key, ok = _eval(probe, text, source_type, values)
    for k, v in enumerate(values):
        try:
            want_kind, want = ref.evaluate(text, v, source_type)
        except ref.Refused:
            assert not ok[k], (text, v)
            continue
        assert ok[k], (text, v)
        assert kind == want_kind, (text, kind, want_kind)
        if kind == "DOUBLE":
            got = float(od[k])
            assert ref.double_order_key(got) == ref.double_order_key(want), (text, v, got, want)
            assert int(key[k]) == ref.double_order_key(want), (text, v)
        else:
            assert int(oi[k]) == want, (text, source_type, v, int(oi[k]), want)


@pytest.mark.parametrize("text", TIME_EXPRS)
def test_time_functions(probe, text):
    values = _edges_ms() + _seeded(hash(text) & 0xFFFF, 300, -B53, B53) + _seeded(7, 100, -10 ** 12, 4 * 10 ** 12)
    past = [B53 + 1, -B53 - 1, INT64_MIN, INT64_MAX]
    _check(probe, text, "LONG", values + past)
    _check(probe, text, "INT", [INT_MIN, INT_MAX, -1, 0, 1, 999, -1000] + _seeded(3, 50, INT_MIN, INT_MAX))


def test_timeconvert_saturates(probe):
    for text in ("timeconvert(x,'DAYS','NANOSECONDS')", "timeconvert(x,'SECONDS','MILLISECONDS')",
                 "datetrunc('DAY',x,'DAYS','UTC','NANOSECONDS')"):
        _check(probe, text, "LONG", [INT64_MIN, INT64_MAX, INT64_MAX // 1000, INT64_MAX // 1000 + 1, -(INT64_MAX // 1000) - 1, 106_751, -106_752, 0])
    _, oi, _, _, _ = _eval(probe, "timeconvert(x,'SECONDS','MILLISECONDS')", "LONG", [INT64_MAX, INT64_MIN])
    assert oi.tolist() == [INT64_MAX, INT64_MIN]


@pytest.mark.parametrize("text", ARITH_EXPRS)
@pytest.mark.parametrize("source_type", ["INT", "LONG", "FLOAT", "DOUBLE"])
def test_arithmetic(probe, text, source_type):
    rng = np.random.default_rng(abs(hash((text, source_type))) & 0xFFFF)
    if source_type == "INT":
        values = [INT_MIN, INT_MAX, 0, -1, 1, 7, -7] + rng.integers(INT_MIN, INT_MAX, size=200).tolist()
    elif source_type == "LONG":
        values = [INT64_MIN, INT64_MAX, B53, B53 + 1, -B53 - 1, 0, -1] + rng.integers(INT64_MIN, INT64_MAX, size=200, dtype=np.int64).tolist()
    else:
        base = rng.normal(0, 1e6, size=200)
        if source_type == "FLOAT":
            base = base.astype(np.float32).astype(np.float64)
        values = [0.0, -0.0, 1.5, -2.5, math.inf, -math.inf, math.nan, 1e300, -1e-300] + base.tolist()
    _check(probe, text, source_type, values)


def test_double_order(probe):
    """Results order like Double.compare: -0.0 before 0.0 (distinct groups), every NaN one group after +inf."""
    _, _, od, key, _ = _eval(probe, "divide(x,'0')", "DOUBLE", [1.0, -1.0, 0.0, -0.0, math.nan])
    k = [int(v) for v in key]
    assert k[1] < k[0] and k[4] > k[0] and k[2] == k[3] == k[4]    # -inf < inf < NaN; 0/0 and -0/0 are one NaN
    _, _, od, key, _ = _eval(probe, "times(x,'1')", "DOUBLE", [-0.0, 0.0])
    assert int(key[0]) < int(key[1])

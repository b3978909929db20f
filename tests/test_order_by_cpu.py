"""CPU tests of ORDER BY: the broker-side ordering of pinot_b200.cli.final_rows, the resolution of ORDER BY expressions
(pinot_b200.sql.resolve_order_by), and the library's key function (pinot_b200/csrc/pb200_order.h, shared by the device
sort and the host sort) compiled with g++ and checked against Python's sort of the same doubles and integers."""
import ctypes as C
import os
import struct
import subprocess

import pytest

from pinot_b200 import cli, sql

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _q(text, **kw):
    return sql.parse(text, **kw)


# ------------------------------------------------------------------------------------------------ cli.final_rows
TABLE = {  # key values: [COUNT, SUM, AVG (sum, count), DISTINCTCOUNT set, MIN]
    ("a", 1): [3, 10.0, (10.0, 3), {1, 2}, -0.0],
    ("b", 1): [3, -5.0, (-5.0, 3), {1}, 0.0],
    ("a", 2): [1, 10.0, (10.0, 1), {1, 2, 3}, 2.0],
    ("c", 0): [7, 0.0, (0.0, 0), set(), float("inf")],
    ("b", 0): [3, 10.0, (9.0, 3), {4, 5}, float("-inf")],
}
SELECT = "SELECT COUNT(*), SUM(m), AVG(m), DISTINCTCOUNT(d), MIN(m) FROM t GROUP BY s, k"


def _keys(rows):
    return [tuple(r[:2]) for r in rows]


def test_final_rows_desc_with_ties_by_key_values():
    rows = cli.final_rows(_q(SELECT + " ORDER BY COUNT(*) DESC LIMIT 10"), TABLE)
    assert _keys(rows) == [("c", 0), ("a", 1), ("b", 0), ("b", 1), ("a", 2)]


def test_final_rows_asc_and_limit():
    rows = cli.final_rows(_q(SELECT + " ORDER BY SUM(m) LIMIT 3"), TABLE)
    assert _keys(rows) == [("b", 1), ("c", 0), ("a", 1)]


def test_final_rows_avg_orders_by_the_quotient_and_empty_avg_is_lowest():
    rows = cli.final_rows(_q(SELECT + " ORDER BY AVG(m) DESC LIMIT 10"), TABLE)
    assert _keys(rows) == [("a", 2), ("a", 1), ("b", 0), ("b", 1), ("c", 0)]
    assert rows[-1][4] == float("-inf")


def test_final_rows_distinctcount_then_key_desc():
    rows = cli.final_rows(_q(SELECT + " ORDER BY DISTINCTCOUNT(d) DESC, s DESC LIMIT 10"), TABLE)
    assert _keys(rows) == [("a", 2), ("b", 0), ("a", 1), ("b", 1), ("c", 0)]


def test_final_rows_minus_zero_before_zero():
    rows = cli.final_rows(_q(SELECT + " ORDER BY MIN(m) LIMIT 10"), TABLE)
    assert _keys(rows) == [("b", 0), ("a", 1), ("b", 1), ("a", 2), ("c", 0)]


def test_final_rows_without_order_by_unchanged():
    rows = cli.final_rows(_q(SELECT + " LIMIT 2"), TABLE)
    assert _keys(rows) == [("a", 1), ("a", 2)]


# ------------------------------------------------------------------------------------------------ resolution
def test_order_by_resolution():
    q = _q("SELECT k, SUM(m), COUNT(x), MAX(m) FROM t GROUP BY k, s ORDER BY s DESC, count(*), MAX(m) DESC, k")
    assert sql.resolve_order_by(q) == [("GROUP_BY", 1, False), ("AGG", 1, True), ("AGG", 2, False), ("GROUP_BY", 0, True)]


@pytest.mark.parametrize("text", ["SELECT SUM(m) FROM t GROUP BY k ORDER BY MAX(m)",
                                  "SELECT SUM(m) FROM t GROUP BY k ORDER BY SUM(x)",
                                  "SELECT SUM(m) FROM t GROUP BY k ORDER BY s",
                                  "SELECT SUM(m) FROM t GROUP BY k ORDER BY AVG(m) DESC"])
def test_order_by_outside_the_select_list_is_refused(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


# ------------------------------------------------------------------------------------------------ key function
SHIM = r"""
#include "pb200_order.h"
extern "C" uint64_t probe_order_key(int cmp, int desc, uint64_t mask, double dv, int64_t lv) {
  return pb200::order_key(cmp, desc != 0, mask, dv, lv);
}
extern "C" int probe_order_cmp_of(int fn) { return pb200::order_cmp_of(fn); }
"""


@pytest.fixture(scope="module")
def keyfn(tmp_path_factory):
    d = tmp_path_factory.mktemp("order_probe")
    src, out = d / "probe.cpp", d / "libprobe.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{os.path.join(ROOT, 'pinot_b200', 'csrc')}",
                    "-o", str(out), str(src)], check=True)
    lib = C.CDLL(str(out))
    lib.probe_order_key.restype = C.c_uint64
    lib.probe_order_key.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_double, C.c_int64]
    lib.probe_order_cmp_of.argtypes = [C.c_int]
    return lib


LONG, DOUBLE, AVG = 0, 1, 2
ALL = (1 << 64) - 1
DOUBLES = [float("-inf"), -1.7976931348623157e308, -1.0, -5e-324, -0.0, 0.0, 5e-324, 2.2250738585072014e-308, 1.0,
           2.0 ** 53, 1.7976931348623157e308, float("inf")]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def test_function_to_comparison(keyfn):
    assert [keyfn.probe_order_cmp_of(f) for f in range(6)] == [LONG, DOUBLE, DOUBLE, DOUBLE, AVG, LONG]


def test_double_keys_follow_double_compare(keyfn):
    shuffled = DOUBLES[::-1][1::2] + DOUBLES[::-1][0::2]
    asc = sorted(shuffled, key=lambda x: keyfn.probe_order_key(DOUBLE, 0, ALL, x, 0))
    assert [_bits(x) for x in asc] == [_bits(x) for x in DOUBLES]   # -0.0 before 0.0, bit for bit
    desc = sorted(shuffled, key=lambda x: keyfn.probe_order_key(DOUBLE, 1, ALL, x, 0))
    assert [_bits(x) for x in desc] == [_bits(x) for x in DOUBLES[::-1]]


def test_long_keys_and_narrowed_desc(keyfn):
    vals = [0, 1, 2, 1000, (1 << 53) + 1, (1 << 63) - 1]
    assert sorted(vals[::-1], key=lambda v: keyfn.probe_order_key(LONG, 0, ALL, 0.0, v)) == vals
    assert sorted(vals, key=lambda v: keyfn.probe_order_key(LONG, 1, ALL, 0.0, v)) == vals[::-1]
    small = [0, 3, 5, 7]   # 3 bits in use: DESC keys stay inside them
    keys = [keyfn.probe_order_key(LONG, 1, 7, 0.0, v) for v in small]
    assert keys == [7, 4, 2, 0]


def test_avg_keys(keyfn):
    rows = [(10.0, 4), (-3.0, 1), (0.0, 0), (9.0, 3), (-(2.0 ** 63), 1), (1e308, 1)]
    want = sorted(rows, key=lambda r: r[0] / r[1] if r[1] else float("-inf"))
    assert sorted(rows, key=lambda r: keyfn.probe_order_key(AVG, 0, ALL, r[0], r[1])) == want
    assert keyfn.probe_order_key(AVG, 0, ALL, 5.0, 0) == keyfn.probe_order_key(DOUBLE, 0, ALL, float("-inf"), 0)

"""Multi-column expression aggregations without a GPU (DESIGN.md section 3.15): the host compiler (canonical text, leaves,
refusals), the per-row evaluator of pb200_expr.h through a g++ probe against the independent reference tests/expr_ref.py
on seeded values and at the edges (INT / LONG ends, 2^53 + 1, x / 0, 0 / 0, -0.0, NaN, +-inf), the MIN / MAX key, the
program check, the Python-side test of the per-row route, and the cross-GPU refusal."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

from expr_ref import columns, evaluate, order_key, parse
from pinot_b200 import _lib
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED
from pinot_b200.query import Aggregation, QueryContext, is_multi_column_expression

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
T_COLUMN, T_LONG, T_DOUBLE, T_PLUS, T_TIMES, T_DATETRUNC = 0, 1, 2, 3, 5, 11
MIN, MAX = 2, 3


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "expr_probe", "expr_probe.cpp")
    out = os.path.join(HERE, "expr_probe", "libexpr_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    deps = [src, _lib.LIB_PATH, os.path.join(ROOT, "pinot_b200", "csrc", "pb200_expr.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.ep_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32]
    lib.ep_is_multi.argtypes = [C.c_char_p]
    lib.ep_compile_single.argtypes = [C.c_char_p]
    lib.ep_eval.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double),
                            C.POINTER(C.c_double)]
    lib.ep_check.argtypes = [C.POINTER(_lib.TransformOp), C.c_int32, C.POINTER(C.c_int32)]
    lib.ep_key.restype = C.c_uint64
    lib.ep_key.argtypes = [C.c_double]
    lib.ep_key_value.restype = C.c_double
    lib.ep_key_value.argtypes = [C.c_int32, C.c_uint64]
    return lib


def compile_multi(probe, text):
    canon, leaves = C.create_string_buffer(1024), C.create_string_buffer(1024)
    n = probe.ep_compile(text.encode(), canon, leaves, 1024)
    return n, canon.value.decode(), leaves.value.decode()


@pytest.mark.parametrize("a,b", [("times(price,qty)", "TIMES( price , qty )"), ("times(price,qty)", "mult(price,qty)"),
                                 ("divide(b,plus(a,'1'))", "div(b, add(a, 1.0))"), ("plus(a,a)", "PLUS(a,a)")])
def test_canonical_text(probe, a, b):
    na, ca, la = compile_multi(probe, a)
    nb, cb, lb = compile_multi(probe, b)
    assert na > 0 and (na, ca, la) == (nb, cb, lb)
    assert ca == a


def test_leaves(probe):
    assert compile_multi(probe, "minus(plus(a,b),times(a,'2'))")[2] == "a,b,a"
    assert compile_multi(probe, "plus(a,a)")[2] == "a,a"


@pytest.mark.parametrize("text,rc", [
    ("plus(a,'1')", E_UNSUPPORTED),                         # one column leaf: the derived-column route
    ("plus(datetrunc('DAY',ts),b)", E_UNSUPPORTED),         # a time function
    ("plus(" * 8 + "a" + ",b)" * 8, E_UNSUPPORTED),         # nine column leaves
    ("concat(a,b)", E_UNSUPPORTED),                         # outside the grammar
    ("plus(a,", E_INVALID),
])
def test_compile_refusals(probe, text, rc):
    assert compile_multi(probe, text)[0] == rc


def test_single_column_compiler_keeps_its_refusals(probe):
    assert probe.ep_compile_single(b"plus(a,b)") == E_UNSUPPORTED
    assert probe.ep_compile_single(b"plus(a,a)") == E_UNSUPPORTED
    assert probe.ep_is_multi(b"plus(a,b)") == 1 and probe.ep_is_multi(b"plus(a,a)") == 1
    assert probe.ep_is_multi(b"plus(a,'1')") == 0 and probe.ep_is_multi(b"a") == 0 and probe.ep_is_multi(b"concat(a,b)") == 0


def test_program_check(probe):
    def ops(*items):
        arr = (_lib.TransformOp * len(items))()
        for k, (op, i) in enumerate(items):
            arr[k].op, arr[k].i = op, i
        return arr, len(items)
    leaves = C.c_int32()
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_COLUMN, 1), (T_TIMES, 0)), C.byref(leaves)) == 0 and leaves.value == 2
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_COLUMN, 0), (T_PLUS, 0)), C.byref(leaves)) == 0
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_LONG, 3), (T_PLUS, 0)), C.byref(leaves)) == E_UNSUPPORTED
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_DATETRUNC, 4), (T_COLUMN, 1), (T_PLUS, 0)), C.byref(leaves)) == E_UNSUPPORTED
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_PLUS, 0)), C.byref(leaves)) == E_INVALID
    assert probe.ep_check(*ops((T_COLUMN, 0), (T_COLUMN, 1)), C.byref(leaves)) == E_INVALID
    assert probe.ep_check(*ops((T_COLUMN, -1), (T_COLUMN, 1), (T_PLUS, 0)), C.byref(leaves)) == E_INVALID


def _same(x, y):
    return (math.isnan(x) and math.isnan(y)) or struct.pack("<d", x) == struct.pack("<d", y)


def _run(probe, text, rows, kinds):
    """rows: {column: values}; kinds: {column: True for INT / LONG}.  Device-side values vs the reference, row by row."""
    tree = parse(text)
    leaves = columns(tree)
    n = len(next(iter(rows.values())))
    integral = (C.c_int32 * len(leaves))(*[int(kinds[c]) for c in leaves])
    ints = (C.c_int64 * (n * len(leaves)))()
    dbls = (C.c_double * (n * len(leaves)))()
    for r in range(n):
        for k, c in enumerate(leaves):
            if kinds[c]:
                ints[r * len(leaves) + k] = int(rows[c][r])
            else:
                dbls[r * len(leaves) + k] = float(rows[c][r])
    out = (C.c_double * n)()
    assert probe.ep_eval(text.encode(), n, len(leaves), integral, ints, dbls, out) == 0
    for r in range(n):
        want = evaluate(tree, {c: rows[c][r] for c in set(leaves)})
        assert _same(out[r], want), f"{text} row {r}: {out[r]!r} != {want!r} ({ {c: rows[c][r] for c in set(leaves)} })"


EDGE_INTS = [0, 1, -1, INT_MIN, INT_MAX, INT64_MIN, INT64_MAX, (1 << 53) + 1, -(1 << 53) - 1, (1 << 53), 3, -7]
EDGE_DBLS = [0.0, -0.0, 1.0, -1.0, math.nan, math.inf, -math.inf, 1e308, -1e308, 5e-324, 0.1, -2.5, 3.0, 7.5]
TEXTS = ["plus(a,b)", "minus(a,b)", "times(a,b)", "divide(a,b)", "mod(a,b)", "plus(a,a)", "floor(divide(a,b))",
         "ceil(divide(a,b))", "abs(minus(a,b))", "divide(b,plus(a,'1'))", "times(minus(a,'3.5'),b)", "plus(times(a,b),divide(a,'0'))",
         "mod(times(a,'2'),plus(b,'0.5'))"]


@pytest.mark.parametrize("text", TEXTS)
@pytest.mark.parametrize("ka,kb", [(True, True), (True, False), (False, False)])
def test_evaluator_edges(probe, text, ka, kb):
    A = EDGE_INTS if ka else EDGE_DBLS
    B = EDGE_INTS if kb else EDGE_DBLS
    pairs = [(x, y) for x in A for y in B]
    _run(probe, text, {"a": [p[0] for p in pairs], "b": [p[1] for p in pairs]}, {"a": ka, "b": kb})


@pytest.mark.parametrize("seed", range(4))
def test_evaluator_seeded(probe, seed):
    rng = np.random.default_rng(seed)
    n = 2000
    rows = {"a": rng.integers(INT_MIN, INT_MAX, size=n).tolist(), "b": (rng.standard_normal(n) * 1e3).tolist(),
            "c": rng.integers(INT64_MIN, INT64_MAX, size=n, dtype=np.int64).tolist(),
            "d": np.float32(rng.standard_normal(n)).astype(np.float64).tolist()}
    kinds = {"a": True, "b": False, "c": True, "d": False}
    for text in ("plus(times(a,b),c)", "divide(minus(c,a),d)", "mod(c,plus(a,'1'))", "abs(times(d,minus(b,a)))",
                 "floor(divide(times(a,d),plus(b,c)))", "times(plus(a,'0.25'),ceil(d))"):
        _run(probe, text, rows, kinds)


def test_min_max_key(probe):
    vals = [-math.inf, -1e308, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, 1e308, math.inf, math.nan]
    keys = [probe.ep_key(v) for v in vals]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    assert keys == [order_key(v) for v in vals]
    assert 0 not in keys and (1 << 64) - 1 not in keys               # the empty MIN / MAX entries are no double's key
    for v, k in zip(vals, keys):
        assert _same(probe.ep_key_value(MIN, k), v) and _same(probe.ep_key_value(MAX, k), v)
    assert probe.ep_key_value(MIN, (1 << 64) - 1) == math.inf and probe.ep_key_value(MAX, 0) == -math.inf
    # every NaN is one key
    assert probe.ep_key(struct.unpack("<d", struct.pack("<Q", 0xFFF0000000000123))[0]) == probe.ep_key(math.nan)


def test_python_route_test():
    assert is_multi_column_expression("SUM", "times(price,qty)") and is_multi_column_expression("MAX", "plus(a,a)")
    assert not is_multi_column_expression("SUM", "plus(a,'1')") and not is_multi_column_expression("COUNT", "times(a,b)")
    assert not is_multi_column_expression("DISTINCTCOUNT", "times(a,b)") and not is_multi_column_expression("SUM", "a")
    assert not is_multi_column_expression("SUM", "times(a,1e5)")


def test_group_by_refused_across_gpus_before_any_collective():
    from pinot_b200._lib import UnsupportedQueryError
    from pinot_b200.distributed import execute_and_combine

    class NoCollective:
        def __getattr__(self, name):
            raise AssertionError(f"collective {name} issued")
    q = QueryContext(aggregations=[Aggregation("SUM", "times(a,b)")], group_by=["g"])
    with pytest.raises(UnsupportedQueryError):
        execute_and_combine(object(), [], q, NoCollective())

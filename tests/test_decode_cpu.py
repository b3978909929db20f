"""CPU test: the result decoder of pinot_b200/csrc/pb200_decode.h (through tests/decode_probe) gives, for every function
over a one-entry table, the values an aggregation-only result has always had: no row at count 0, raw INT MIN / MAX at the
ends of u32, INT dictionary values with the device copy's bias and without it, expression keys and sums."""
import ctypes as C
import math
import os
import struct
import subprocess

import pytest

from pinot_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
A = _lib.AGG_CODES
VAL_NONE, VAL_DICT_I32, VAL_DICT_I64, VAL_DICT_F32, VAL_DICT_F64, VAL_RAW_I32 = range(6)   # pb200_desc.h
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("decode_probe") / "libdecode_probe.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out,
                    os.path.join(HERE, "decode_probe", "decode_probe.cpp")], check=True)
    lib = C.CDLL(out)
    lib.dp_decode.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int32,
                              C.c_int64, C.c_uint32, C.c_int64, C.POINTER(C.c_int64), C.c_int32, C.POINTER(C.c_uint64),
                              C.c_int64, C.c_int32, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_int64),
                              C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    return lib


def decode(probe, fn, vk=VAL_NONE, cnt=1, word=0, dict_buf=None, bias=0, pack_shift=0, pack_vmin=0, pct_n=0, wt_time=0,
           mom=(0, 0, 0), mom_e=0, ds=(0,) * 6, hll=0, xkey=None, counted=True):
    dv, lv, id_ = C.c_double(), C.c_int64(), C.c_int32()
    row = (C.c_uint64 * 3)()
    probe.dp_decode(A[fn], vk, int(counted), cnt, word, C.cast(dict_buf, C.c_void_p) if dict_buf is not None else None, bias,
                    pack_shift, pack_vmin, pct_n, wt_time, (C.c_int64 * 3)(*mom), mom_e, (C.c_uint64 * 6)(*ds), hll,
                    int(xkey is not None), xkey or 0, C.byref(dv), C.byref(lv), C.byref(id_), row)
    return dv.value, lv.value, id_.value, tuple(row)


def u64(x):
    return x & (2 ** 64 - 1)


def double_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def compare_key(x):   # Double.compare order key of a double (pb200_transform.h double_order_bits)
    b = double_bits(x)
    return b | (1 << 63) if not b >> 63 else u64(~b)


def i32_dict(values, biased):
    return (C.c_uint32 * len(values))(*[(v & 0xFFFFFFFF) ^ (0x80000000 if biased else 0) for v in values])


def test_count_and_sums(probe):
    assert decode(probe, "COUNT", cnt=5)[:3] == (5.0, 5, -1)
    assert decode(probe, "SUM", VAL_DICT_I32, cnt=3, word=u64(-7))[:3] == (-7.0, 3, -1)
    assert decode(probe, "AVG", VAL_DICT_F64, cnt=2, word=double_bits(2.5))[:3] == (2.5, 2, -1)
    assert decode(probe, "SUM", VAL_DICT_I64, cnt=2, word=double_bits(-1e300))[:3] == (-1e300, 2, -1)
    # a count-carrying entry: low field sum(value - vmin) = 9 over 3 rows with vmin -4 -> 9 - 12
    assert decode(probe, "SUM", VAL_DICT_I32, cnt=3, word=(3 << 40) | 9, pack_shift=40, pack_vmin=-4)[:3] == (-3.0, 3, -1)


@pytest.mark.parametrize("vk", [VAL_DICT_I32, VAL_DICT_I64, VAL_DICT_F64, VAL_RAW_I32])
def test_min_max_without_rows(probe, vk):
    for word_min, word_max in ((0xFFFFFFFF, 0), (0, 0xFFFFFFFF), (5, 6)):   # whatever the entries hold
        assert decode(probe, "MIN", vk, cnt=0, word=word_min)[:3] == (math.inf, 0, -1)
        assert decode(probe, "MAX", vk, cnt=0, word=word_max)[:3] == (-math.inf, 0, -1)


def test_min_max_dictionary_sentinels(probe):
    # a dictionary entry at its start value has no row even where no count is kept (a GROUP BY table without COUNT)
    assert decode(probe, "MIN", VAL_DICT_I32, cnt=0, word=0xFFFFFFFF, counted=False)[:3] == (math.inf, 0, -1)
    assert decode(probe, "MAX", VAL_DICT_I32, cnt=0, word=0, counted=False)[:3] == (-math.inf, 0, -1)


def test_raw_int_min_max_at_the_ends(probe):
    assert decode(probe, "MIN", VAL_RAW_I32, cnt=4, word=0)[:3] == (float(INT_MIN), 0, 0)
    assert decode(probe, "MAX", VAL_RAW_I32, cnt=4, word=0xFFFFFFFF)[:3] == (float(INT_MAX), 0, -1)
    assert decode(probe, "MIN", VAL_RAW_I32, cnt=4, word=0xFFFFFFFF)[:3] == (float(INT_MAX), 0, -1)
    assert decode(probe, "MAX", VAL_RAW_I32, cnt=4, word=0)[:3] == (float(INT_MIN), 0, 0)
    x = (-17 & 0xFFFFFFFF) ^ 0x80000000   # the order-preserving encoding; its int32 is the dictId column's value
    assert decode(probe, "MIN", VAL_RAW_I32, cnt=1, word=x)[:3] == (-17.0, 0, x)


@pytest.mark.parametrize("biased", [False, True])
def test_int_dictionary_bias(probe, biased):
    values = [INT_MIN, -3, 0, 7, INT_MAX]
    d = i32_dict(values, biased)
    bias = 0x80000000 if biased else 0
    for x, v in enumerate(values):
        assert decode(probe, "MIN", VAL_DICT_I32, word=x, dict_buf=d, bias=bias)[:3] == (float(v), 0, x)
        assert decode(probe, "MAX", VAL_DICT_I32, word=x + 1, dict_buf=d, bias=bias)[:3] == (float(v), 0, x)
        assert decode(probe, "PERCENTILE", VAL_DICT_I32, word=x, dict_buf=d, bias=bias, pct_n=9)[:3] == (float(v), 9, x)
        assert decode(probe, "LASTWITHTIME", VAL_DICT_I32, word=x, dict_buf=d, bias=bias, wt_time=-5)[:3] == (float(v), -5, x)


def test_other_dictionaries_and_ids(probe):
    longs = (C.c_int64 * 2)(-(2 ** 62), 2 ** 53 + 1)
    assert decode(probe, "MAX", VAL_DICT_I64, word=2, dict_buf=longs)[:3] == (float(2 ** 53 + 1), 0, 1)
    floats = (C.c_float * 2)(0.1, -2.5)
    assert decode(probe, "MIN", VAL_DICT_F32, word=0, dict_buf=floats)[:3] == (float(C.c_float(0.1).value), 0, 0)
    doubles = (C.c_double * 2)(-0.0, math.inf)
    assert decode(probe, "MAX", VAL_DICT_F64, word=2, dict_buf=doubles)[:3] == (math.inf, 0, 1)
    # a column without a value dictionary (STRING): the dictId is the value
    assert decode(probe, "MIN", VAL_DICT_I32, word=4)[:3] == (4.0, 0, 4)


def test_percentile_and_withtime_without_rows(probe):
    d = i32_dict([1, 2], False)
    for fn in ("PERCENTILE", "FIRSTWITHTIME", "LASTWITHTIME"):
        assert decode(probe, fn, VAL_DICT_I32, cnt=0, word=0, dict_buf=d)[:3] == (-math.inf, 0, -1)
        assert decode(probe, fn, VAL_DICT_I32, cnt=3, word=0xFFFFFFFF, dict_buf=d)[:3] == (-math.inf, 0, -1)
    assert decode(probe, "FIRSTWITHTIME", VAL_DICT_I32, cnt=3, word=1, dict_buf=d, wt_time=2 ** 40)[:3] == (2.0, 2 ** 40, 1)


def limbs(ks):   # the three limb sums (pb200_moments.h) of grid values k
    n, s1, s2 = len(ks), sum(ks), sum(k * k for k in ks)
    bias = n << 31
    return (s1 - bias, (s2 >> 32) - bias, (s2 & 0xFFFFFFFF) - bias)


def test_moments(probe):
    ks = [1, 2, 3, 4]
    m = limbs(ks)
    assert decode(probe, "VARPOP", cnt=4, mom=m) == (1.25, 4, -1, (10, 30, 0))
    assert decode(probe, "VARPOP", cnt=4, mom=m, mom_e=1)[:2] == (5.0, 4)
    assert decode(probe, "VARSAMP", cnt=4, mom=m)[:2] == (20 / 12, 4)
    assert decode(probe, "STDDEVPOP", cnt=4, mom=m)[:2] == (math.sqrt(1.25), 4)
    big = [2 ** 31 + 5, 3, 2 ** 30]
    s2 = sum(k * k for k in big)
    assert decode(probe, "STDDEVSAMP", cnt=3, mom=limbs(big))[3] == (sum(big), s2 & (2 ** 64 - 1), s2 >> 64)
    assert decode(probe, "VARPOP", cnt=0, mom=limbs([]))[:3] == (-math.inf, 0, -1)
    assert decode(probe, "VARSAMP", cnt=1, mom=limbs([7]))[:3] == (-math.inf, 1, -1)


def test_distinct_sets(probe):
    state = (11, 0, 3, 0, double_bits(11.0), double_bits(11.0 / 3))
    assert decode(probe, "DISTINCTSUM", ds=state)[:3] == (11.0, 3, -1)
    assert decode(probe, "DISTINCTAVG", ds=state)[:3] == (11.0 / 3, 3, -1)
    assert decode(probe, "DISTINCTCOUNTHLL", hll=12345)[:3] == (12345.0, 12345, -1)
    assert decode(probe, "DISTINCTCOUNT", cnt=7)[:3] == (0.0, 0, -1)   # sizes come from the decoded sets


def test_expressions(probe):
    for x in (-2.5, -0.0, 0.0, 1e308, -math.inf, math.inf):
        assert decode(probe, "MIN", VAL_DICT_F64, xkey=compare_key(x))[:3] == (x, 0, -1)
        assert decode(probe, "MAX", VAL_DICT_F64, xkey=compare_key(x))[:3] == (x, 0, -1)
    nan = decode(probe, "MAX", VAL_DICT_F64, xkey=compare_key(math.nan))[0]
    assert math.isnan(nan)
    assert decode(probe, "MIN", VAL_DICT_F64, cnt=0, xkey=2 ** 64 - 1)[:3] == (math.inf, 0, -1)
    assert decode(probe, "MAX", VAL_DICT_F64, cnt=0, xkey=0)[:3] == (-math.inf, 0, -1)
    # an expression sum is an f64 table: the caller's function over a DOUBLE value
    assert decode(probe, "SUM", VAL_DICT_F64, cnt=6, word=double_bits(-12.75))[:3] == (-12.75, 6, -1)
    assert decode(probe, "AVG", VAL_DICT_F64, cnt=0, word=double_bits(0.0))[:3] == (0.0, 0, -1)

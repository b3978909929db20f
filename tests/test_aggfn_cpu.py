"""CPU test: the library's and the package's views of the aggregation functions agree.  The PB200_AGG_* enum of
include/pinot_b200.h, _lib.AGG_CODES and query.AGG_FUNCTIONS name the same codes, and each descriptor of
pinot_b200/csrc/pb200_aggfn.h (through tests/aggfn_probe) has the name, family, argument and dictId use of the package's."""
import ctypes as C
import os
import re
import subprocess

import pytest

from pinot_b200 import _lib
from pinot_b200.query import AGG_FUNCTIONS

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ARGS = {None: 0, "percentile": 1, "log2m": 2, "time": 3}   # pb200_aggfn.h AggArg


def header_codes():
    with open(os.path.join(ROOT, "include", "pinot_b200.h")) as f:
        return {name: int(code) for name, code in re.findall(r"\bPB200_AGG_(\w+) = (\d+)", f.read())}


def test_codes_agree():
    codes = header_codes()
    assert sorted(codes.values()) == list(range(len(codes)))
    assert codes == _lib.AGG_CODES
    assert list(AGG_FUNCTIONS) == sorted(codes, key=codes.get)   # the table is in code order


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("aggfn_probe") / "libaggfn_probe.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", out, os.path.join(HERE, "aggfn_probe", "aggfn_probe.cpp")],
                   check=True)
    lib = C.CDLL(out)
    lib.ap_name.restype = C.c_char_p
    lib.ap_family.restype = C.c_char_p
    return lib


def test_descriptors_agree(probe):
    codes = _lib.AGG_CODES
    for name, code in codes.items():
        f = AGG_FUNCTIONS[name]
        assert probe.ap_known(code)
        assert probe.ap_name(code).decode() == name
        assert probe.ap_family(code).decode() == f.family, name
        assert probe.ap_arg(code) == ARGS[f.arg], name
        assert bool(probe.ap_dict_ids(code)) == f.dict_ids, name
    for code in (-1, len(codes), 99):
        assert not probe.ap_known(code)

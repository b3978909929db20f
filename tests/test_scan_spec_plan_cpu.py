"""CPU tests of the planner's choice of the group-by kernel specialised for the shared-table shape (ScanVariant::spec,
pb200_scan.cuh SPEC): the named shapes of tests/test_scan_plan_cpu.py that take it and those that must not, and, over the
same seeded sweep of random shapes, that the choice never changes any other part of the plan -- geometry, layouts,
carrier and descriptors stay byte-identical (tests/spec_probe/spec_probe.cpp plans each query with and without it)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pinot_b200 import _lib
from test_scan_plan_cpu import (AVG, C3, C5, C6, COUNT, H100, MAX, MIN, Q_MERGE, SUM, UPPER_TENTH, ProbeCol, _random_shape,
                                col, make_query, node)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "spec_probe", "spec_probe.cpp")
    out = os.path.join(HERE, "spec_probe", "libspec_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.probe_spec_route.restype = C.c_int32
    lib.probe_spec_route.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.c_int32,
                                     C.POINTER(_lib.Query), C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                     C.c_int32, C.POINTER(C.c_int64)]
    core = C.CDLL(_lib.LIB_PATH)
    core.pb200_last_error.restype = C.c_char_p
    lib.last_error = lambda: core.pb200_last_error().decode()
    return lib


def route(probe, seg_cols, num_docs, q, knobs=None, carrier=True):
    """Returns (status, spec, spec with the knob off, other plan fields identical, warps, CTAs per SM)."""
    knobs = knobs or {}
    ncols = len(seg_cols[0])
    cols = (ProbeCol * (len(seg_cols) * ncols))()
    for s, cs in enumerate(seg_cols):
        for k, c in enumerate(cs):
            host = c.get("cbuf")
            cols[s * ncols + k] = ProbeCol(c["kind"], c["stored"], c["bits"], c["card"], int(c["native"]), int(c["shared"]),
                                           int(c["inv"]), 0, c["hash"], C.cast(host, C.c_void_p) if host else None,
                                           len(c["host"]) if host else 0)
    names = (C.c_char_p * max(len(knobs), 1))(*[k.encode() for k in knobs])
    values = (C.c_int64 * max(len(knobs), 1))(*knobs.values())
    docs = (C.c_int32 * len(num_docs))(*num_docs)
    out = (C.c_int64 * 6)()
    probe.probe_spec_route(H100[0], H100[1], names, values, len(knobs), C.byref(q), cols, ncols, docs, len(num_docs),
                           int(carrier), out)
    return tuple(out)


def grouped(probe, filters, aggs, group_by=(0,), cols=(C3, C5, C6), nseg=8, rows=100_000_000, flags=Q_MERGE, **kw):
    q, keep = make_query(filters, aggs, group_by=list(group_by), flags=flags)
    r = route(probe, [list(cols)] * nseg, [rows] * nseg, q, **kw)
    assert r[0] == 0, probe.last_error()
    assert r[2] == 0 and r[3] == 1, r   # the knob off never picks it, and the choice changes nothing else
    return r


HEADLINE_AGGS = [(SUM, 1), (COUNT, -1)]


# ---- shapes that take the specialised kernel ----
def test_headline_takes_the_specialised_8_warp_kernel(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS)[1:] == (1, 0, 1, 8, 1)


def test_1000_groups_take_the_specialised_6_warp_kernel(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, cols=(col(1_000, 0, 1), C5, C6))[1:] == (1, 0, 1, 6, 2)


def test_two_range_leaves(probe):
    two = [node("SCAN_RANGE", 2, lo=899_999, hi=1_000_000), node("SCAN_RANGE", 1, lo=10, hi=60_000), node("AND", children=2)]
    assert grouped(probe, two, HEADLINE_AGGS)[1] == 1
    lt_not = [node("SCAN_RANGE", 2, lo=0, hi=500), node("SCAN_NOT_IN", 1, ids=[7]), node("AND", children=2)]
    assert grouped(probe, lt_not, HEADLINE_AGGS)[1] == 1


def test_two_group_by_columns(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, group_by=(0, 3), cols=(col(100, 0, 1), C5, C6, col(50, 3, 2)))[1] == 1


def test_count_only_sum_only_two_sums_and_no_filter(probe):
    assert grouped(probe, UPPER_TENTH, [(COUNT, -1)])[1] == 1
    assert grouped(probe, UPPER_TENTH, [(SUM, 1)])[1] == 1
    assert grouped(probe, [], [(SUM, 1), (COUNT, -1), (AVG, 0)], cols=(col(1_000, 0, 1), C5, C6))[1] == 1


def test_per_segment_results_and_no_carrier(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, flags=0, nseg=17, rows=1_000_000)[1] == 1
    # without the carrier the table has a count array: 12-byte entries, 1 000 groups still fit
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, cols=(col(1_000, 0, 1), C5, C6), carrier=False)[1] == 1


# ---- shapes that must not ----
def test_lut_leaf_takes_the_generic_kernel(probe):
    assert grouped(probe, [node("SCAN_IN", 2, ids=[1, 5, 9])], HEADLINE_AGGS)[1] == 0


def test_doc_mask_leaf_takes_the_generic_kernel(probe):
    cols = (C3, C5, col(1_000, 0, 1, inv=True))
    assert grouped(probe, [node("INV_IN", 2, ids=[3])], HEADLINE_AGGS, cols=cols)[1] == 0


@pytest.mark.parametrize("fn", [MIN, MAX])
def test_min_max_take_the_generic_kernel(probe, fn):
    assert grouped(probe, UPPER_TENTH, [(SUM, 1), (fn, 1)])[1] == 0


def test_16000_groups_global_table_takes_the_generic_kernel(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, cols=(col(16_000, 0, 1), C5, C6))[1] == 0


def test_hash_table_takes_the_generic_kernel(probe):
    big = col(1 << 20, 0, 1)
    assert grouped(probe, [], HEADLINE_AGGS, group_by=(0, 2), cols=(big, C5, big), nseg=2, rows=1_000_000)[1] == 0


def test_or_tree_takes_the_generic_kernel(probe):
    either = [node("SCAN_RANGE", 2, lo=899_999, hi=1_000_000), node("SCAN_RANGE", 1, lo=0, hi=10), node("OR", children=2)]
    assert grouped(probe, either, HEADLINE_AGGS)[1] == 0


def test_three_sums_take_the_generic_kernel(probe):
    small = (col(1_000, 0, 1), C5, C6, col(300, -7, 3))
    r = grouped(probe, UPPER_TENTH, [(SUM, 1), (SUM, 3), (SUM, 2), (COUNT, -1)], cols=small)
    assert r[1] == 0


def test_knob_off_takes_the_generic_kernel(probe):
    assert grouped(probe, UPPER_TENTH, HEADLINE_AGGS, knobs={"spec": 0})[1] == 0


# ---- the choice changes nothing else, over the sweep of tests/test_scan_plan_cpu.py ----
def test_spec_flag_never_changes_any_other_plan_field(probe):
    rng = np.random.default_rng(20261015)
    planned = chosen = 0
    for i in range(3000):
        seg_cols, docs, (q, keep), knobs, shape = _random_shape(rng)
        r = route(probe, seg_cols, docs, q, knobs=knobs, carrier=bool(rng.random() < 0.9))
        if r[0] != 0:
            continue
        planned += 1
        ctx = (i, knobs, shape)
        assert r[2] == 0 and r[3] == 1, ctx
        if r[1]:
            chosen += 1
            assert shape["group_by"] and (r[4], r[5]) in ((8, 1), (6, 2)), ctx
            assert all(f in (COUNT, SUM, AVG) for f, _ in shape["aggs"]), ctx
    assert planned > 1000 and chosen > 0, (planned, chosen)

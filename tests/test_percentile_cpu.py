"""CPU tests of PERCENTILE(col, p): the parser (both syntaxes, bounds, fractional p, ORDER BY resolution), the index rule
against a brute force, the planner (pb200::plan_scan through tests/percentile_probe/percentile_probe.cpp: histogram
sizes, sharing across percentiles of one column, no spreading / shared-memory table / deferral, every refusal with its
code), the value-space reference on oracle-built segments and the CLI's by-value merge of per-segment histograms."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import percentile_oracle
from percentile_ref import group_values, percentile
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import ExecutionStatistics, ResultsBlock
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext, percentile_index, percentile_of_counts

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H100 = (132, 232_448)
SEG, AGG = 20, 6
JUST_BELOW_100 = math.nextafter(100.0, 0.0)
PS = [0.0, 0.1, 1.0, 50.0, 95.0, 99.0, 99.9, 100.0, JUST_BELOW_100]


# ---- parser --------------------------------------------------------------------------------------------------------
def test_parse_both_syntaxes():
    q = sql.parse("SELECT PERCENTILE(a, 95), PERCENTILE99(a), percentile(b, 99.9), PERCENTILE0(c) FROM t GROUP BY g")
    assert [(x.function, x.column, x.arg) for x in q.aggregations] == [
        ("PERCENTILE", "a", 95.0), ("PERCENTILE", "a", 99.0), ("PERCENTILE", "b", 99.9), ("PERCENTILE", "c", 0.0)]
    assert str(q.aggregations[2]) == "percentile(b, 99.9)"
    q = sql.parse("SELECT PERCENTILE100(a), PERCENTILE(a, 0.5) FROM t")
    assert [x.arg for x in q.aggregations] == [100.0, 0.5]
    assert not sql.is_selection("SELECT PERCENTILE95(a) FROM t")
    assert not sql.is_selection("SELECT PERCENTILE(a, 5) FROM t")


@pytest.mark.parametrize("text", ["SELECT PERCENTILE(a, 101) FROM t", "SELECT PERCENTILE(a, -1) FROM t",
                                  "SELECT PERCENTILE101(a) FROM t", "SELECT PERCENTILE(a) FROM t",
                                  "SELECT PERCENTILE(a, 'x') FROM t", "SELECT PERCENTILE(a, b) FROM t",
                                  "SELECT PERCENTILEEST(a, 95) FROM t", "SELECT PERCENTILETDIGEST(a, 95) FROM t",
                                  "SELECT PERCENTILEKLL(a, 95) FROM t", "SELECT SMARTTDIGEST(a, 95) FROM t",
                                  "SELECT MODE(a) FROM t"])
def test_parse_refusals(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


def test_order_by_resolution():
    q = sql.parse("SELECT g, PERCENTILE(a, 50), PERCENTILE(a, 99) FROM t GROUP BY g ORDER BY PERCENTILE(a, 99) DESC LIMIT 10")
    assert sql.resolve_order_by(q) == [("AGG", 1, False)]
    q = sql.parse("SELECT g, PERCENTILE99(a), PERCENTILE(a, 50) FROM t GROUP BY g ORDER BY PERCENTILE(a, 50), PERCENTILE99(a) DESC")
    assert sql.resolve_order_by(q) == [("AGG", 1, True), ("AGG", 0, False)]
    with pytest.raises(sql.SqlError):   # not in the SELECT list
        sql.parse("SELECT g, PERCENTILE(a, 50) FROM t GROUP BY g ORDER BY PERCENTILE(a, 95)")


# ---- index rule ----------------------------------------------------------------------------------------------------
def test_index_rule_brute_force():
    """The reference's rule over n sorted values: p == 100 the largest, else (int)((double)n * p / 100.0), clamped."""
    for n in range(1, 201):
        values = list(range(n))
        for p in PS:
            want = values[-1] if p == 100.0 else values[min(int(float(n) * p / 100.0), n - 1)]
            assert values[percentile_index(n, p)] == want
            assert 0 <= percentile_index(n, p) < n
    # near 100 the double product can round up to n (the reference would index past its list): the clamp keeps the
    # index inside.  With p the double just below 100 that first happens around n = 7.2e14 -- above the 2^32 values one
    # device result can hold, so the device's clamp is exercised here, on the rule both share.
    hit = [n for n in range(720_640_156_790_000, 720_640_156_800_000) if int(float(n) * JUST_BELOW_100 / 100.0) >= n]
    assert hit, "no n reaches the clamp"
    assert all(percentile_index(n, JUST_BELOW_100) == n - 1 for n in hit)
    assert all(int(float(n) * JUST_BELOW_100 / 100.0) < n for n in range(1, 1 << 16))
    assert percentile_of_counts((50.0, {})) == float("-inf")
    assert percentile_of_counts((50.0, {3.0: 2, 1.0: 1, 7.0: 1})) == 3.0


# ---- planner probe -------------------------------------------------------------------------------------------------
FIELDS = ([(n, 1) for n in ("nres", "group_by", "hashed", "groups", "stride", "smem_groups", "num_defer_codes",
                            "num_agg_codes", "hist_total")]
          + [(n, AGG) for n in ("pct_rep", "code_agg", "code_fn", "hist_per_group", "seg0_entries")]
          + [("hist_entries", SEG * AGG)])


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32),
                ("dict_native", C.c_int32), ("dict_hash", C.c_int32)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "percentile_probe", "percentile_probe.cpp")
    out = os.path.join(HERE, "percentile_probe", "libpercentile_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.pct_probe_plan_size.restype = C.c_int64
    assert lib.pct_probe_plan_size() == C.sizeof(ProbePlan)
    lib.pct_probe_index.restype = C.c_int64
    lib.pct_probe_index.argtypes = [C.c_int64, C.c_double]
    lib.pct_probe_plan_scan.restype = C.c_int32
    lib.pct_probe_plan_scan.argtypes = [C.c_int32, C.c_int32, C.POINTER(_lib.Query), C.POINTER(C.c_double),
                                        C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int64,
                                        C.POINTER(ProbePlan)]
    return lib


D, R, S = _lib.FWD_DICT_FIXEDBIT, _lib.FWD_RAW_FIXEDBYTE, _lib.STRING
P, SUM, COUNT, MAX, DC = 6, 1, 0, 3, 5
# columns: 0 INT card 10, 1 LONG card 1000, 2 DOUBLE card 2^20, 3 STRING card 100, 4 raw INT streamed, 5 INT card 5000,
#          6 FLOAT card 3 (other dictionary hash), 7 INT card 2^24
COLS = [(D, _lib.INT, 4, 10, 1, 1), (D, _lib.LONG, 10, 1000, 1, 2), (D, _lib.DOUBLE, 20, 1 << 20, 1, 3), (D, S, 7, 100, 0, 4),
        (R, _lib.INT, 32, 0, 0, 0), (D, _lib.INT, 13, 5000, 1, 6), (D, _lib.FLOAT, 2, 3, 1, 7), (D, _lib.INT, 24, 1 << 24, 1, 8)]


def plan(probe, aggs, args, group_by=(), num_docs=(100_000,), merge=False, cols=None, dense_max=0, flags=0):
    n = len(num_docs)
    pc = (ProbeCol * (n * len(COLS)))()
    for s in range(n):
        for k, c in enumerate(cols[s] if cols is not None else COLS):
            pc[s * len(COLS) + k] = ProbeCol(*c)
    ag = (_lib.Agg * len(aggs))(*[_lib.Agg(f, c) for f, c in aggs])
    gb = (C.c_int32 * max(1, len(group_by)))(*group_by)
    q = _lib.Query(0, len(group_by), len(aggs), 100_000, 10_000, flags | (_lib_merge() if merge else 0), None, gb, ag, 0, 0, 0)
    a = None if args is None else (C.c_double * len(args))(*args)
    out = ProbePlan()
    rc = probe.pct_probe_plan_scan(H100[0], H100[1], C.byref(q), a, pc, len(COLS), (C.c_int32 * n)(*num_docs), n, dense_max,
                                   C.byref(out))
    return rc, out


def _lib_merge():
    return 2   # PB200_Q_MERGE_SEGMENTS


def test_device_index_rule(probe):
    """The C++ copy of the rule the finalize kernel runs (pb200_desc.h), on the same n as the Python one, clamp included."""
    for n in range(1, 201):
        for p in PS:
            assert probe.pct_probe_index(n, p) == percentile_index(n, p)
    hit = [n for n in range(720_640_156_790_000, 720_640_156_800_000) if int(float(n) * JUST_BELOW_100 / 100.0) >= n]
    assert hit
    for n in hit[:50] + [720_640_156_790_000, 720_640_156_799_999]:
        assert probe.pct_probe_index(n, JUST_BELOW_100) == percentile_index(n, JUST_BELOW_100)
    assert all(probe.pct_probe_index(n, JUST_BELOW_100) == n - 1 for n in hit[:50])


def test_probe_aggregation_only_sizes_and_sharing(probe):
    rc, o = plan(probe, [(P, 1), (SUM, 0), (P, 1), (P, 2), (P, 1)], [50.0, 0.0, 95.0, 99.9, 100.0], num_docs=(1000, 2000))
    assert rc == 0 and o.nres == 2 and not o.group_by
    assert list(o.pct_rep[:5]) == [0, -1, 0, 3, 0]
    # one histogram per result and column: 2^bits entries
    assert [o.hist_entries[r * AGG + a] for r in range(2) for a in range(5)] == [1 << 10, 0, 0, 1 << 20, 0] * 2
    assert o.hist_total == 2 * ((1 << 10) + (1 << 20))
    # one agg code per histogram: the SUM and the owners 0 and 3
    codes = sorted(zip(o.code_agg[:o.num_agg_codes], o.code_fn[:o.num_agg_codes]))
    assert codes == [(0, P), (1, SUM), (3, P)]
    rc, o = plan(probe, [(P, 1)], [50.0], num_docs=(1000, 2000), merge=True)
    assert rc == 0 and o.nres == 1 and o.hist_entries[0] == 1 << 10
    # few dictIds: the dense route adds equal ids of a warp once (flag in the segment descriptor); many: one add per row
    rc, o = plan(probe, [(P, 0), (P, 1), (P, 6)], [50.0, 50.0, 50.0])
    assert rc == 0 and list(o.seg0_entries[:3]) == [1, 0, 1]


def test_probe_group_by_layout(probe):
    rc, o = plan(probe, [(COUNT, -1), (P, 5), (P, 5), (P, 1)], [0.0, 50.0, 99.0, 1.0], group_by=[0])
    assert rc == 0 and o.group_by and not o.hashed
    assert o.groups == 10 and o.stride == 1          # no spreading
    assert o.smem_groups == 0 and o.num_defer_codes == 0   # no shared-memory table, nothing deferred
    assert list(o.hist_per_group[:4]) == [0, 5000, 0, 1000]
    assert o.seg0_entries[1] == 5000 and o.seg0_entries[3] == 1000
    assert o.hist_total == 10 * 5000 + 10 * 1000
    assert sorted(o.code_agg[:o.num_agg_codes]) == [1, 3]
    # the same GROUP BY without PERCENTILE does spread its table and uses the shared-memory table
    rc, o2 = plan(probe, [(COUNT, -1), (SUM, 0)], [0.0, 0.0], group_by=[0])
    assert rc == 0 and (o2.stride > 1 or o2.smem_groups > 0)
    # hash table: slots x cardinality
    rc, o = plan(probe, [(P, 0), (MAX, 1)], [95.0, 0.0], group_by=[5], dense_max=1)
    assert rc == 0 and o.hashed and o.hist_per_group[0] == 10 and o.hist_total == o.groups * 10


def test_probe_refusals(probe):
    E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
    assert plan(probe, [(P, 1)], None)[0] == E_INVALID                 # pb200_execute / _ordered: no percentile
    for bad in (-0.5, 100.5, float("nan"), float("inf")):
        assert plan(probe, [(P, 1)], [bad])[0] == E_INVALID
    assert plan(probe, [(P, 1)], [0.0])[0] == 0 and plan(probe, [(P, 1)], [100.0])[0] == 0
    assert plan(probe, [(P, 3)], [50.0])[0] == E_UNSUPPORTED           # STRING
    assert plan(probe, [(P, 4)], [50.0])[0] == E_UNSUPPORTED           # raw column streamed as 32-bit values
    # deferred finalize (cross-GPU reduce of the tables)
    assert plan(probe, [(P, 1)], [50.0], group_by=[0], num_docs=(1000, 1000), merge=True, flags=4)[0] == E_UNSUPPORTED
    # histogram budget: 2^24 entries per result, 2^28 per call
    assert plan(probe, [(P, 7)], [50.0], num_docs=(1000,) * 16)[0] == 0
    assert plan(probe, [(P, 7)], [50.0], num_docs=(1000,) * 17)[0] == E_UNSUPPORTED
    assert plan(probe, [(P, 7)], [50.0], num_docs=(1000,) * 17, merge=True)[0] == 0
    assert plan(probe, [(P, 2)], [50.0], group_by=[5])[0] == E_UNSUPPORTED   # 5000 groups x 2^20 dictIds
    # u32 bins: a result over 2^32 docs
    big = (2_000_000_000, 2_000_000_000, 300_000_000)
    assert plan(probe, [(P, 0)], [50.0], num_docs=big, merge=True)[0] == E_UNSUPPORTED
    assert plan(probe, [(P, 0)], [50.0], num_docs=big)[0] == 0
    # merged: the column's dictionary must be the same in every segment
    other = [COLS, COLS[:1] + [(D, _lib.LONG, 10, 1000, 1, 99)] + COLS[2:]]
    assert plan(probe, [(P, 1)], [50.0], num_docs=(1000, 1000), merge=True, cols=other)[0] == E_UNSUPPORTED
    assert plan(probe, [(P, 1)], [50.0], num_docs=(1000, 1000), cols=other)[0] == 0


# ---- the oracle's PERCENTILE against the value-space reference on oracle-built segments ---------------------------
def test_oracle_percentile_against_reference(oracle):
    rng = np.random.default_rng(7)
    segs = []
    for k, n in enumerate((1, 777, 5000)):
        f = (rng.integers(-40, 40, size=n) / 4.0).astype(np.float32)
        f[rng.integers(0, n, size=max(1, n // 100))] = np.inf
        cols = {"i": rng.integers(-50, 50, size=n).astype(np.int32), "g": rng.integers(0, 4, size=n).astype(np.int32),
                "l": rng.choice(np.array([-(1 << 63), (1 << 53) + 1, 1 << 53, 7, (1 << 63) - 1], dtype=np.int64), size=n),
                "f": f, "d": rng.integers(-90, 90, size=n) / 7.0,
                "r": rng.integers(-9, 9, size=n).astype(np.int32) * 1000, "inv": rng.integers(0, 20, size=n).astype(np.int32)}
        segs.append(oracle.build_segment(f"pct_oracle_{k}", cols, inverted=["inv"], raw=["r"]))
    filters = [None, Predicate("RANGE", "i", [], -10, 30, True, False), Predicate("EQ", "inv", [3]),
               Filter("OR", [Predicate("IN", "g", [1, 2]), Filter("NOT", [Predicate("RANGE", "d", [], 0.0, None, True, True)])]),
               Predicate("RANGE", "r", [], 0, None, True, True), Predicate("EQ", "i", [1000])]
    for flt in filters:
        for gb in ([], ["g"]):
            for col in ("i", "l", "f", "d", "r"):
                for group in ([s] for s in segs):
                    got = percentile_oracle.percentiles(oracle, group, flt, gb, col, PS)
                    ref = group_values(oracle, group, flt, gb, col)
                    assert set(got) == set(ref), (flt, gb, col)
                    for key, vals in got.items():
                        want = [percentile(ref[key], p) for p in PS]
                        assert np.array_equal(np.array(vals), np.array(want)), (flt, gb, col, key)
                got = percentile_oracle.percentiles(oracle, segs, flt, gb, "l", [50.0])   # across segments, by value
                ref = group_values(oracle, segs, flt, gb, "l")
                assert {k: v[0] for k, v in got.items()} == {k: percentile(v, 50.0) for k, v in ref.items()}


# ---- CLI by-value merge --------------------------------------------------------------------------------------------
class _Seg:
    def __init__(self, dicts):
        self.dicts = dicts

    def dictionary_value(self, column, dict_id):
        return self.dicts[column][dict_id]


def _block(keys, hists, doubles):
    rows = len(keys) if keys is not None else 1
    b = ResultsBlock(-1 if keys is None else rows, "ARRAY", False, ExecutionStatistics(0, 0, 0, 0),
                     np.zeros((0 if keys is None else rows, 1), dtype=np.int32) if keys is None else np.array(keys, dtype=np.int32).reshape(rows, 1),
                     [np.array(doubles, dtype=np.float64)], [np.zeros(rows, dtype=np.int64)], [np.full(rows, -1, dtype=np.int32)])
    b.histograms = {(0, r): (np.array(h[0], dtype=np.int32), np.array(h[1], dtype=np.int64)) for r, h in enumerate(hists)}
    return b


def test_cli_merge_by_value():
    q = QueryContext(aggregations=[Aggregation("PERCENTILE", "v", arg=50.0)], group_by=["k"], limit=10)
    # two segments with different dictionaries: values 1, 3, 5 and 2, 3, 9
    s0 = _Seg({"k": ["x", "y"], "v": [1, 3, 5]})
    s1 = _Seg({"k": ["y", "z"], "v": [2, 3, 9]})
    b0 = _block([0, 1], [([0, 2], [3, 1]), ([1], [2])], [1.0, 3.0])
    b1 = _block([0, 1], [([0, 1, 2], [1, 1, 1]), ([2], [1])], [3.0, 9.0])
    rows = cli.final_rows(q, cli.merge_blocks(q, [s0, s1], [b0, b1]))
    # x: {1 x3, 5}: n 4, index 2 -> 1;  y: {3 x3, 2, 9}: sorted 2 3 3 3 9, index 2 -> 3;  z: {9}
    assert rows == [["x", 1.0], ["y", 3.0], ["z", 9.0]]
    q = QueryContext(aggregations=[Aggregation("PERCENTILE", "v", arg=100.0)], limit=10)
    rows = cli.final_rows(q, cli.merge_blocks(q, [s0, s1], [_block(None, [([0, 2], [1, 1])], [5.0]), _block(None, [([], [])], [float("-inf")])]))
    assert rows == [[5.0]]
    # ORDER BY PERCENTILE DESC over merged values
    q = QueryContext(aggregations=[Aggregation("PERCENTILE", "v", arg=50.0)], group_by=["k"], limit=2,
                     order_by=[("percentile(v,50.0)", False)])
    rows = cli.final_rows(q, cli.merge_blocks(q, [s0, s1], [b0, b1]))
    assert rows == [["z", 9.0], ["y", 3.0]]


def test_distributed_refuses_percentile():
    from pinot_b200 import distributed
    q = QueryContext(aggregations=[Aggregation("PERCENTILE", "v", arg=50.0)], limit=10)

    class _Dist:
        def get_world_size(self):
            return 2

    with pytest.raises(_lib.UnsupportedQueryError):
        distributed.execute_and_combine(object(), [], q, _Dist())

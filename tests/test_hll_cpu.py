"""CPU tests of DISTINCTCOUNTHLL (DESIGN.md section 3.17): the parser (spellings, canonical text, ORDER BY and HAVING
naming, parse errors), the ABI code, the hash / offer / estimate of pinot_b200/csrc/pb200_hll.h (the code the device
runs, through tests/hll_probe) and query.hll_final against the independent restatement tests/hll_ref.py, the
linear-counting margin, the planner's bitset sharing (through tests/distinct_sum_probe), the CLI merge and the cross-GPU
host route under gloo."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import hll_ref
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import ExecutionStatistics, ResultsBlock
from pinot_b200.query import HllSet, hll_final

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HLL, DCOUNT, DSUM, SUM = 15, 5, 13, 1
LONG_MAX = (1 << 63) - 1


# ---- parser --------------------------------------------------------------------------------------------------------
def test_parse_and_canonical_text():
    q = sql.parse("SELECT DISTINCTCOUNTHLL(a), distinctcounthll(a, 12), DistinctCountHLL(b, 8), DISTINCTCOUNTHLL(a, 0) FROM t")
    assert [(x.function, x.column, x.arg) for x in q.aggregations] == [
        ("DISTINCTCOUNTHLL", "a", 8), ("DISTINCTCOUNTHLL", "a", 12), ("DISTINCTCOUNTHLL", "b", 8), ("DISTINCTCOUNTHLL", "a", 0)]
    assert [str(x) for x in q.aggregations] == ["distinctcounthll(a)", "distinctcounthll(a, 12)", "distinctcounthll(b)",
                                                "distinctcounthll(a, 0)"]


def test_order_by_and_having_naming():
    q = sql.parse("SELECT g, DISTINCTCOUNTHLL(m), DISTINCTCOUNTHLL(m, 12) FROM t GROUP BY g "
                  "HAVING DISTINCTCOUNTHLL(m, 12) > 3 AND distinctcounthll(m) < 100 "
                  "ORDER BY DISTINCTCOUNTHLL(m, 12) DESC, distinctcounthll(m) LIMIT 5")
    assert sql.resolve_order_by(q) == [("AGG", 1, False), ("AGG", 0, True)]
    assert [n[1] for n in sql.resolve_having(q) if n[0] == "RANGE"] == [1, 0]
    q = sql.parse("SELECT g, COUNT(*) FROM t GROUP BY g HAVING DISTINCTCOUNTHLL(m, 10) >= 1")   # named only in HAVING
    assert q.aggregations[1].function == "DISTINCTCOUNTHLL" and q.aggregations[1].arg == 10 and q.aggregations[1].hidden


@pytest.mark.parametrize("text", ["SELECT DISTINCTCOUNTHLL(a, 31) FROM t", "SELECT DISTINCTCOUNTHLL(a, -1) FROM t",
                                  "SELECT DISTINCTCOUNTHLL(a, 8.5) FROM t", "SELECT DISTINCTCOUNTHLL(a, 'x') FROM t",
                                  "SELECT DISTINCTCOUNTHLL(*) FROM t", "SELECT DISTINCTCOUNTHLL(a, 8, 9) FROM t",
                                  "SELECT g, COUNT(*) FROM t GROUP BY g ORDER BY DISTINCTCOUNTHLL(a, 40)"])
def test_parse_errors(text):
    with pytest.raises(sql.SqlError):
        sql.parse(text)


def test_abi_code_matches_the_header():
    import re
    text = open(os.path.join(ROOT, "include", "pinot_b200.h")).read()
    assert re.search(r"PB200_AGG_DISTINCTCOUNTHLL = 15\b", text)
    assert _lib.AGG_CODES["DISTINCTCOUNTHLL"] == 15
    assert re.search(r"#define PB200_ABI_VERSION 3\b", text)


def test_headers_compile_as_c99(tmp_path):
    src = tmp_path / "c99.c"
    src.write_text('#include "pinot_b200.h"\n#include "pinot_b200_host.h"\nint main(void) { return PB200_AGG_DISTINCTCOUNTHLL - 15; }\n')
    subprocess.run(["gcc", "-std=c99", "-pedantic", "-Werror", "-fsyntax-only", f"-I{os.path.join(ROOT, 'include')}", str(src)], check=True)


# ---- probe of pb200_hll.h ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe():
    src = os.path.join(HERE, "hll_probe", "hll_probe.cpp")
    out = os.path.join(HERE, "hll_probe", "libhll_probe.so")
    header = os.path.join(ROOT, "pinot_b200", "csrc", "pb200_hll.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(header)):
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.hp_hash_long.restype = C.c_uint32
    lib.hp_hash_long.argtypes = [C.c_uint64]
    lib.hp_hash_bytes.restype = C.c_uint32
    lib.hp_hash_bytes.argtypes = [C.c_char_p, C.c_int32, C.c_uint32]
    lib.hp_hash_value.restype = C.c_uint32
    lib.hp_hash_value.argtypes = [C.c_int32, C.c_uint64]
    lib.hp_utf8_valid.restype = C.c_int32
    lib.hp_utf8_valid.argtypes = [C.c_char_p, C.c_int32]
    lib.hp_alpha_mm.restype = C.c_double
    lib.hp_alpha_mm.argtypes = [C.c_int32]
    lib.hp_linear_table.argtypes = [C.c_int32, C.POINTER(C.c_longlong)]
    lib.hp_estimate.restype = C.c_int64
    lib.hp_estimate.argtypes = [C.POINTER(C.c_uint32), C.c_int64, C.c_int32]
    return lib


def u32(x):
    return x & 0xFFFFFFFF


LONGS = [0, 1, -1, (1 << 31) - 1, -(1 << 31), (1 << 63) - 1, -(1 << 63) + 1, -(1 << 63), 1 << 32, 123456789012345]
FLOATS = [0.0, -0.0, math.nan, math.inf, -math.inf, 1e-45, -1e-45, 1.17549435e-38, 3.4028235e38, 1.5, -2.25]
DOUBLES = [0.0, -0.0, math.nan, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 0.1]


def raw_bits(v, t):
    if t == _lib.FLOAT:
        return struct.unpack("<I", struct.pack("<f", v))[0]
    if t == _lib.DOUBLE:
        return struct.unpack("<Q", struct.pack("<d", v))[0]
    return v & (0xFFFFFFFF if t == _lib.INT else 0xFFFFFFFFFFFFFFFF)


def test_hash_of_numbers(probe):
    for v in LONGS:
        assert probe.hp_hash_long(v & 0xFFFFFFFFFFFFFFFF) == u32(hll_ref.hash_long(v)), v
        assert probe.hp_hash_value(_lib.LONG, raw_bits(v, _lib.LONG)) == u32(hll_ref.hash_value(v, "LONG")), v
    for v in [x for x in LONGS if -(1 << 31) <= x < (1 << 31)]:   # INT: sign-extended, the same as the LONG of its value
        assert probe.hp_hash_value(_lib.INT, raw_bits(v, _lib.INT)) == u32(hll_ref.hash_value(v, "INT")), v
    for v in FLOATS:
        assert probe.hp_hash_value(_lib.FLOAT, raw_bits(v, _lib.FLOAT)) == u32(hll_ref.hash_value(v, "FLOAT")), v
    for v in DOUBLES:
        assert probe.hp_hash_value(_lib.DOUBLE, raw_bits(v, _lib.DOUBLE)) == u32(hll_ref.hash_value(v, "DOUBLE")), v
    # -0.0 and 0.0 are two members with two hashes
    assert probe.hp_hash_value(_lib.DOUBLE, raw_bits(-0.0, _lib.DOUBLE)) != probe.hp_hash_value(_lib.DOUBLE, 0)


def test_hash_of_bytes_every_tail_length(probe):
    rng = np.random.default_rng(3)
    for n in range(0, 10):
        for _ in range(20):
            b = bytes(rng.integers(0, 256, size=n, dtype=np.uint8))
            assert probe.hp_hash_bytes(b, n, 0xFFFFFFFF) == u32(hll_ref.hash_bytes(b)), b
    for b in [b"\x80", b"\xff\xfe", b"ab\xc3", b"abcd\xe2\x82\xac", "é€😀".encode()]:   # tail bytes >= 0x80: sign-extended
        assert probe.hp_hash_bytes(b, len(b), 0xFFFFFFFF) == u32(hll_ref.hash_bytes(b)), b


def test_utf8_validity(probe):
    good = ["", "abc", "é", "€", "😀", "߿", "￿", "\U0010ffff", "퟿"]
    bad = [b"\x80", b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xed\xa0\x80", b"\xf0\x80\x80\xaf", b"\xf4\x90\x80\x80",
           b"\xf5\x80\x80\x80", b"\xe2\x82", b"ab\xff", b"\xfe"]
    for s in good:
        b = s.encode("utf-8")
        assert probe.hp_utf8_valid(b, len(b)) == 1, s
    for b in bad:
        assert probe.hp_utf8_valid(b, len(b)) == 0, b
        with pytest.raises(UnicodeDecodeError):   # what Java would replace by U+FFFD
            b.decode("utf-8")


def probe_estimate(probe, hashes, p):
    arr = np.ascontiguousarray(np.asarray([u32(h) for h in hashes], dtype=np.uint32))
    return probe.hp_estimate(arr.ctypes.data_as(C.POINTER(C.c_uint32)), len(arr), p)


@pytest.mark.parametrize("p", range(4, 13))
def test_estimate_every_log2m(probe, p):
    rng = np.random.default_rng(100 + p)
    m = 1 << p
    sizes = [0, 1, 2, m // 4, m, 2 * m, 3 * m, 5 * m, 20 * m]   # both sides of estimate <= 2.5 m
    for n in sizes:
        vals = [int(x) for x in rng.choice(1 << 40, size=n, replace=False)] if n else []
        hashes = [hll_ref.hash_value(v, "LONG") for v in vals]
        want = hll_ref.cardinality(hll_ref.registers(hashes, p), p)
        assert probe_estimate(probe, hashes, p) == want, (p, n)
        assert hll_final(vals, p) == want, (p, n)
    assert probe.hp_alpha_mm(p) == hll_ref.alpha_mm(p, m)


def test_small_range_without_zero_registers(probe):
    """p = 4: sixteen hashes putting rank 1 into every register -- the estimate 0.673 * 256 / 8 is below 2.5 m, and
    m * log(m / 0) is +inf: Math.round gives Long.MAX_VALUE."""
    hashes = [(j << 28) | (1 << 27) for j in range(16)]
    reg = hll_ref.registers(hashes, 4)
    assert reg == [1] * 16
    assert hll_ref.cardinality(reg, 4) == LONG_MAX
    assert probe_estimate(probe, hashes, 4) == LONG_MAX


@pytest.mark.parametrize("p", range(4, 13))
def test_linear_counting_margin(probe, p):
    """Every linear-counting result m * log(m / z) is at least 1e-6 away from a rounding tie, so a 1-ulp difference
    between Java's Math.log and the C library's log cannot change the long; and the host table is that rounding."""
    m = 1 << p
    table = (C.c_longlong * (m + 1))()
    probe.hp_linear_table(p, table)
    assert table[0] == LONG_MAX
    for z in range(1, m + 1):
        x = m * math.log(m / z)
        frac = x - math.floor(x)
        assert abs(frac - 0.5) >= 1e-6, (p, z, x)
        assert table[z] == hll_ref.java_round(x), (p, z)


def test_hll_final_against_reference_every_type():
    rng = np.random.default_rng(11)
    ints = [int(x) for x in rng.integers(-(1 << 31), 1 << 31, size=3000)] + [-(1 << 31), (1 << 31) - 1]
    longs = [int(x) for x in rng.integers(-(1 << 62), 1 << 62, size=3000)] + [LONG_MAX, -LONG_MAX]
    floats = [float(np.float32(x)) for x in rng.normal(size=2000)] + [0.0, -0.0, math.nan, math.inf, -math.inf, 1e-45]
    doubles = list(rng.normal(size=2000)) + [0.0, -0.0, math.nan, math.inf, 5e-324]
    strings = ["", "a", "é", "日本語", "😀x", "abcdefghi"] + [f"user{k}" for k in range(2000)]
    for p in (4, 8, 12):
        assert hll_final(ints, p, "INT") == hll_ref.hll(ints, p, "INT")
        assert hll_final(longs, p) == hll_ref.hll(longs, p, "LONG")
        assert hll_final(floats, p, "FLOAT") == hll_ref.hll(floats, p, "FLOAT")
        assert hll_final(doubles, p) == hll_ref.hll(doubles, p, "DOUBLE")
        assert hll_final(strings, p) == hll_ref.hll(strings, p, "STRING")
    assert hll_final([], 8) == 0


def test_reference_relative_error_is_plausible():
    """A sanity check of the restatement (not a parity proof): over random sets of 10^2 .. 10^6 members the relative
    error stays within a generous multiple of the standard error 1.04 / sqrt(m)."""
    rng = np.random.default_rng(7)
    for p in (8, 12):
        se = 1.04 / math.sqrt(1 << p)
        for n in (100, 1000, 10_000, 100_000, 1_000_000):
            vals = rng.choice(1 << 40, size=n, replace=False)
            est = hll_ref.cardinality(hll_ref.registers([hll_ref.hash_long(int(v)) for v in vals], p), p)
            assert abs(est - n) / n < 5 * se, (p, n, est)


# ---- planner (pb200::plan_scan through tests/distinct_sum_probe) ------------------------------------------------------
@pytest.fixture(scope="module")
def plan_probe():
    """The planner probe of the DISTINCTSUM tests (tests/distinct_sum_probe), built the same way."""
    import test_distinct_sum_cpu as ds
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
    lib.ds_probe_plan_scan.restype = C.c_int32
    lib.ds_probe_plan_scan.argtypes = [C.POINTER(_lib.Query), C.POINTER(ds.ProbeCol), C.c_int32, C.POINTER(C.c_int32),
                                       C.c_int32, C.POINTER(ds.ProbePlan)]
    return ds, lib


def _plan(ds, lib, aggs, cols, group_by=()):
    return ds.plan(lib, aggs, cols, group_by=group_by)


def test_plan_sharing(plan_probe):
    ds, lib = plan_probe
    cols = [ds.dcol(_lib.INT, range(200)), ds.dcol(_lib.INT, range(10), 4)]
    # DISTINCTCOUNT, two HLLs and a DISTINCTSUM of one column: one bitset, one agg code
    rc, p = _plan(ds, lib, [(DCOUNT, 0), (HLL, 0), (HLL, 0), (DSUM, 0)], cols)
    assert rc == 0 and list(p.ds_rep[:4]) == [-1, 0, 0, 0] and list(p.slot[1:4]) == [-1, -1, -1]
    assert set(zip(p.code_fn[:p.num_agg_codes], p.code_agg[:p.num_agg_codes])) == {(DCOUNT, 0)}
    # an HLL first owns the set and carries the DISTINCTCOUNT code
    rc, p = _plan(ds, lib, [(HLL, 0), (DCOUNT, 0), (SUM, 0)], cols, group_by=[1])
    assert rc == 0 and list(p.ds_rep[:3]) == [0, -1, -1]
    assert set(zip(p.code_fn[:p.num_agg_codes], p.code_agg[:p.num_agg_codes])) == {(DCOUNT, 0), (DCOUNT, 1), (SUM, 2)}


def test_plan_refusals(plan_probe):
    ds, lib = plan_probe
    assert _plan(ds, lib, [(HLL, 0)], [(_lib.INT, 32, 0, 1, 1, None)])[0] == _lib.E_UNSUPPORTED   # raw INT
    cols = [ds.dcol(_lib.INT, range(1 << 16), 16), ds.dcol(_lib.INT, range(1 << 15), 15)]
    assert _plan(ds, lib, [(HLL, 0)], cols, group_by=[0, 1])[0] == _lib.E_UNSUPPORTED   # the bitset budget


# ---- CLI merge -----------------------------------------------------------------------------------------------------
class _Seg:
    def __init__(self, dicts, types):
        self.dicts, self.types = dicts, types

    def dictionary_value(self, column, d):
        return self.dicts[column][d]

    def column_info(self, column):
        return {"data_type": self.types[column]}


def _block(groups, keys, longs, distinct):
    n = len(keys)
    z = np.zeros(max(n, 1))
    return ResultsBlock(groups, "ARRAY", False, ExecutionStatistics(0, 0, 0, 0), np.asarray(keys, dtype=np.int32).reshape(n, -1),
                        [z] * len(longs), longs, [np.full(max(n, 1), -1, dtype=np.int32)] * len(longs), distinct, 0.0, "GROUP_BY")


def test_cli_merges_sets_then_estimates():
    q = sql.parse("SELECT g, DISTINCTCOUNTHLL(m), DISTINCTCOUNTHLL(m, 4) FROM t GROUP BY g "
                  "ORDER BY DISTINCTCOUNTHLL(m) DESC LIMIT 10")
    x1 = [float(np.float32(v)) for v in np.linspace(-3, 3, 300)]
    x2 = [float(np.float32(v)) for v in np.linspace(0, 9, 500)] + [-0.0, math.nan]
    s1 = _Seg({"g": ["x", "y"], "m": sorted(set(x1)) + [1e30]}, {"g": _lib.STRING, "m": _lib.FLOAT})
    s2 = _Seg({"g": ["x"], "m": x2}, {"g": _lib.STRING, "m": _lib.FLOAT})
    n1, n2 = len(s1.dicts["m"]), len(x2)
    z = np.zeros(2, dtype=np.int64)
    b1 = _block(2, [[0], [1]], [z, z], {(a, 0): list(range(n1 - 1)) for a in (0, 1)} | {(a, 1): [n1 - 1] for a in (0, 1)})
    b2 = _block(1, [[0]], [z[:1], z[:1]], {(a, 0): list(range(n2)) for a in (0, 1)})
    rows = cli.final_rows(q, cli.merge_blocks(q, [s1, s2], [b1, b2]))
    members = set(map(struct.Struct("<f").pack, x1 + x2))   # by bits: -0.0 apart, NaN once
    vals = [struct.unpack("<f", b)[0] for b in members]
    assert rows[0] == ["x", hll_ref.hll(vals, 8, "FLOAT"), hll_ref.hll(vals, 4, "FLOAT")]
    assert rows[1] == ["y", hll_ref.hll([1e30], 8, "FLOAT"), hll_ref.hll([1e30], 4, "FLOAT")]


def test_hll_set_keeps_its_type_through_unions():
    s = HllSet([1.5], _lib.FLOAT)
    s |= {2.5}
    assert s.data_type == "FLOAT" and hll_final(s, 8, s.data_type) == hll_ref.hll([1.5, 2.5], 8, "FLOAT")


# ---- the cross-GPU host route under gloo ------------------------------------------------------------------------------
class _SetSegment:
    def __init__(self, domain, rows):
        self.domain, self.rows = domain, rows

    def dictionary_value(self, column, d):
        return self.domain[column][d]

    def column_info(self, column):
        return {"data_type": _lib.STRING if column == "s" else _lib.LONG}


class _SetPlanMaker:
    """Stands in for the device: the merged block of a rank's segments, sets of domain ids per group (sets=True: the
    DISTINCTCOUNTHLL sets are read)."""
    ctx = None

    def execute_segments(self, segments, query, merge=True, ordered=False, sets=False):
        assert sets
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
        z = np.zeros(max(n, 1))
        distinct = {(a, g): sorted(groups[k][a]) for g, k in enumerate(keys) for a in range(len(query.aggregations))}
        stats = ExecutionStatistics(0, 0, 0, 0)
        return [ResultsBlock(n if gb else -1, "ARRAY", False, stats,
                             np.asarray(keys, dtype=np.int32).reshape(len(keys), len(gb)) if gb else np.zeros((0, 0), dtype=np.int32),
                             [z.copy() for _ in query.aggregations], [z.astype(np.int64) for _ in query.aggregations],
                             [np.full(max(n, 1), -1, dtype=np.int32) for _ in query.aggregations], distinct, 0.0, "GROUP_BY")]


DIST_QUERIES = ["SELECT g, DISTINCTCOUNTHLL(l), DISTINCTCOUNTHLL(s, 6) FROM t GROUP BY g ORDER BY DISTINCTCOUNTHLL(l) DESC LIMIT 3",
                "SELECT DISTINCTCOUNTHLL(l, 12), DISTINCTCOUNTHLL(s) FROM t"]


def _domain():
    rng = np.random.default_rng(5)
    return {"g": list(range(8)), "l": sorted({int(x) for x in rng.integers(-(1 << 62), 1 << 62, size=3000)}),
            "s": sorted({f"k{int(x)}é" for x in rng.integers(0, 5000, size=2000)})}


def _rank_rows(rank, dom):
    rng = np.random.default_rng(70 + rank)
    return [{"g": int(rng.integers(0, 8)), "l": int(rng.integers(0, len(dom["l"]))), "s": int(rng.integers(0, len(dom["s"])))}
            for _ in range(2000)]


def _hll_worker(rank, world, port, out_dir):
    import pickle
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pinot_b200.distributed import execute_and_combine
    dom = _domain()
    segs = [_SetSegment(dom, _rank_rows(rank, dom))]
    out = {}
    for text in DIST_QUERIES:
        got = execute_and_combine(_SetPlanMaker(), segs, sql.parse(text), dist, dst=0)
        if rank == 0:
            rows = 1 if got.num_groups < 0 else got.num_groups
            out[text] = [(tuple(int(x) for x in got.keys[g]) if got.num_groups >= 0 else (),
                          [int(got.longs[a][g]) for a in range(len(got.longs))], [float(got.doubles[a][g]) for a in range(len(got.doubles))])
                         for g in range(rows)]
    if rank == 0:
        pickle.dump(out, open(os.path.join(out_dir, "hll.pkl"), "wb"))
    dist.destroy_process_group()


def test_distributed_set_route_world_size_2(tmp_path):
    import pickle
    import torch.multiprocessing as mp
    world, port = 2, 35100 + (os.getpid() % 1500)
    mp.spawn(_hll_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    got = pickle.load(open(tmp_path / "hll.pkl", "rb"))
    dom = _domain()
    rows = [r for k in range(world) for r in _rank_rows(k, dom)]
    per_group = {}
    for r in rows:
        e = per_group.setdefault(r["g"], (set(), set()))
        e[0].add(dom["l"][r["l"]])
        e[1].add(dom["s"][r["s"]])
    est = {g: (hll_ref.hll(v[0], 8, "LONG"), hll_ref.hll(v[1], 6, "STRING")) for g, v in per_group.items()}
    ranked = sorted(est, key=lambda g: (-est[g][0], g))
    assert [(k, l) for k, l, _ in got[DIST_QUERIES[0]]] == [((g,), list(est[g])) for g in ranked]
    assert all(d == [float(x) for x in l] for _, l, d in got[DIST_QUERIES[0]])
    every_l = {dom["l"][r["l"]] for r in rows}
    every_s = {dom["s"][r["s"]] for r in rows}
    assert got[DIST_QUERIES[1]][0][1] == [hll_ref.hll(every_l, 12, "LONG"), hll_ref.hll(every_s, 8, "STRING")]

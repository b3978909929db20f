"""-m gpu: SUM / AVG / MIN / MAX over expressions of two or more columns against the per-row reference
(tests/expr_ref.py): sums within gamma_n * sum|x| of the exact sum of the row values (NaN / +-inf / +0.0 by rule), MIN / MAX
bit for bit in Double.compare order, AVG counts exact.

Segments of 1 .. 100 003 rows hold INT columns at the INT ends, LONG columns at the int64 ends and at 2^53 + 1, FLOAT and
DOUBLE columns with NaN, +-inf and -0.0, a raw INT and a raw DOUBLE column (dictionaries synthesised at load, or the raw
INT streamed as 32-bit values with raw_dict_max=0), and two group-by columns.  Aggregation only and GROUP BY on the
shared-memory, dense and hash tables, with and without a filter, with the count carrier on, off and overflowing; 17
merged segments whose operand dictionaries differ; ORDER BY ... LIMIT, HAVING, a FILTER clause, an EMPTY segment, DataTable
bytes and CLI rows by value, the loopback cross-GPU routes (scalars exact, group-by refused before any collective), the
refusals of a deferred or reduced group-by, the statistics and every other refusal."""
import dataclasses
import math
import struct

import numpy as np
import pytest

from expr_ref import check_value, row_values
from filter_ref import matching_docs
from gpu_util import to_device, tuned
from pinot_b200 import cli, sql
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED, Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 33, 4096, 8193, 100_003]
EXPRS = ["times(i,j)", "minus(l,i)", "divide(d,f)", "plus(f,d)", "mod(l,j)", "times(ri,rd)", "abs(minus(floor(d),ceil(f)))",
         "plus(i,i)", "divide(d,plus(j,'1'))", "times(minus(i,'3.5'),l)"]
FNS = ["SUM", "AVG", "MIN", "MAX"]


def _segment(oracle, n, seed, name=None, edges=True, raw_double=True):
    rng = np.random.default_rng(seed)
    i = (rng.integers(-3000, 3000, size=n) * 7).astype(np.int32)
    j = rng.integers(-5, 6, size=n).astype(np.int32)
    longs = np.array([INT64_MIN, INT64_MAX, (1 << 53) + 1, -(1 << 53) - 1, 0, 7, -12], dtype=np.int64)
    lv = rng.integers(-10_000, 10_000, size=n).astype(np.int64)
    f = (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32)
    d = rng.integers(-600, 600, size=n) / 3.0
    if edges:
        i[rng.integers(0, n, size=max(1, n // 60))] = INT_MAX
        i[rng.integers(0, n, size=max(1, n // 60))] = INT_MIN
        lv[rng.integers(0, n, size=max(1, n // 40))] = longs[rng.integers(0, len(longs), size=max(1, n // 40))]
        f[rng.integers(0, n, size=max(1, n // 90))] = -0.0
        d[rng.integers(0, n, size=max(1, n // 90))] = -0.0
        if n > 1000:   # the special values in the larger segments only, so that small groups stay finite too
            d[rng.integers(0, n, size=2)] = np.nan
            f[rng.integers(0, n, size=1)] = np.inf
            d[rng.integers(0, n, size=1)] = -np.inf
    cols = {"rid": np.arange(n, dtype=np.int32), "i": i, "j": j, "l": lv, "f": f, "d": d,
            "ri": rng.integers(-1_000_000, 1_000_000, size=n).astype(np.int32),
            "rd": rng.integers(-50, 50, size=n) / 4.0 if raw_double else rng.integers(-50, 50, size=n).astype(np.int32),
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 3000, size=n).astype(np.int32),
            "s": np.array([b"a", b"bb", b"c"])[rng.integers(0, 3, size=n)]}
    return oracle.build_segment(name or f"ex{n}_{seed}", cols, raw=["ri", "rd"])


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def segs(oracle, ctx):
    out = []
    for n in SIZES:
        seg = _segment(oracle, n, n)
        out.append((seg, to_device(ctx, seg)))
    yield out
    for _, dev in out:
        dev.destroy()


def _query(aggs, flt=None, group_by=(), **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), limit=kw.pop("limit", 100_000), **kw)


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _check(oracle, data, dev, q, b, what):
    """Every expression aggregation of block b (over the segments `data`, one result) against the reference."""
    rows = 1 if b.num_groups < 0 else b.num_groups
    got = {}
    for r in range(rows):
        got[tuple(_py(dev.dictionary_value(c, int(b.keys[r, k]))) for k, c in enumerate(q.group_by))] = r
    for a, agg in enumerate(q.aggregations):
        if agg.function not in FNS or "(" not in (agg.column or ""):
            continue
        ref = row_values(oracle, data, q.filter, q.group_by, agg.column)
        if q.group_by:
            assert set(got) == set(ref), f"{what} {agg}: groups differ"
        for key, r in got.items():
            xs = ref.get(key, [])
            d, l = float(b.doubles[a][r]), int(b.longs[a][r])
            assert check_value(agg.function, d, l, xs), f"{what} {agg.function}({agg.column}) {key}: {d!r} ({l}) over {len(xs)} rows"


FILTERS = [None, Predicate("RANGE", "i", [], -5000, 9000, True, False),
           Filter("AND", [Predicate("IN", "g", [1, 4, 7]), Predicate("RANGE", "rid", [], 3, None, True, True)])]


def _aggs(exprs):
    return [Aggregation(fn, e) for fn, e in zip(FNS * 3, exprs)][:6]


def test_aggregation_only(oracle, pm, segs):
    for seg, dev in segs:
        for fi, flt in enumerate(FILTERS):
            for k in range(0, len(EXPRS), 5):
                q = _query(_aggs(EXPRS[k:k + 5]) + [Aggregation("COUNT")], flt)
                _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"n={seg.num_docs} f={fi} k={k}")


@pytest.mark.parametrize("dense_max", [1 << 24, 1])
def test_group_by(oracle, ctx, pm, segs, dense_max):
    """Shared-memory (g), dense and hash (dense_max=1) tables, with a filter and without."""
    with tuned(ctx, dense_max=dense_max):
        for seg, dev in segs:
            for gb in (["g"], ["h"], ["g", "h"]):
                for flt in FILTERS[:2]:
                    q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("COUNT"), Aggregation("MIN", "divide(d,f)"),
                                Aggregation("AVG", "plus(f,d)"), Aggregation("MAX", "minus(l,i)"), Aggregation("SUM", "i")], flt, group_by=gb)
                    _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"dense_max={dense_max} n={seg.num_docs} {gb}")


@pytest.mark.parametrize("knobs", [dict(pack_count=0), dict(pack_count=1), dict(pack_shift=2), dict(smem_groups=0), dict(warps=8),
                                   dict(raw_dict_max=0)], ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()))
def test_knobs(oracle, ctx, pm, knobs):
    """The count carrier on, off and overflowing (a retry rebuilds the expression tables), other scan shapes, and raw
    INT columns streamed as 32-bit values (raw_dict_max=0)."""
    with tuned(ctx, **knobs):
        for n in (8193, 100_003):
            # a raw DOUBLE column is only loaded with a synthesised dictionary: streamed raw leaves are 32-bit
            seg = _segment(oracle, n, 77 + n, raw_double=knobs.get("raw_dict_max") != 0)
            dev = to_device(ctx, seg)
            try:
                for gb in ([], ["g"], ["h"]):
                    for flt in FILTERS[:2]:
                        q = _query([Aggregation("SUM", "i"), Aggregation("SUM", "times(ri,j)"), Aggregation("AVG", "plus(ri,i)"),
                                    Aggregation("MAX", "minus(ri,j)"), Aggregation("MIN", "times(rd,ri)"), Aggregation("COUNT")], flt, group_by=gb)
                        _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"{knobs} n={n} {gb}")
            finally:
                dev.destroy()


def _column_aggs_equal(q, a_block, b_block, idx_a, idx_b):
    rows = 1 if a_block.num_groups < 0 else a_block.num_groups
    assert a_block.num_groups == b_block.num_groups
    for r in range(rows):
        assert list(a_block.keys[r]) == list(b_block.keys[r]) if a_block.num_groups >= 0 else True
        for x, y in zip(idx_a, idx_b):
            fn = q.aggregations[x].function
            da, db = float(a_block.doubles[x][r]), float(b_block.doubles[y][r])
            assert int(a_block.longs[x][r]) == int(b_block.longs[y][r])
            if fn == "SUM" and q.aggregations[x].column in ("d", "l"):
                assert da == pytest.approx(db, rel=1e-12) or (math.isnan(da) and math.isnan(db))
            else:
                assert struct.pack("<d", da) == struct.pack("<d", db), f"{fn} row {r}"


def test_column_aggregations_unchanged(pm, segs):
    """Adding expression aggregations leaves the column aggregations as they were: COUNT, MIN, MAX, INT sums bit-identical,
    floating sums within the bound."""
    for seg, dev in segs[3:]:
        for gb in ([], ["g"], ["h"]):
            base = _query([Aggregation("COUNT"), Aggregation("SUM", "i"), Aggregation("MIN", "d"), Aggregation("MAX", "l")], FILTERS[1], group_by=gb)
            withx = dataclasses.replace(base, aggregations=[Aggregation("SUM", "times(i,j)")] + base.aggregations + [Aggregation("MAX", "plus(d,f)")])
            a = pm.execute_segments([dev], base)[0]
            b = pm.execute_segments([dev], withx)[0]
            _column_aggs_equal(base, a, b, [0, 1, 2, 3], [1, 2, 3, 4])


def test_statistics(oracle, pm, segs):
    seg, dev = segs[4]
    q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("MAX", "plus(d,i)")], FILTERS[1], group_by=["g"])
    plain = _query([Aggregation("COUNT")], FILTERS[1], group_by=["g"])
    b, p = pm.execute_segments([dev], q)[0], pm.execute_segments([dev], plain)[0]
    matched = int(np.count_nonzero(matching_docs(oracle, seg, FILTERS[1])))
    assert b.stats.num_docs_scanned == p.stats.num_docs_scanned == matched
    assert b.stats.num_entries_scanned_in_filter == p.stats.num_entries_scanned_in_filter
    assert b.stats.num_entries_scanned_post_filter == matched * 4   # g, i, j, d: each column once


def test_seventeen_segments_merged(oracle, ctx, pm):
    """Merged on the device: the group-by key bound to a domain, the operand columns each with their own dictionary."""
    data = [_segment(oracle, 5000 + 37 * k, 500 + k, name=f"ex17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = DictionaryDomain.build(ctx, devs, ["g", "h"])
    try:
        for d in devs:
            d.bind_domain(domain)
        for gb in ([], ["g"], ["g", "h"]):
            q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("AVG", "divide(d,plus(j,'1'))"), Aggregation("MIN", "minus(l,i)"),
                        Aggregation("MAX", "times(ri,rd)"), Aggregation("COUNT")], FILTERS[1], group_by=gb)
            _check(oracle, data, devs[0], q, pm.execute_segments(devs, q, merge=True)[0], f"merged {gb}")
    finally:
        for d in devs:
            d.destroy()
        domain.release()


def test_order_by_having_filter_clause(oracle, pm, segs):
    seg, dev = segs[5]
    q = sql.parse("SELECT g, SUM(i * j), MAX(d - f) FROM t WHERE i >= -5000 GROUP BY g ORDER BY SUM(i * j) DESC LIMIT 4")
    b = pm.execute_segments([dev], q, merge=True)[0]
    ref = row_values(oracle, [seg], q.filter, ["g"], "times(i,j)")
    sums = sorted(((float(sum(x for x in xs)), k) for k, xs in ref.items()), reverse=True)   # integral sums below 2^53: exact
    assert b.num_groups >= 4
    assert [_py(dev.dictionary_value("g", int(b.keys[r, 0]))) for r in range(4)] == [k[0] for _, k in sums[:4]]
    _check(oracle, [seg], dev, q, b, "order by")
    q = sql.parse("SELECT g, SUM(i * j) FROM t GROUP BY g HAVING SUM(i * j) > 0")
    b = pm.execute_segments([dev], q, merge=True)[0]
    ref = row_values(oracle, [seg], None, ["g"], "times(i,j)")
    assert b.num_groups == sum(1 for xs in ref.values() if sum(xs) > 0)
    q = sql.parse("SELECT g, SUM(i * j) FILTER (WHERE j > 0), COUNT(*) FROM t GROUP BY g")
    b = pm.execute_segments([dev], q)[0]
    ref = row_values(oracle, [seg], Predicate("RANGE", "j", [], 0, None, False, True), ["g"], "times(i,j)")
    for r in range(b.num_groups):
        key = (_py(dev.dictionary_value("g", int(b.keys[r, 0]))),)
        assert check_value("SUM", float(b.doubles[0][r]), 0, ref.get(key, [])), key


def test_datatable_and_cli(oracle, ctx, pm, segs, tmp_path, capsys):
    """DataTable bytes: an expression SUM / AVG / MIN / MAX written like the function over a DOUBLE column, under its
    canonical name, with the reference's values; the CLI's rows over two segment directories, per segment and merged on
    the device, against the reference over both."""
    import json

    from datatable_util import parse as parse_datatable
    from segment_dir_util import write_segment_dir
    seg, dev = segs[3]
    q = sql.parse("SELECT g, SUM(i * j), AVG(i * j), MIN(i * j), MAX(i * j) FROM t GROUP BY g")
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        dt = parse_datatable(pm.to_datatable(dev, q, b))
    finally:
        b.release(ctx)
    assert dt["column_names"] == ["g", "sum(times(i,j))", "avg(times(i,j))", "min(times(i,j))", "max(times(i,j))"]
    assert dt["column_types"][1] == "DOUBLE" and dt["column_types"][3] == "DOUBLE" and dt["column_types"][4] == "DOUBLE"
    ref = row_values(oracle, [seg], None, ["g"], "times(i,j)")
    assert len(dt["rows"]) == len(ref)
    for row in dt["rows"]:
        xs = ref[(row[0],)]
        assert check_value("SUM", row[1], 0, xs) and check_value("AVG", row[2][0], row[2][1], xs)
        assert check_value("MIN", row[3], 0, xs) and check_value("MAX", row[4], 0, xs)
    data = [_segment(oracle, 3000 + k, 900 + k, name=f"excli{k}", edges=False) for k in range(2)]
    dirs = [str(write_segment_dir(tmp_path / f"s{k}", s)) for k, s in enumerate(data)]
    ref_sum = row_values(oracle, data, None, ["g"], "times(i,j)")
    ref_max = row_values(oracle, data, None, ["g"], "minus(d,f)")
    for extra in ([], ["--merge-on-device"]):
        argv = ["SELECT g, SUM(i * j), MAX(d - f) FROM t GROUP BY g ORDER BY g LIMIT 100", "--json"]
        for d in dirs:
            argv += ["--segment-dir", d]
        capsys.readouterr()
        assert cli.main(argv + extra) == 0
        out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
        assert len(out["rows"]) == len(ref_sum), extra
        for g, total, mx in out["rows"]:
            assert check_value("SUM", float(total), 0, ref_sum[(int(g),)]), (extra, g)
            assert check_value("MAX", float(mx), 0, ref_max[(int(g),)]), (extra, g)


def test_refusals(oracle, pm, segs):
    seg, dev = segs[3]
    for text in ("SELECT SUM(datetrunc('DAY', l) + i) FROM t", "SELECT DISTINCTCOUNT(i * j) FROM t",
                 "SELECT PERCENTILE(i * j, 50) FROM t", "SELECT VAR_POP(i * j) FROM t",
                 "SELECT COUNT(*) FROM t GROUP BY i * j"):
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], sql.parse(text))
    nine = "plus(" * 8 + "i" + ",j)" * 8
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], _query([Aggregation("SUM", nine)]))
    with pytest.raises(Pb200Error):
        pm.execute_segments([dev], _query([Aggregation("SUM", "times(i,nosuch)")]))
    for agg in (Aggregation("DISTINCTSUM", "times(i,j)"), Aggregation("DISTINCTAVG", "times(i,j)"),
                Aggregation("LASTWITHTIME", "times(i,j)", time_column="i", value_type="DOUBLE"),
                Aggregation("SUM", "times(s,i)")):   # the last: a STRING leaf
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([agg]))


def test_group_by_not_combined_across_gpus(pm, ctx, segs):
    """With GROUP BY the expression tables are not among the reducible blocks: a deferred finalize, reduce_world > 1 and
    the device-buffer and combine entry points all refuse, so no reduce can keep only one rank's expression values."""
    seg, dev = segs[3]
    q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("COUNT")], group_by=["g"])
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], q, merge=True, keep_handle=True)                 # PB200_Q_DEFER_FINALIZE
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], q, merge=True, reduce_world=2)
    b = pm.execute_segments([dev], q, merge=True, keep_handle=True, defer=False)[0]
    try:
        import ctypes as C
        p, n = C.c_void_p(), C.c_int64()
        assert ctx.lib.pb200_result_device_buffers(b.handle, 1, C.byref(p), C.byref(n)) == E_UNSUPPORTED
    finally:
        b.release(ctx)
    # aggregation only: the scalars are combined by value, never through the INT exact sum
    q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("SUM", "i")])
    b = pm.execute_segments([dev], q, merge=True, keep_handle=True, defer=False)[0]
    try:
        import ctypes as C
        v = C.c_int64()
        assert ctx.lib.pb200_result_exact_sum(b.handle, 0, C.byref(v)) == 0
        assert ctx.lib.pb200_result_exact_sum(b.handle, 1, C.byref(v)) == 1
    finally:
        b.release(ctx)


def test_empty_segment_next_to_expressions(oracle, pm, segs):
    """Per-segment submission where one segment's filter folds to EMPTY: its result is built on the host."""
    data = [s for s, _ in segs[2:4]]
    devs = [d for _, d in segs[2:4]]
    flt = Predicate("RANGE", "rid", [], 40, None, True, True)    # segs[2] has 33 rows: no match there
    for gb in ([], ["g"]):
        q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("MIN", "plus(d,i)"), Aggregation("MAX", "minus(l,i)")], flt, group_by=gb)
        blocks = pm.execute_segments(devs, q)
        for seg, dev, b in zip(data, devs, blocks):
            _check(oracle, [seg], dev, q, b, f"empty {gb} n={seg.num_docs}")


@pytest.mark.parametrize("world", [2, 3])
def test_loopback_scalars(oracle, world):
    """execute_and_combine with `world` ranks on one GPU (tests/loopback_dist.py), each with its own segments and
    dictionaries: aggregation-only expression SUM / AVG / MIN / MAX take the scalars route, and the root's values hold to
    the reference over every rank's rows."""
    from loopback_dist import run_ranks, values
    from pinot_b200.distributed import execute_and_combine
    hosts = [[_segment(oracle, 3_000 + 101 * r + 7 * k, 700 + 10 * r + k, name=f"exl{r}_{k}") for k in range(1 + r % 2)]
             for r in range(world)]
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [[to_device(c, h) for h in hs] for c, hs in zip(ctxs, hosts)]
    try:
        everything = [h for hs in hosts for h in hs]
        q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("AVG", "divide(d,plus(j,'1'))"), Aggregation("MIN", "minus(l,i)"),
                    Aggregation("MAX", "times(ri,rd)"), Aggregation("COUNT")], FILTERS[1])
        got = values(run_ranks(world, lambda dist: execute_and_combine(B200PlanMaker(ctxs[dist.get_rank()]), devs[dist.get_rank()], q, dist)))
        assert all(g is None for g in got[1:])
        _check(oracle, everything, devs[0][0], q, got[0], f"world {world}")
        assert int(got[0].longs[4][0]) == sum(int(np.count_nonzero(matching_docs(oracle, h, q.filter))) for h in everything)
    finally:
        for ds in devs:
            for d in ds:
                d.destroy()
        for c in ctxs:
            c.close()


def test_loopback_group_by_refused_before_any_collective(oracle):
    from loopback_dist import run_ranks
    from pinot_b200.distributed import execute_and_combine
    world = 2
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [to_device(c, _segment(oracle, 2_000 + r, 60 + r, name=f"exr{r}")) for r, c in enumerate(ctxs)]
    try:
        q = _query([Aggregation("SUM", "times(i,j)"), Aggregation("COUNT")], group_by=["g"])
        outs = run_ranks(world, lambda dist: execute_and_combine(B200PlanMaker(ctxs[dist.get_rank()]), [devs[dist.get_rank()]], q, dist))
        for o in outs:
            assert isinstance(o.error, UnsupportedQueryError) and o.calls == [], (o.error, o.calls)
    finally:
        for d in devs:
            d.destroy()
        for c in ctxs:
            c.close()

"""-m gpu: FIRSTWITHTIME / LASTWITHTIME(v, t, 'T') against the per-row reference (tests/withtime_ref.py): the data value
(through its dictId), the double column and the exact time value of every row.

Segments of 1 .. 196 609 rows hold INT, LONG (at the int64 ends and beyond 2^53), FLOAT, DOUBLE and STRING data
columns, an INT time column with heavy ties, a LONG time column at the int64 extremes, an epoch-millis column for
DATETRUNC and a raw INT time column whose dictionary is synthesised at load.  Aggregation only and GROUP BY, next to SUM,
COUNT, MIN and PERCENTILE, on the dense and the hash table and under the scan knobs; 17 domain-bound segments merged on
the device and by value; ORDER BY ... DESC LIMIT, HAVING, empty and single-row groups, ties inside and across segments,
and the refusals."""
import numpy as np
import pytest

from gpu_util import to_device, tuned
from withtime_ref import withtime
from pinot_b200 import cli
from pinot_b200._lib import E_INVALID, Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import DictionaryDomain, B200Context, B200PlanMaker
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 1_025, 49_157, 196_609]
TYPES = {"i": "INT", "l": "LONG", "f": "FLOAT", "d": "DOUBLE", "s": "STRING"}
HOUR = 3_600_000
HOUR_EXPR = "datetrunc('HOUR',ts)"


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 3000, size=n) * 7 - 9000).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i,
            "l": np.array([INT64_MIN, INT64_MAX, -1, 0, 5, (1 << 53) + 1, 1 << 53, INT64_MAX - 1], dtype=np.int64)[rng.integers(0, 8, size=n)],
            "f": (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32),
            "d": rng.integers(-600, 600, size=n) / 3.0,
            "s": np.array([b"a", b"ab", b"b", b"zz", b"q"])[rng.integers(0, 5, size=n)],
            "ti": (rng.integers(0, 40, size=n) * 1000 - 20_000).astype(np.int32),                # heavy ties
            "tl": np.array([INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1, (1 << 53) + 1, 1 << 53, 0],
                           dtype=np.int64)[rng.integers(0, 7, size=n)],                           # int64 ends, beyond 2^53
            "ts": (1_700_000_000_000 + rng.integers(0, 48, size=n) * 1_800_000 + rng.integers(0, 1000, size=n)).astype(np.int64),
            "tr": rng.integers(-500, 500, size=n).astype(np.int32) * 1000,                      # raw: dictionary synthesised at load
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 300, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"wt{n}_{seed}", cols, raw=["tr"])


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


def _query(aggs, flt=None, group_by=(), order_by=(), limit=100_000, **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), order_by=list(order_by), limit=limit, **kw)


def _wt(fn, v, t):
    return Aggregation(fn, v, time_column=t, value_type=TYPES[v])


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _time_of(t):
    if t == HOUR_EXPR:
        return lambda si, x: (x // HOUR) * HOUR
    return None


def _source(t):
    return "ts" if t == HOUR_EXPR else t


def _check(oracle, data, dev, q, b, what):
    """Every FIRST/LASTWITHTIME of block b (over the segments `data`, one result) against the reference."""
    gb = q.group_by
    rows = 1 if b.num_groups < 0 else b.num_groups
    for a, agg in enumerate(q.aggregations):
        if agg.function not in ("FIRSTWITHTIME", "LASTWITHTIME"):
            continue
        ref = withtime(oracle, data, q.filter, gb, agg.function, agg.column, _source(agg.time_column), _time_of(agg.time_column))
        got = {}
        for r in range(rows):
            key = tuple(_py(dev.dictionary_value(c, int(b.keys[r, j]))) for j, c in enumerate(gb))
            got[key] = r
        assert set(got) == set(ref), f"{what}: groups differ"
        for key, r in got.items():
            want = ref[key]
            d, t, i = float(b.doubles[a][r]), int(b.longs[a][r]), int(b.dict_ids[a][r])
            if want is None:
                assert i == -1 and d == float("-inf"), f"{what} {agg} {key}: expected no row"
                continue
            assert t == want[0], f"{what} {agg} {key}: time {t} != {want[0]}"
            assert _py(dev.dictionary_value(agg.column, i)) == want[1], f"{what} {agg} {key}: value"
            assert d == (float(i) if agg.value_type == "STRING" else float(want[1])), f"{what} {agg} {key}: double {d}"


FILTERS = [None,
           Predicate("RANGE", "i", [], -5000, 9000, True, False),
           Filter("AND", [Predicate("IN", "g", [1, 4, 7]), Predicate("RANGE", "rid", [], 3, None, True, True)])]


@pytest.mark.parametrize("fn", ["FIRSTWITHTIME", "LASTWITHTIME"])
def test_aggregation_only_every_type(oracle, pm, segs, fn):
    for seg, dev in segs:
        for fi, flt in enumerate(FILTERS):
            aggs = [_wt(fn, v, t) for v, t in (("i", "ti"), ("l", "tl"), ("f", "ti"), ("d", "tl"), ("s", "ti"))]
            aggs.append(Aggregation("COUNT"))
            q = _query(aggs, flt)
            _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"n={seg.num_docs} f={fi}")
            # next to SUM / MIN / PERCENTILE in the same query
            q = _query([Aggregation("SUM", "i"), _wt(fn, "l", "ti"), Aggregation("MIN", "i"), Aggregation("PERCENTILE", "d", arg=50.0),
                        _wt(fn, "s", "tl")], flt)
            _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"mixed n={seg.num_docs} f={fi}")


@pytest.mark.parametrize("dense_max", [1 << 24, 1])
def test_group_by(oracle, ctx, pm, segs, dense_max):
    with tuned(ctx, dense_max=dense_max):
        for seg, dev in segs:
            for gb in (["g"], ["h"], ["g", "h"]):
                for flt in FILTERS[:2]:
                    q = _query([Aggregation("COUNT"), _wt("LASTWITHTIME", "i", "ti"), Aggregation("SUM", "i"),
                                _wt("FIRSTWITHTIME", "s", "ti"), _wt("LASTWITHTIME", "l", "tl"), Aggregation("PERCENTILE", "f", arg=90.0)],
                               flt, group_by=gb)
                    _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"dense_max={dense_max} n={seg.num_docs} {gb}")
                # the key table alone: no count, no carrier, no MIN / MAX marks the groups
                q = _query([_wt("FIRSTWITHTIME", "d", "tl"), _wt("LASTWITHTIME", "f", "ti")], group_by=gb)
                _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"alone dense_max={dense_max} {gb}")


@pytest.mark.parametrize("fn", ["FIRSTWITHTIME", "LASTWITHTIME"])
def test_time_kinds(oracle, pm, segs, fn):
    """Time as a derived column (DATETRUNC), as a raw column with a synthesised dictionary, and v == t."""
    for seg, dev in segs[1:]:
        for gb in ([], ["g"]):
            q = _query([_wt(fn, "i", HOUR_EXPR), _wt(fn, "s", "tr"), Aggregation(fn, "ti", time_column="ti", value_type="INT"),
                        Aggregation(fn, "l", time_column="l", value_type="LONG")], group_by=gb)
            _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"n={seg.num_docs} {gb}")


KNOBS = [dict(sparse_max_agg=0), dict(sparse_max_agg=32), dict(warps=8), dict(skip=0), dict(grid=1), dict(grid=7),
         dict(smem_groups=0), dict(smem_groups=1)]


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()))
def test_knobs(oracle, ctx, pm, segs, knobs):
    with tuned(ctx, **knobs):
        for seg, dev in segs[2:]:
            for gb in ([], ["g"]):
                for flt in FILTERS:
                    q = _query([Aggregation("COUNT"), Aggregation("SUM", "i"), _wt("LASTWITHTIME", "d", "ti"), _wt("FIRSTWITHTIME", "i", "tl")],
                               flt, group_by=gb)
                    _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"{knobs} n={seg.num_docs} {gb}")


def test_seventeen_segments_merged(oracle, ctx, pm):
    """Ties across segments: the later segment wins for LAST, the earlier one for FIRST -- on the device (one merged
    result) and in the CLI's by-value merge of per-segment results."""
    data = [_segment(oracle, 20_000 + 37 * k, 1000 + k, name=f"wt17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = None
    try:
        for gb in ([], ["g"]):
            q = _query([_wt("LASTWITHTIME", "i", "ti"), _wt("FIRSTWITHTIME", "s", "ti"), _wt("LASTWITHTIME", "l", "tl"), Aggregation("COUNT")],
                       Predicate("RANGE", "i", [], -5000, 9000, True, False), group_by=gb)
            refs = [withtime(oracle, data, q.filter, gb, a.function, a.column, a.time_column) for a in q.aggregations[:3]]
            per_seg = cli.final_rows(q, cli.merge_blocks(q, devs, pm.execute_segments(devs, q)))
            assert len(per_seg) == len(refs[0])
            for row in per_seg:
                key = tuple(row[:len(gb)])
                assert [_py(x) for x in row[len(gb):len(gb) + 3]] == [r[key][1] for r in refs], f"{gb} {key}"
            if domain is None:
                with pytest.raises(UnsupportedQueryError):   # no shared dictionary: refused, never merged by dictId
                    pm.execute_segments(devs, q, merge=True)
                domain = DictionaryDomain.build(ctx, devs, ["i", "s", "l", "ti", "tl", "g"])
                for d in devs:
                    d.bind_domain(domain)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            _check(oracle, data, devs[0], q, merged, f"merged {gb}")
            assert [[_py(x) for x in r] for r in cli.final_rows(q, cli.merge_blocks(q, devs[:1], [merged]))] == \
                   [[_py(x) for x in r] for r in per_seg]
    finally:
        for d in devs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_order_by_and_having(oracle, pm, segs):
    seg, dev = segs[-1]
    agg = _wt("LASTWITHTIME", "d", "ti")
    ref = withtime(oracle, [seg], None, ["h"], "LASTWITHTIME", "d", "ti")
    # ORDER BY LASTWITHTIME(...) DESC LIMIT 7, trimmed on the device; ties by key ascending
    q = _query([agg, Aggregation("COUNT")], group_by=["h"], order_by=[(str(agg), False)], limit=7)
    b = pm.execute_segments([dev], q)[0]
    want = sorted(ref, key=lambda k: (-ref[k][1], k))[:7]
    got = [(_py(dev.dictionary_value("h", int(b.keys[r, 0]))),) for r in range(b.num_groups)][:7]
    assert got == want
    # HAVING compares the double value
    q = _query([agg, Aggregation("COUNT")], group_by=["h"],
               having=Predicate("RANGE", str(agg), [], 0.0, None, False, True))
    b = pm.execute_segments([dev], q)[0]
    got = {_py(dev.dictionary_value("h", int(b.keys[r, 0]))) for r in range(b.num_groups)}
    assert got == {k[0] for k, v in ref.items() if v[1] > 0.0}


def test_empty_and_single_row(oracle, pm, segs):
    seg, dev = segs[0]   # one row: every group has a single row
    for gb in ([], ["g"], ["h"]):
        q = _query([_wt("LASTWITHTIME", "s", "tl"), _wt("FIRSTWITHTIME", "i", "ti")], group_by=gb)
        _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"one row {gb}")
    seg, dev = segs[2]
    for flt in (Predicate("RANGE", "i", [], 10 ** 10, None, True, True),      # folds to EMPTY on the host
                Predicate("RANGE", "rid", [], 5, 4, True, True),              # matches nothing on the device
                Predicate("EQ", "rid", [17])):                                 # one row
        q = _query([_wt("LASTWITHTIME", "d", "ti"), _wt("FIRSTWITHTIME", "l", "tl"), Aggregation("COUNT")], flt)
        _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"{flt}")


def test_refusals(oracle, ctx, pm, segs):
    seg, dev = segs[2]
    for bad in (Aggregation("LASTWITHTIME", "i", time_column="d", value_type="INT"),       # DOUBLE time
                Aggregation("LASTWITHTIME", "i", time_column="s", value_type="INT"),       # STRING time
                Aggregation("LASTWITHTIME", "i", time_column="ti", value_type="LONG"),     # type literal mismatch
                Aggregation("FIRSTWITHTIME", "f", time_column="ti", value_type="DOUBLE")):
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([bad]))
    agg = _wt("LASTWITHTIME", "i", "ti")
    with pytest.raises(UnsupportedQueryError):   # FILTER (WHERE ...) clause anywhere in the query
        pm.execute_segments([dev], _query([agg, Aggregation("SUM", "i", filter=Predicate("EQ", "g", [1]))]))
    with pytest.raises(UnsupportedQueryError):   # deferred (cross-GPU) finalize
        pm.execute_segments([dev], _query([agg], group_by=["g"]), merge=True, keep_handle=True)
    b = pm.execute_segments([dev], _query([agg], group_by=["g"]), keep_handle=True, defer=False)[0]
    try:
        with pytest.raises(UnsupportedQueryError):   # DataTable bytes
            pm.to_datatable(dev, _query([agg], group_by=["g"]), b)
    finally:
        b.release(ctx)
    with tuned(ctx, raw_dict_max=0):   # raw INT streamed as 32-bit values: no dictIds
        raw = to_device(ctx, _segment(oracle, 5_000, 5))
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([raw], _query([Aggregation("LASTWITHTIME", "i", time_column="tr", value_type="INT")]))
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([raw], _query([Aggregation("LASTWITHTIME", "tr", time_column="ti", value_type="INT")]))
    finally:
        raw.destroy()
    # the older entry points carry no time column: PB200_E_INVALID
    import ctypes as C
    from pinot_b200.plan_maker import _marshal_query
    hq, _keep = _marshal_query(_query([agg]), False)
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * 1)()
    assert ctx.lib.pb200h_execute(ctx.handle, C.byref(hq), (C.c_void_p * 1)(dev.handle), 1, res, kinds) == E_INVALID
    assert isinstance(E_INVALID, int) and issubclass(UnsupportedQueryError, Pb200Error)

"""-m gpu: PERCENTILE(col, p) against the value-space reference (tests/percentile_ref.py): every value bit-exact, and the
selected dictId names the reference's stored value (a LONG beyond 2^53 is checked through it).

Segments of 1 .. 196 609 rows hold INT (at INT_MIN / INT_MAX), LONG (at the int64 ends and 2^53 + 1), FLOAT (with
+-inf), DOUBLE columns and a raw INT column whose dictionary is synthesised at load.  Filters: none, folded to EMPTY,
scan ranges, IN, an inverted-index leaf and doc ranges of the sorted column.  Percentiles 0 .. 100 including 99.9 and the
double just below 100.  Aggregation only on the dense and the per-row route under the scan knobs; GROUP BY on the dense
table and the hash table, with and without a count carrier; ORDER BY PERCENTILE ASC / DESC with a trim; 17 domain-bound
segments merged on the device against per-segment histograms merged by value; every refusal."""
import math

import numpy as np
import pytest

from gpu_util import to_device, tuned
import percentile_oracle
from percentile_ref import group_values, percentile, pick
from pinot_b200 import cli
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED, Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain  # noqa: F401
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 1_025, 49_157, 196_609]
PS = [0.0, 0.1, 1.0, 50.0, 95.0, 99.0, 99.9, 100.0, math.nextafter(100.0, 0.0)]
COLUMNS = ["i", "l", "f", "d", "r"]


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 3000, size=n) * 7 - 9000).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    f = (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32)
    f[rng.integers(0, n, size=max(1, n // 100))] = np.inf
    f[rng.integers(0, n, size=max(1, n // 100))] = -np.inf
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i,
            "l": np.array([INT64_MIN, INT64_MAX, -1, 0, 5, (1 << 53) + 1, 1 << 53, INT64_MAX - 1], dtype=np.int64)[rng.integers(0, 8, size=n)],
            "f": f,
            "d": rng.integers(-600, 600, size=n) / 3.0,
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 300, size=n).astype(np.int32),
            "s": np.array([b"a", b"ab", b"b"])[rng.integers(0, 3, size=n)],
            "inv": rng.integers(0, 40, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"pct{n}_{seed}", cols, inverted=["inv"], raw=["r"])


def _filters(n):
    return [None,
            Predicate("RANGE", "i", [], 10 ** 10, None, True, True),                    # folds to EMPTY on the host
            Predicate("RANGE", "i", [], -5000, 9000, True, False),
            Predicate("IN", "g", [1, 4, 7]),
            Predicate("EQ", "inv", [7]),
            Predicate("RANGE", "rid", [], n // 3, n - 2, True, True),                   # sorted column: doc ranges
            Filter("AND", [Predicate("RANGE", "f", [], -20.0, 30.0, True, True), Predicate("RANGE", "l", [], 0, None, True, True)])]


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


def _query(aggs, flt=None, group_by=(), order_by=(), limit=10, **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), order_by=list(order_by), limit=limit, **kw)


def _check_value(seg, dev, column, got_value, got_id, got_n, values, p, what):
    want = percentile(values, p)
    assert got_value == want or (math.isnan(got_value) and math.isnan(want)), f"{what}: {got_value!r} != {want!r}"
    assert np.float64(got_value).tobytes() == np.float64(want).tobytes(), what   # bit-exact (+-inf, 0.0)
    assert got_n == len(values), what
    v = pick(values, p)
    if v is None:
        assert got_id == -1, what
    elif seg.column(column).has_dictionary:
        assert seg.value_of(column, int(got_id)) == v, f"{what}: dictId {got_id} is not the value {v!r}"
    else:   # dictionary synthesised at load: the product's own lookup
        assert dev.dictionary_value(column, int(got_id)) == v, what


def _key_of(seg, group_by, keys_row):
    out = []
    for j, c in enumerate(group_by):
        v = seg.value_of(c, int(keys_row[j]))
        out.append(v.decode() if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v))
    return tuple(out)


ORACLE_MAX_DOCS = 50_000   # the oracle's chain runs per doc in Python: checked up to this segment size


def _check_block(oracle, seg, dev, q, b, what):
    """Every PERCENTILE of block b (one segment) against the value-space reference, and against the oracle's operator
    chain (tests/percentile_oracle.py) for segments up to ORACLE_MAX_DOCS, rows matched by key values."""
    refs = {}
    for a, agg in enumerate(q.aggregations):
        if agg.function != "PERCENTILE":
            continue
        if agg.column not in refs:
            refs[agg.column] = group_values(oracle, [seg], q.filter, q.group_by, agg.column)
        ref = refs[agg.column]
        if seg.num_docs <= ORACLE_MAX_DOCS:
            po = percentile_oracle.percentiles(oracle, [seg], q.filter, q.group_by, agg.column, [agg.arg])
            rows_po = 1 if b.num_groups < 0 else b.num_groups
            got = {(() if b.num_groups < 0 else _key_of(seg, q.group_by, b.keys[g])): float(b.doubles[a][g]) for g in range(rows_po)}
            assert got == {k: v[0] for k, v in po.items()}, f"{what} a={a}: against the oracle's chain"
        rows = 1 if b.num_groups < 0 else b.num_groups
        if q.group_by:
            assert b.num_groups == len(ref), what
        for g in range(rows):
            key = () if b.num_groups < 0 else _key_of(seg, q.group_by, b.keys[g])
            _check_value(seg, dev, agg.column, float(b.doubles[a][g]), int(b.dict_ids[a][g]), int(b.longs[a][g]),
                         ref[key], agg.arg, f"{what} a={a} key={key}")
            ids, counts = b.histograms[(a, g)]
            vals = np.repeat([seg.value_of(agg.column, int(d)) if seg.column(agg.column).has_dictionary
                              else dev.dictionary_value(agg.column, int(d)) for d in ids], counts)
            assert np.array_equal(np.asarray(vals, dtype=ref[key].dtype), ref[key]), f"{what}: histogram of {key}"
    return refs


def test_aggregation_only(oracle, pm, segs):
    for seg, dev in segs:
        n = seg.num_docs
        for fi, flt in enumerate(_filters(n)):
            for col in COLUMNS:
                q = _query([Aggregation("PERCENTILE", col, arg=p) for p in PS[:6]], flt)
                _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], f"n={n} f={fi} {col}")
                q = _query([Aggregation("PERCENTILE", col, arg=p) for p in PS[6:]], flt)
                _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], f"n={n} f={fi} {col} high")


def test_next_to_other_functions(oracle, pm, segs):
    seg, dev = segs[-1]
    q = _query([Aggregation("SUM", "i"), Aggregation("PERCENTILE", "l", arg=50.0), Aggregation("COUNT"),
                Aggregation("PERCENTILE", "l", arg=99.0), Aggregation("DISTINCTCOUNT", "g"), Aggregation("PERCENTILE", "d", arg=95.0)],
               Predicate("RANGE", "i", [], -5000, 9000, True, False))
    b = pm.execute_segments([dev], q)[0]
    _check_block(oracle, seg, dev, q, b, "mixed")
    q2 = _query([Aggregation("MIN", "l"), Aggregation("MAX", "f"), Aggregation("AVG", "i"), Aggregation("PERCENTILE", "f", arg=100.0)])
    b2 = pm.execute_segments([dev], q2)[0]
    _check_block(oracle, seg, dev, q2, b2, "mixed2")
    ref = group_values(oracle, [seg], None, [], "f")[()]
    assert float(b2.doubles[1][0]) == float(ref[-1]) == float(b2.doubles[3][0])   # MAX == PERCENTILE 100
    assert isinstance(b2.get_results(q2)[3], float)


@pytest.mark.parametrize("knobs", [{"sparse_max_agg": 0}, {"sparse_max_agg": 32}, {"warps": 8}, {"skip": 0}, {"grid": 1}, {"grid": 7}])
def test_routes_and_knobs(oracle, ctx, pm, segs, knobs):
    with tuned(ctx, **knobs):
        for seg, dev in segs[2:]:
            n = seg.num_docs
            for fi, flt in enumerate(_filters(n)):
                q = _query([Aggregation("PERCENTILE", "i", arg=p) for p in (0.0, 50.0, 99.9)] + [Aggregation("SUM", "i")], flt)
                _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], f"{knobs} n={n} f={fi}")
                # at most 64 dictIds: warp-private shared-memory histograms; 300 dictIds: one reduction per row
                q = _query([Aggregation("PERCENTILE", "g", arg=p) for p in (1.0, 50.0, 100.0)] +
                           [Aggregation("PERCENTILE", "l", arg=95.0), Aggregation("PERCENTILE", "h", arg=99.0)], flt)
                _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], f"{knobs} few ids n={n} f={fi}")
                q = _query([Aggregation("PERCENTILE", "d", arg=95.0), Aggregation("COUNT")], flt, group_by=["g"])
                _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], f"{knobs} gb n={n} f={fi}")


@pytest.mark.parametrize("dense_max", [1 << 24, 1])
def test_group_by(oracle, ctx, pm, segs, dense_max):
    with tuned(ctx, dense_max=dense_max):
        for seg, dev in segs:
            n = seg.num_docs
            for fi, flt in enumerate(_filters(n)[:5]):
                for aggs, gb in (([Aggregation("PERCENTILE", "l", arg=50.0), Aggregation("PERCENTILE", "l", arg=99.0)], ["g"]),
                                 # a count carrier: COUNT rides in the INT sum's reductions
                                 ([Aggregation("SUM", "i"), Aggregation("COUNT"), Aggregation("PERCENTILE", "f", arg=95.0)], ["g", "s"]),
                                 ([Aggregation("PERCENTILE", "i", arg=99.9), Aggregation("MAX", "i")], ["h"]),
                                 ([Aggregation("PERCENTILE", "r", arg=1.0)], ["rid"] if n <= 1025 else ["h", "g"])):
                    # hash tables: slots x cardinality entries, the slots sized by numGroupsLimit
                    q = _query(aggs, flt, group_by=gb, limit=100000, num_groups_limit=20_000)
                    b = pm.execute_segments([dev], q)[0]
                    _check_block(oracle, seg, dev, q, b, f"dense_max={dense_max} n={n} f={fi} {gb}")


def test_order_by_percentile(oracle, pm, segs):
    for seg, dev in segs[2:]:
        for asc in (True, False):
            for limit in (1, 3, 10):
                q = _query([Aggregation("COUNT"), Aggregation("PERCENTILE", "i", arg=99.0)], None, group_by=["h"],
                           order_by=[("percentile(i,99.0)", asc)], limit=limit, min_segment_group_trim_size=1)
                b = pm.execute_segments([dev], q)[0]
                ref = group_values(oracle, [seg], None, ["h"], "i")
                want = sorted(ref, key=lambda k: (percentile(ref[k], 99.0) if asc else -percentile(ref[k], 99.0), k))
                got = [_key_of(seg, ["h"], b.keys[g]) for g in range(b.num_groups)]
                assert got == want[:len(got)] and len(got) >= limit, (asc, limit)
                for g, key in enumerate(got):
                    assert float(b.doubles[1][g]) == percentile(ref[key], 99.0)
                # ties (the same percentile in many groups) are broken by the key ascending
                q = _query([Aggregation("PERCENTILE", "g", arg=50.0)], None, group_by=["h"], order_by=[("percentile(g,50.0)", asc)],
                           limit=limit, min_segment_group_trim_size=1)
                b = pm.execute_segments([dev], q)[0]
                ref = group_values(oracle, [seg], None, ["h"], "g")
                want = sorted(ref, key=lambda k: (percentile(ref[k], 50.0) if asc else -percentile(ref[k], 50.0), k))
                assert [_key_of(seg, ["h"], b.keys[g]) for g in range(b.num_groups)] == want[:b.num_groups]


def test_seventeen_segments_merged_on_device(oracle, ctx, pm):
    data = [_segment(oracle, 20_000 + 37 * k, 1000 + k, name=f"pct17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = None
    try:
        for gb in ([], ["g"]):
            q = _query([Aggregation("PERCENTILE", "i", arg=95.0), Aggregation("PERCENTILE", "i", arg=50.0), Aggregation("COUNT")],
                       Predicate("RANGE", "i", [], -5000, 9000, True, False), group_by=gb, limit=1000)
            per_seg = cli.final_rows(q, cli.merge_blocks(q, devs, pm.execute_segments(devs, q)))
            ref = group_values(oracle, data, q.filter, gb, "i")
            assert len(per_seg) == len(ref)
            for row in per_seg:
                key = tuple(row[:len(gb)])
                assert row[len(gb)] == percentile(ref[key], 95.0) and row[len(gb) + 1] == percentile(ref[key], 50.0)
            if domain is None:
                with pytest.raises(UnsupportedQueryError):   # no shared dictionary: refused, never merged by dictId
                    pm.execute_segments(devs, q, merge=True)
                domain = DictionaryDomain.build(ctx, devs, ["i", "g"])
                for d in devs:
                    d.bind_domain(domain)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            on_device = cli.final_rows(q, cli.merge_blocks(q, devs[:1], [merged]))
            assert on_device == per_seg
            if not gb:   # a domain id: the domain's dictionary holds the selected value at it
                assert devs[0].dictionary_value("i", int(merged.dict_ids[0][0])) == pick(ref[()], 95.0)
    finally:
        for d in devs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_empty_and_single_row_groups(oracle, pm, segs):
    seg, dev = segs[0]   # one row
    q = _query([Aggregation("PERCENTILE", "l", arg=p) for p in PS[:6]], group_by=["g"])
    _check_block(oracle, seg, dev, q, pm.execute_segments([dev], q)[0], "one row")
    seg, dev = segs[-1]
    q = _query([Aggregation("PERCENTILE", "d", arg=50.0), Aggregation("COUNT")], Predicate("EQ", "i", [INT_MAX + 1]))
    b = pm.execute_segments([dev], q)[0]
    assert float(b.doubles[0][0]) == float("-inf") and int(b.dict_ids[0][0]) == -1 and int(b.longs[0][0]) == 0
    # scanned on the device, no match: every leaf matches rows, their conjunction none
    absent = next(x for x in range(40) if x not in set(_segment_inv(seg, oracle)[:6].tolist()))
    flt = Filter("AND", [Predicate("RANGE", "rid", [], 0, 5, True, True), Predicate("EQ", "inv", [absent])])
    for col in ("d", "g"):   # one reduction per row / warp-private histograms
        q = _query([Aggregation("PERCENTILE", col, arg=50.0), Aggregation("COUNT")], flt)
        b = pm.execute_segments([dev], q)[0]
        assert b.operator_kind == "AGGREGATION" and b.stats.num_docs_scanned == 0 and int(b.longs[1][0]) == 0
        assert float(b.doubles[0][0]) == float("-inf") and int(b.dict_ids[0][0]) == -1 and int(b.longs[0][0]) == 0


def _segment_inv(seg, oracle):
    from exact_ref import column_values
    return column_values(oracle, seg, "inv", np.arange(seg.num_docs))


def test_refusals(oracle, ctx, pm, segs):
    seg, dev = segs[-1]
    # a FILTER clause on another function next to a PERCENTILE: the whole query goes to the stock operator
    q = _query([Aggregation("COUNT", filter=Predicate("RANGE", "i", [], 1, None, False, True)), Aggregation("PERCENTILE", "i", arg=50.0)])
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], q)
    q = _query([Aggregation("SUM", "i", filter=Predicate("EQ", "g", [1])), Aggregation("PERCENTILE", "l", arg=99.0)], group_by=["g"])
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], q)
    # histograms are not among the reducible device blocks
    import ctypes as C
    for gb in ([], ["g"]):
        q = _query([Aggregation("PERCENTILE", "i", arg=50.0), Aggregation("SUM", "i")], group_by=gb)
        b = pm.execute_segments([dev], q, merge=True, keep_handle=True, defer=False)[0]
        try:
            p, n = C.c_void_p(), C.c_int64()
            for kind in range(4):
                assert ctx.lib.pb200_result_device_buffers(b.handle, kind, C.byref(p), C.byref(n)) == E_UNSUPPORTED
        finally:
            b.release(ctx)
    with pytest.raises(UnsupportedQueryError):   # STRING
        pm.execute_segments([dev], _query([Aggregation("PERCENTILE", "s", arg=50.0)]))
    with pytest.raises(Pb200Error) as e:         # out-of-range percentile
        pm.execute_segments([dev], _query([Aggregation("PERCENTILE", "i", arg=100.5)]))
    assert e.value.code == E_INVALID
    with pytest.raises(Pb200Error) as e:
        pm.execute_segments([dev], _query([Aggregation("PERCENTILE", "i", arg=float("nan"))]))
    assert e.value.code == E_INVALID
    q = _query([Aggregation("PERCENTILE", "i", arg=50.0, filter=Predicate("EQ", "g", [1]))])
    with pytest.raises(UnsupportedQueryError):   # FILTER (WHERE ...) clause
        pm.execute_segments([dev], q)
    q = _query([Aggregation("PERCENTILE", "i", arg=50.0)], group_by=["g"])
    with pytest.raises(UnsupportedQueryError):   # deferred finalize (cross-GPU reduce)
        pm.execute_segments([dev], q, merge=True, keep_handle=True)
    q = _query([Aggregation("PERCENTILE", "rid", arg=50.0)], group_by=["rid"], limit=1 << 20, num_groups_limit=1 << 20)
    with pytest.raises(UnsupportedQueryError):   # 196 609 groups x 196 609 dictIds: above 2^28 histogram entries
        pm.execute_segments([dev], q)
    q = _query([Aggregation("PERCENTILE", "i", arg=50.0)])
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        with pytest.raises(UnsupportedQueryError):   # DataTable bytes of the reference's DoubleArrayList
            pm.to_datatable(dev, q, b)
    finally:
        b.release(ctx)
    # the library without percentiles: pb200h_execute refuses PERCENTILE
    from pinot_b200.plan_maker import _marshal_query
    import ctypes as C
    hq, _keep = _marshal_query(q, False)
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * 1)()
    segs_c = (C.c_void_p * 1)(dev.handle)
    assert ctx.lib.pb200h_execute(ctx.handle, C.byref(hq), segs_c, 1, res, kinds) == E_INVALID


def test_raw_column_without_dictionary_is_refused(oracle, ctx, pm):
    with tuned(ctx, raw_dict_max=0):   # raw INT streamed as 32-bit values: no dictIds
        seg = _segment(oracle, 5_000, 5)
        dev = to_device(ctx, seg)
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([Aggregation("PERCENTILE", "r", arg=50.0)]))
        pm.execute_segments([dev], _query([Aggregation("MAX", "r")]))   # the column itself is fine
    finally:
        dev.destroy()

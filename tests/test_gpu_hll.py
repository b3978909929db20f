"""-m gpu: DISTINCTCOUNTHLL against the independent restatement tests/hll_ref.py over the doc set of tests/filter_ref.py,
as an exact long, on every route.

Columns: INT at INT_MIN and INT_MAX, LONG at +-(2^63 - 1), FLOAT and DOUBLE with -0.0, 0.0, NaN, +-inf and subnormals,
STRING with multi-byte UTF-8, a raw INT column whose dictionary is synthesised at load, and a DATETRUNC derived column.
Routes: aggregation only (an empty filter, 1 to 100 003 rows), the dense, spread, hash and shared-memory tables with the
count carrier on and off under the scan knobs, 17 segments merged over a domain, ORDER BY ... LIMIT with ties, HAVING,
two log2m on one column and a bitset shared with DISTINCTCOUNT, the answer without a scan, the lazily decoded sets, a
loopback 2-rank combine and the refusals."""
import math

import numpy as np
import pytest

import hll_ref
from gpu_util import to_device, tuned
from percentile_ref import group_values
from pinot_b200 import cli, sql
from pinot_b200._lib import UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Predicate, QueryContext, value_key

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
LONG_MAX = (1 << 63) - 1
TYPES = {"i": "INT", "l": "LONG", "f": "FLOAT", "d": "DOUBLE", "s": "STRING", "r": "INT", "g": "INT", "h": "INT", "ts": "LONG"}
COLUMNS = ["i", "l", "f", "d", "s", "r"]
HOUR = 3_600_000
WORDS = ["a", "é", "日本", "€uro", "😀", "ñandú", "x" * 9, "Ω", "", "abc"]


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 3000, size=n) * 7 - 9000).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    lv = rng.integers(-(1 << 62), 1 << 62, size=n).astype(np.int64) // (1 << 50) * (1 << 50)
    lv[rng.integers(0, n, size=max(1, n // 50))] = LONG_MAX
    lv[rng.integers(0, n, size=max(1, n // 50))] = -LONG_MAX
    f = (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32)
    d = rng.integers(-6000, 6000, size=n) / 7.0
    for arr, sub in ((f, np.float32(1e-45)), (d, 5e-324)):
        for k, v in enumerate([-0.0, 0.0, math.nan, math.inf, -math.inf, sub, -sub]):
            arr[rng.integers(0, n, size=max(1, n // 97))] = v
    words = np.array([w.encode("utf-8") for w in WORDS] + [f"u{k}é".encode() for k in range(500)], dtype=object)
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i, "l": lv, "f": f, "d": d,
            "s": np.array(list(words[rng.integers(0, len(words), size=n)])),
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "ts": (1_700_000_000_000 + rng.integers(0, 10 * 24 * HOUR, size=n)).astype(np.int64),
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 300, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"hll{n}_{seed}", cols, raw=["r"])


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def seg(oracle, ctx):
    s = _segment(oracle, 49_157, 3)
    dev = to_device(ctx, s)
    yield s, dev
    dev.destroy()


def _query(aggs, flt=None, group_by=(), order_by=(), limit=100_000, **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), order_by=list(order_by), limit=limit,
                        num_groups_limit=100_000, **kw)


def _plain(v):
    return v.decode() if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def ref_hll(values, log2m, column):
    """hll_ref over the distinct stored values (floats by identity: -0.0 and 0.0 apart, one NaN)."""
    members = {value_key(_plain(v)) for v in values}
    return hll_ref.hll([float(v) if isinstance(v, float) else v for v in members], log2m, TYPES.get(column, "LONG"))


def _key_of(data, group_by, keys_row):
    return tuple(_plain(data.value_of(c, int(keys_row[j]))) for j, c in enumerate(group_by))


def _check(oracle, data, q, b, what, values=None, keys_seg=None):
    """Every DISTINCTCOUNTHLL of block b against hll_ref: the long column exactly, the double column equal to it."""
    got, refs = {}, {}
    rows = 1 if b.num_groups < 0 else b.num_groups
    for a, agg in enumerate(q.aggregations):
        if agg.function != "DISTINCTCOUNTHLL":
            continue
        if agg.column not in refs:
            refs[agg.column] = values if values is not None else group_values(oracle, data, q.filter, q.group_by, agg.column)
        ref = refs[agg.column]
        if q.group_by and not q.order_by and q.having is None:
            assert b.num_groups == len(ref), what
        for g in range(rows):
            key = () if b.num_groups < 0 else _key_of(data[0], q.group_by, b.keys[g]) if keys_seg is None else \
                tuple(_plain(keys_seg.dictionary_value(c, int(b.keys[g][j]))) for j, c in enumerate(q.group_by))
            want = ref_hll(ref.get(key, []), agg.arg, agg.column)
            assert int(b.longs[a][g]) == want, f"{what} a={a} {agg} key={key}: {int(b.longs[a][g])} vs {want}"
            assert float(b.doubles[a][g]) == float(want), what
            got[(a, key)] = want
    return got


def test_aggregation_only(oracle, pm, seg):
    data, dev = seg
    flts = [Predicate("RANGE", "i", [], 10 ** 10, None, True, True), Predicate("RANGE", "i", [], -5000, 9000, True, False),
            Predicate("IN", "g", [1, 4, 7]), Predicate("RANGE", "rid", [], 0, 0, True, True)]
    for fi, flt in enumerate(flts):
        for col in COLUMNS:
            q = _query([Aggregation("DISTINCTCOUNTHLL", col, arg=8), Aggregation("DISTINCTCOUNTHLL", col, arg=4),
                        Aggregation("DISTINCTCOUNTHLL", col, arg=12), Aggregation("COUNT")], flt)
            _check(oracle, [data], q, pm.execute_segments([dev], q)[0], f"f={fi} {col}")
    b = pm.execute_segments([dev], _query([Aggregation("DISTINCTCOUNTHLL", "d", arg=8)], Predicate("RANGE", "rid", [], -5, -1, True, True)))[0]
    assert int(b.longs[0][0]) == 0 and float(b.doubles[0][0]) == 0.0   # an empty S


@pytest.mark.parametrize("n", [1, 2, 31, 33, 1000, 100_003])
def test_row_counts(oracle, ctx, pm, n):
    data = _segment(oracle, n, 17 + n, name=f"hll_n{n}")
    dev = to_device(ctx, data)
    try:
        for gb in ([], ["g"]):
            q = _query([Aggregation("DISTINCTCOUNTHLL", "l", arg=8), Aggregation("DISTINCTCOUNTHLL", "s", arg=10)], group_by=gb,
                       flt=Predicate("RANGE", "i", [], -9000, None, True, True))
            _check(oracle, [data], q, pm.execute_segments([dev], q)[0], f"n={n} {gb}")
    finally:
        dev.destroy()


ROUTES = [("default", {}), ("spread_off", {"table_stride": 1}), ("spread4", {"table_stride": 4}), ("hash", {"dense_max": 1}),
          ("no_smem", {"smem_groups": 0}), ("no_carrier", {"pack_count": 0}), ("warps8", {"warps": 8}),
          ("no_defer", {"defer": 0, "gb_defer": 0}), ("grid1", {"grid": 1}), ("no_skip", {"skip": 0})]


def test_group_by_routes(oracle, ctx, pm, seg):
    data, dev = seg
    shapes = [([Aggregation("DISTINCTCOUNTHLL", "i", arg=8), Aggregation("SUM", "i"), Aggregation("COUNT")], ["g"]),
              ([Aggregation("DISTINCTCOUNTHLL", "d", arg=12), Aggregation("DISTINCTCOUNTHLL", "f", arg=5)], ["h"]),
              ([Aggregation("DISTINCTCOUNTHLL", "s", arg=8), Aggregation("DISTINCTCOUNTHLL", "l", arg=9)], ["g", "h"])]
    for si, (aggs, gb) in enumerate(shapes):
        for flt in (None, Predicate("RANGE", "i", [], -5000, 9000, True, False)):
            q = _query(aggs, flt, group_by=gb)
            first = None
            for name, knobs in ROUTES:
                with tuned(ctx, **knobs):
                    got = _check(oracle, [data], q, pm.execute_segments([dev], q, merge=True)[0], f"shape {si} {name}")
                first = first or got
                assert got == first, f"shape {si}: {name} differs"


def test_two_log2m_and_a_shared_bitset(oracle, pm, seg):
    data, dev = seg
    q = sql.parse("SELECT g, DISTINCTCOUNT(i), DISTINCTCOUNTHLL(i), DISTINCTCOUNTHLL(i, 12), SUM(DISTINCT i) FROM t GROUP BY g LIMIT 100")
    b = pm.execute_segments([dev], q, merge=True, sets=True)[0]
    _check(oracle, [data], q, b, "shared")
    ref = group_values(oracle, [data], None, ["g"], "i")
    for g in range(b.num_groups):   # DISTINCTCOUNT's results are unchanged by the readers of its bitset
        key = _key_of(data, ["g"], b.keys[g])
        assert int(b.longs[0][g]) == len(set(ref[key].tolist()))
        assert list(b.distinct[(0, g)]) == list(b.distinct[(1, g)]) == list(b.distinct[(2, g)]) == list(b.distinct[(3, g)])


def test_order_by_and_having(oracle, pm, seg):
    data, dev = seg
    ref = group_values(oracle, [data], None, ["h"], "i")
    val = {k: ref_hll(v, 8, "i") for k, v in ref.items()}
    for asc in (True, False):
        for limit in (1, 3, 10):
            q = _query([Aggregation("DISTINCTCOUNTHLL", "i", arg=8)], group_by=["h"], order_by=[("distinctcounthll(i,8)", asc)],
                       limit=limit, min_segment_group_trim_size=1)
            b = pm.execute_segments([dev], q)[0]
            want = sorted(ref, key=lambda k: (val[k] if asc else -val[k], k))
            got = [_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)]
            assert got == want[:len(got)] and len(got) >= limit
    # ties: a column constant in the filtered rows estimates 1 everywhere; the keys break the ties
    q = _query([Aggregation("DISTINCTCOUNTHLL", "g", arg=8)], Predicate("EQ", "g", [3]), group_by=["h"],
               order_by=[("distinctcounthll(g,8)", False)], limit=5, min_segment_group_trim_size=1)
    b = pm.execute_segments([dev], q)[0]
    keys = sorted(group_values(oracle, [data], q.filter, ["h"], "g"))
    assert [_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)] == keys[:b.num_groups]
    assert all(int(b.longs[0][g]) == 1 for g in range(b.num_groups))
    q = sql.parse("SELECT h, DISTINCTCOUNTHLL(i) FROM t GROUP BY h HAVING DISTINCTCOUNTHLL(i) > 150 AND DISTINCTCOUNTHLL(i, 6) < 1000 LIMIT 1000")
    b = pm.execute_segments([dev], q, merge=True)[0]
    want = {k for k, v in ref.items() if val[k] > 150 and ref_hll(v, 6, "i") < 1000}
    assert {_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)} == want and want
    _check(oracle, [data], q, b, "having")


def test_non_scan_answer(oracle, pm, seg):
    data, dev = seg
    q = _query([Aggregation("DISTINCTCOUNTHLL", "s", arg=8), Aggregation("DISTINCTCOUNTHLL", "d", arg=11), Aggregation("COUNT")])
    b = pm.execute_segments([dev], q)[0]
    assert b.operator_kind == "NON_SCAN_AGGREGATION"
    assert b.stats.num_docs_scanned == data.num_docs and b.stats.num_entries_scanned_in_filter == 0
    assert b.stats.num_entries_scanned_post_filter == 0 and b.stats.num_total_docs == data.num_docs
    _check(oracle, [data], q, b, "non-scan")
    scanned = pm.execute_segments([dev], q, merge=True)[0]   # the scan gives the same estimates
    assert [int(scanned.longs[a][0]) for a in range(2)] == [int(b.longs[a][0]) for a in range(2)]


def test_sets_are_decoded_lazily_to_the_same_sets(oracle, pm, seg):
    data, dev = seg
    for gb in ([], ["g"]):
        q = _query([Aggregation("DISTINCTCOUNTHLL", "l", arg=8), Aggregation("DISTINCTCOUNT", "d"), Aggregation("DISTINCTCOUNTHLL", "d", arg=8)],
                   Predicate("RANGE", "i", [], -5000, 9000, True, False), group_by=gb)
        merged = pm.execute_segments([dev], q, merge=True)[0]
        assert all(a != 0 for a, _ in merged.distinct)   # nothing asked for the HLL-only set: never decoded
        per_seg = pm.execute_segments([dev], q)[0]   # per-segment blocks read every set through pb200_result_distinct
        ref = group_values(oracle, [data], q.filter, gb, "l")
        for g in range(1 if per_seg.num_groups < 0 else per_seg.num_groups):
            key = () if not gb else _key_of(data, gb, per_seg.keys[g])
            assert {_plain(dev.dictionary_value("l", int(x))) for x in per_seg.distinct[(0, g)]} == set(ref[key].tolist())
            assert list(per_seg.distinct[(1, g)]) == list(per_seg.distinct[(2, g)])
        _check(oracle, [data], q, per_seg, f"per-segment {gb}")


def test_derived_and_raw_columns(oracle, pm, seg):
    data, dev = seg
    q = sql.parse("SELECT g, DISTINCTCOUNTHLL(DATETRUNC('HOUR', ts)) FROM t GROUP BY g LIMIT 100")
    b = pm.execute_segments([dev], q)[0]
    ts = group_values(oracle, [data], None, ["g"], "ts")
    _check(oracle, [data], q, b, "datetrunc", values={k: (v // HOUR) * HOUR for k, v in ts.items()})
    q = _query([Aggregation("DISTINCTCOUNTHLL", "r", arg=7)], group_by=["g"])   # a dictionary synthesised at load
    _check(oracle, [data], q, pm.execute_segments([dev], q)[0], "raw")


def test_seventeen_segments_merged_on_device(oracle, ctx, pm):
    data = [_segment(oracle, 20_000 + 37 * k, 1000 + k, name=f"hll17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = None
    flt = Predicate("RANGE", "i", [], -5000, 9000, True, False)
    try:
        for gb in ([], ["g"]):
            q = _query([Aggregation("DISTINCTCOUNTHLL", "i", arg=8), Aggregation("DISTINCTCOUNTHLL", "d", arg=12),
                        Aggregation("DISTINCTCOUNTHLL", "l", arg=4), Aggregation("DISTINCTCOUNT", "d")], flt, group_by=gb)
            per_seg = cli.final_rows(q, cli.merge_blocks(q, devs, pm.execute_segments(devs, q)))
            if domain is None:
                with pytest.raises(UnsupportedQueryError):   # no shared dictionary: refused
                    pm.execute_segments(devs, q, merge=True)
                domain = DictionaryDomain.build(ctx, devs, ["i", "d", "g", "l"])
                for d in devs:
                    d.bind_domain(domain)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            _check(oracle, data, q, merged, f"merged {gb}")
            on_device = cli.final_rows(q, cli.merge_blocks(q, devs[:1], [merged]))
            assert on_device == per_seg
    finally:
        for d in devs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_refusals(oracle, ctx, pm, seg):
    data, dev = seg
    for log2m in (0, 3, 13, 30):   # 0: the library's default marker; 1..3 and 13..30: the reference's, not accelerated
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([Aggregation("DISTINCTCOUNTHLL", "i", arg=log2m)], group_by=["g"]))
    with pytest.raises(UnsupportedQueryError):   # FILTER (WHERE ...) clause
        pm.execute_segments([dev], _query([Aggregation("DISTINCTCOUNTHLL", "i", arg=8, filter=Predicate("EQ", "g", [1]))]))
    with pytest.raises(UnsupportedQueryError):   # an expression over two columns
        pm.execute_segments([dev], sql.parse("SELECT DISTINCTCOUNTHLL(i + g) FROM t"))
    with tuned(ctx, raw_dict_max=0):   # raw INT streamed as 32-bit values: no dictIds
        raw = to_device(ctx, _segment(oracle, 5_000, 5, name="hll_raw"))
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([raw], _query([Aggregation("DISTINCTCOUNTHLL", "r", arg=8)], group_by=["g"]))
    finally:
        raw.destroy()
    # a STRING dictionary with an entry that is not valid UTF-8
    n = 3_000
    cols = {"g": np.zeros(n, dtype=np.int32), "b": np.array([b"ok", b"\xff\xfe"] * (n // 2))}
    bad = oracle.build_segment("hll_badutf8", cols)
    bdev = to_device(ctx, bad)
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([bdev], _query([Aggregation("DISTINCTCOUNTHLL", "b", arg=8)], Predicate("EQ", "g", [0])))
    finally:
        bdev.destroy()
    # DataTable bytes: the reference serializes registers this library does not restate
    q = _query([Aggregation("DISTINCTCOUNTHLL", "i", arg=8)], group_by=["g"])
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.to_datatable(dev, q, b)
    finally:
        ctx.lib.pb200_result_free(b.handle)


@pytest.mark.parametrize("world", [2])
def test_loopback_combine(oracle, world):
    """execute_and_combine with `world` ranks on one GPU (tests/loopback_dist.py): the host set-union route, the root's
    estimates equal to hll_ref over every rank's docs, ORDER BY ... LIMIT included."""
    from loopback_dist import run_ranks, values
    from pinot_b200.distributed import execute_and_combine, global_domain
    hosts = [[_segment(oracle, 3_000 + 101 * r + 7 * i, 500 + 10 * r + i, name=f"hlll{r}_{i}") for i in range(1 + r % 2)]
             for r in range(world)]
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [[to_device(c, h) for h in hs] for c, hs in zip(ctxs, hosts)]
    doms = []
    try:
        doms = values(run_ranks(world, lambda dist: global_domain(ctxs[dist.get_rank()], devs[dist.get_rank()],
                                                                  ["h", "g", "i", "l"], dist)))
        everything = [h for hs in hosts for h in hs]
        for text in ("SELECT h, DISTINCTCOUNTHLL(l), DISTINCTCOUNT(i) FROM t GROUP BY h ORDER BY DISTINCTCOUNTHLL(l) DESC LIMIT 5",
                     "SELECT g, DISTINCTCOUNTHLL(i, 12) FROM t WHERE i > -5000 GROUP BY g",
                     "SELECT DISTINCTCOUNTHLL(l), DISTINCTCOUNTHLL(i, 5) FROM t"):
            q = sql.parse(text, num_groups_limit=1_000_000)
            got = values(run_ranks(world, lambda dist: execute_and_combine(
                B200PlanMaker(ctxs[dist.get_rank()]), devs[dist.get_rank()], sql.parse(text, num_groups_limit=1_000_000), dist)))
            root = got[0]
            assert all(g is None for g in got[1:])
            if q.order_by:
                ref = group_values(oracle, everything, q.filter, q.group_by, "l")
                order = sorted(ref, key=lambda k: (-ref_hll(ref[k], 8, "l"), k))
                keys = [tuple(_plain(devs[0][0].dictionary_value(c, int(root.keys[g][j]))) for j, c in enumerate(q.group_by))
                        for g in range(root.num_groups)]
                assert keys == order[:len(keys)] and len(keys) >= q.limit, text
            _check(oracle, everything, q, root, f"world {world}: {text}", keys_seg=devs[0][0])
    finally:
        for ds in devs:
            for d in ds:
                d.destroy()
        for dom in doms:
            dom.release()
        for c in ctxs:
            c.close()

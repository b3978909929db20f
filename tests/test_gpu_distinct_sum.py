"""-m gpu: DISTINCTSUM / DISTINCTAVG (and COUNT / SUM / AVG(DISTINCT col)) against a Fraction reference over the doc set of
tests/filter_ref.py, bit for bit, on every route.

Columns: INT at INT_MIN and INT_MAX, LONG near +-2^62, grid FLOAT and DOUBLE (eighths), a raw INT column whose dictionary
is synthesised at load, and a DATETRUNC derived column.  Routes: aggregation only (an empty filter included), the dense
table, the spread dense table, the hash table, the scan knobs, 17 segments merged over a domain, ORDER BY ... LIMIT with
ties, HAVING, one bitset shared with DISTINCTCOUNT.  Every refusal."""
import math
from fractions import Fraction

import numpy as np
import pytest

from gpu_util import to_device, tuned
from percentile_ref import group_values
from pinot_b200 import cli, sql
from pinot_b200._lib import UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Predicate, QueryContext, value_key

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
COLUMNS = ["i", "lp", "ln", "f", "d", "r"]
HOUR = 3_600_000


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 3000, size=n) * 7 - 9000).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i,
            "lp": ((1 << 62) + (rng.integers(0, 3000, size=n) << 28) + 7).astype(np.int64),
            "ln": (-(1 << 62) - (rng.integers(0, 3000, size=n) << 28) - 7).astype(np.int64),
            "f": (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32),
            "d": rng.integers(-6000, 6000, size=n) / 8.0 + 1e9,
            "d3": rng.integers(-600000, 600000, size=n) / 100.0,        # 0.01-steps: refused
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "ts": (1_700_000_000_000 + rng.integers(0, 10 * 24 * HOUR, size=n)).astype(np.int64),
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 300, size=n).astype(np.int32),
            "s": np.array([b"a", b"ab", b"b"])[rng.integers(0, 3, size=n)]}
    return oracle.build_segment(name or f"dsum{n}_{seed}", cols, raw=["r"])


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


def distinct_values(values):
    """The distinct stored values: integers exactly, floats by identity (ValueKey: -0.0 and 0.0 apart, one NaN)."""
    return {value_key(v) for v in (x.item() if hasattr(x, "item") else x for x in values)}


def ref_final(fn, values):
    """The exact reference: the distinct stored values summed as Fractions, rounded once."""
    s = distinct_values(values)
    if fn == "DISTINCTCOUNT":
        return float(len(s))
    if not s:
        return 0.0 if fn == "DISTINCTSUM" else -math.inf
    total = sum((Fraction(v) for v in s), Fraction(0))
    return float(total / len(s) if fn == "DISTINCTAVG" else total)


def _key_of(data, group_by, keys_row):
    out = []
    for j, c in enumerate(group_by):
        v = data.value_of(c, int(keys_row[j]))
        out.append(v.decode() if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v))
    return tuple(out)


def _plain(v):
    return v.decode() if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _bits(x):
    return np.float64(x).tobytes()


def _check(oracle, data, q, b, what, values=None, keys_seg=None):
    """Every distinct-set function of block b against the reference; returns {(a, key): value bytes}.  keys_seg: the
    (domain-bound) segment that decodes the block's key ids, else data[0]'s own dictionaries."""
    got, refs = {}, {}
    rows = 1 if b.num_groups < 0 else b.num_groups
    for a, agg in enumerate(q.aggregations):
        if agg.function not in ("DISTINCTCOUNT", "DISTINCTSUM", "DISTINCTAVG"):
            continue
        if agg.column not in refs:
            refs[agg.column] = values if values is not None else group_values(oracle, data, q.filter, q.group_by, agg.column)
        ref = refs[agg.column]
        if q.group_by and not q.order_by and q.having is None:
            assert b.num_groups == len(ref), what
        for g in range(rows):
            key = () if b.num_groups < 0 else _key_of(data[0], q.group_by, b.keys[g]) if keys_seg is None else \
                tuple(_plain(keys_seg.dictionary_value(c, int(b.keys[g][j]))) for j, c in enumerate(q.group_by))
            want = ref_final(agg.function, ref.get(key, []))
            v = float(b.doubles[a][g]) if agg.function != "DISTINCTCOUNT" else float(b.longs[a][g])
            assert _bits(v) == _bits(want), f"{what} a={a} {agg} key={key}: {v!r} vs {want!r}"
            assert int(b.longs[a][g]) == len(distinct_values(ref.get(key, []))), what
            assert len(b.distinct[(a, g)]) == int(b.longs[a][g]), what
            got[(a, key)] = _bits(v)
    return got


def test_aggregation_only(oracle, pm, seg):
    data, dev = seg
    flts = [None, Predicate("RANGE", "i", [], 10 ** 10, None, True, True), Predicate("RANGE", "i", [], -5000, 9000, True, False),
            Predicate("IN", "g", [1, 4, 7])]
    for fi, flt in enumerate(flts):
        for col in COLUMNS:
            q = _query([Aggregation("DISTINCTSUM", col), Aggregation("DISTINCTAVG", col), Aggregation("COUNT")], flt)
            b = pm.execute_segments([dev], q)[0]
            _check(oracle, [data], q, b, f"f={fi} {col}")
    # an empty filter: 0.0 and -inf
    b = pm.execute_segments([dev], _query([Aggregation("DISTINCTSUM", "i"), Aggregation("DISTINCTAVG", "d")],
                                          Predicate("RANGE", "rid", [], -5, -1, True, True)))[0]
    assert _bits(float(b.doubles[0][0])) == _bits(0.0) and float(b.doubles[1][0]) == -math.inf


ROUTES = [("default", {}), ("spread_off", {"table_stride": 1}), ("spread4", {"table_stride": 4}), ("hash", {"dense_max": 1}),
          ("warps8", {"warps": 8}), ("no_defer", {"defer": 0, "gb_defer": 0}), ("grid1", {"grid": 1}),
          ("no_skip", {"skip": 0})]


def test_group_by_routes_bit_identical(oracle, ctx, pm, seg):
    data, dev = seg
    shapes = [([Aggregation("DISTINCTSUM", "i"), Aggregation("DISTINCTAVG", "i"), Aggregation("SUM", "i")], ["g"]),
              ([Aggregation("DISTINCTAVG", "d"), Aggregation("DISTINCTCOUNT", "d"), Aggregation("DISTINCTSUM", "d")], ["h"]),
              ([Aggregation("DISTINCTSUM", "lp"), Aggregation("DISTINCTAVG", "ln"), Aggregation("COUNT")], ["g", "s"]),
              ([Aggregation("DISTINCTSUM", "f"), Aggregation("DISTINCTAVG", "r")], ["h", "g"])]
    for si, (aggs, gb) in enumerate(shapes):
        for flt in (None, Predicate("RANGE", "i", [], -5000, 9000, True, False)):
            q = _query(aggs, flt, group_by=gb)
            first = None
            for name, knobs in ROUTES:
                with tuned(ctx, **knobs):
                    got = _check(oracle, [data], q, pm.execute_segments([dev], q)[0], f"shape {si} {name}")
                first = first or got
                assert got == first, f"shape {si}: {name} differs"


def test_sharing_with_distinctcount(oracle, pm, seg):
    data, dev = seg
    q = sql.parse("SELECT g, DISTINCTCOUNT(i), SUM(DISTINCT i), AVG(DISTINCT i), COUNT(DISTINCT i) FROM t GROUP BY g LIMIT 100")
    b = pm.execute_segments([dev], q)[0]
    _check(oracle, [data], q, b, "shared")
    for g in range(b.num_groups):
        assert list(b.distinct[(0, g)]) == list(b.distinct[(1, g)]) == list(b.distinct[(2, g)])


def test_order_by_and_having(oracle, pm, seg):
    data, dev = seg
    ref = group_values(oracle, [data], None, ["h"], "i")
    val = {k: ref_final("DISTINCTSUM", v) for k, v in ref.items()}
    for asc in (True, False):
        for limit in (1, 3, 10):
            q = _query([Aggregation("DISTINCTSUM", "i")], group_by=["h"], order_by=[("distinctsum(i)", asc)], limit=limit,
                       min_segment_group_trim_size=1)
            b = pm.execute_segments([dev], q)[0]
            want = sorted(ref, key=lambda k: (val[k] if asc else -val[k], k))
            got = [_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)]
            assert got == want[:len(got)] and len(got) >= limit
    # ties: DISTINCTAVG of a column constant in the filtered rows, keys break them
    q = _query([Aggregation("DISTINCTAVG", "g")], Predicate("EQ", "g", [3]), group_by=["h"], order_by=[("distinctavg(g)", False)],
               limit=5, min_segment_group_trim_size=1)
    b = pm.execute_segments([dev], q)[0]
    keys = sorted(group_values(oracle, [data], q.filter, ["h"], "g"))
    assert [_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)] == keys[:b.num_groups]
    # HAVING on the device (one merged result)
    text = "SELECT h, SUM(DISTINCT i) FROM t GROUP BY h HAVING AVG(DISTINCT i) > 0 AND distinctsum(i) < 1000000000000 LIMIT 1000"
    q = sql.parse(text)
    b = pm.execute_segments([dev], q, merge=True)[0]
    want = {k for k, v in ref.items() if ref_final("DISTINCTAVG", v) > 0 and val[k] < 1e12}
    assert {_key_of(data, ["h"], b.keys[g]) for g in range(b.num_groups)} == want
    _check(oracle, [data], q, b, "having")


def test_seventeen_segments_merged_on_device(oracle, ctx, pm):
    data = [_segment(oracle, 20_000 + 37 * k, 1000 + k, name=f"dsum17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = None
    flt = Predicate("RANGE", "i", [], -5000, 9000, True, False)
    try:
        for gb in ([], ["g"]):
            # lp / ln: LONG members beyond 2^53, which the per-segment route merges as Python integers
            q = _query([Aggregation("DISTINCTSUM", "i"), Aggregation("DISTINCTAVG", "d"), Aggregation("DISTINCTCOUNT", "d"),
                        Aggregation("DISTINCTSUM", "lp"), Aggregation("DISTINCTAVG", "ln")], flt, group_by=gb)
            per_seg = cli.final_rows(q, cli.merge_blocks(q, devs, pm.execute_segments(devs, q)))
            if domain is None:
                with pytest.raises(UnsupportedQueryError):   # no shared dictionary: refused
                    pm.execute_segments(devs, q, merge=True)
                domain = DictionaryDomain.build(ctx, devs, ["i", "d", "g", "lp", "ln"])
                for d in devs:
                    d.bind_domain(domain)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            _check(oracle, data, q, merged, f"merged {gb}")
            on_device = cli.final_rows(q, cli.merge_blocks(q, devs[:1], [merged]))
            assert [[_bits(x) if isinstance(x, float) else x for x in r] for r in on_device] == \
                   [[_bits(x) if isinstance(x, float) else x for x in r] for r in per_seg]
    finally:
        for d in devs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_derived_column(oracle, pm, seg):
    data, dev = seg
    q = sql.parse("SELECT g, SUM(DISTINCT DATETRUNC('HOUR', ts)), AVG(DISTINCT DATETRUNC('HOUR', ts)) FROM t GROUP BY g LIMIT 100")
    b = pm.execute_segments([dev], q)[0]
    ts = group_values(oracle, [data], None, ["g"], "ts")
    _check(oracle, [data], q, b, "datetrunc", values={k: (v // HOUR) * HOUR for k, v in ts.items()})


def test_refusals(oracle, ctx, pm, seg):
    data, dev = seg
    for col in ("s", "d3"):   # STRING, 0.01-steps
        for fn in ("DISTINCTSUM", "DISTINCTAVG"):
            with pytest.raises(UnsupportedQueryError):
                pm.execute_segments([dev], _query([Aggregation(fn, col)]))
    with pytest.raises(UnsupportedQueryError):   # FILTER (WHERE ...) clause
        pm.execute_segments([dev], _query([Aggregation("DISTINCTSUM", "i", filter=Predicate("EQ", "g", [1]))]))
    with tuned(ctx, raw_dict_max=0):   # raw INT streamed as 32-bit values: no dictIds
        raw = to_device(ctx, _segment(oracle, 5_000, 5, name="dsum_raw"))
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([raw], _query([Aggregation("DISTINCTSUM", "r")]))
    finally:
        raw.destroy()


@pytest.mark.parametrize("world", [2, 3])
def test_loopback_combine(oracle, world):
    """execute_and_combine with `world` ranks on one GPU (tests/loopback_dist.py): each rank has its own context,
    segments with their own dictionaries and a global domain; the functions take the host set-union route and the root's
    rows equal the Fraction reference over every rank's docs, LONG members beyond 2^53 and ORDER BY ... LIMIT included."""
    from loopback_dist import run_ranks, values
    from pinot_b200.distributed import execute_and_combine, global_domain
    hosts = [[_segment(oracle, 3_000 + 101 * r + 7 * i, 500 + 10 * r + i, name=f"dsl{r}_{i}") for i in range(1 + r % 2)]
             for r in range(world)]
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [[to_device(c, h) for h in hs] for c, hs in zip(ctxs, hosts)]
    doms = []
    try:
        doms = values(run_ranks(world, lambda dist: global_domain(ctxs[dist.get_rank()], devs[dist.get_rank()],
                                                                  ["h", "g", "i", "lp", "d"], dist)))
        everything = [h for hs in hosts for h in hs]
        for text in ("SELECT h, SUM(DISTINCT lp), AVG(DISTINCT lp), COUNT(DISTINCT i) FROM t GROUP BY h "
                     "ORDER BY SUM(DISTINCT lp) DESC LIMIT 5",
                     "SELECT g, DISTINCTAVG(d), DISTINCTSUM(i) FROM t WHERE i > -5000 GROUP BY g",
                     "SELECT DISTINCTSUM(lp), DISTINCTAVG(i) FROM t"):
            q = sql.parse(text, num_groups_limit=1_000_000)
            got = values(run_ranks(world, lambda dist: execute_and_combine(
                B200PlanMaker(ctxs[dist.get_rank()]), devs[dist.get_rank()], sql.parse(text, num_groups_limit=1_000_000), dist)))
            root = got[0]
            assert all(g is None for g in got[1:])
            if q.order_by:
                ref = group_values(oracle, everything, q.filter, q.group_by, "lp")
                order = sorted(ref, key=lambda k: (-ref_final("DISTINCTSUM", ref[k]), k))
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

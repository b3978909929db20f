"""-m gpu: aggregations with FILTER (WHERE ...) clauses through the product (pinot_b200/csrc/host/filtered_agg.cpp: one
device submission per distinct clause over main AND clause, aligned by group key) against the oracle's restatement of
AggregationFunctionUtils.buildFilteredAggregationInfos / FilteredGroupByOperator (tests/test_oracle_filtered.py pins that
restatement on the reference's own FilteredAggregationsTest queries)."""
import re

import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, UnsupportedQueryError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


QUERIES = [
    # the reference's FilteredAggregationsTest shapes
    "SELECT SUM(v) FILTER(WHERE v > 100) FROM t WHERE v < 400",
    "SELECT COUNT(*) FILTER(WHERE k = 4) FROM t",
    "SELECT SUM(v) FILTER(WHERE raw <= 1) FROM t WHERE v > 1",                                         # clause matches nothing
    "SELECT AVG(v) FILTER(WHERE raw > -1000000) FROM t",                                               # clause matches everything
    "SELECT MIN(v) FILTER(WHERE raw > 900), MAX(v) FILTER(WHERE v > 450) FROM t",
    "SELECT SUM(v) FILTER(WHERE v > 3), SUM(v) FILTER(WHERE v < 4), MIN(w) FILTER(WHERE w > 5000000000) FROM t WHERE v > -300",
    "SELECT SUM(v) FILTER(WHERE k IN (1, 3, 5)), SUM(raw), MAX(v), COUNT(*) FROM t WHERE raw > 5",
    "SELECT DISTINCTCOUNT(k) FILTER(WHERE v > 0), DISTINCTCOUNT(k), COUNT(*) FILTER(WHERE v > 0) FROM t WHERE j != 2",
    # GROUP BY: every group of the main filter exists, functions a clause never saw keep their defaults
    "SELECT SUM(v) FILTER(WHERE v > 100) FROM t WHERE v < 400 GROUP BY k",
    "SELECT SUM(v) FILTER(WHERE v > 100 AND v < 300) FROM t GROUP BY j",
    "SELECT SUM(v) FILTER(WHERE j = 1), COUNT(*) FILTER(WHERE j = 1), MIN(w) FILTER(WHERE j = 5), MAX(v), COUNT(*) FROM t WHERE v > -400 GROUP BY k",
    "SELECT AVG(v) FILTER(WHERE k < 3), AVG(v) FILTER(WHERE k >= 3), AVG(v) FROM t GROUP BY j, k",
    "SELECT COUNT(*) FILTER(WHERE v > 490), SUM(f) FILTER(WHERE v > 490) FROM t WHERE k != 0 GROUP BY k, j",   # sparse clause
    "SELECT DISTINCTCOUNT(v) FILTER(WHERE j < 3), COUNT(*) FROM t WHERE v > 0 GROUP BY j",
    "SELECT MAX(raw) FILTER(WHERE raw < 0), SUM(v) FILTER(WHERE raw < 0) FROM t GROUP BY raw_k",              # raw key + raw clause
]


def _segment(oracle, n, seed):
    rng = np.random.default_rng(seed)
    return oracle.build_segment(f"flt{seed}", {
        "k": rng.integers(0, 9, size=n).astype(np.int32), "j": rng.integers(0, 7, size=n).astype(np.int32),
        "v": rng.integers(-500, 500, size=n).astype(np.int32),
        "w": rng.integers(0, 30, size=n).astype(np.int64) * 1_000_000_007,
        "f": (rng.integers(0, 300, size=n) / 8.0).astype(np.float64),
        "raw": rng.integers(-1000, 1000, size=n).astype(np.int32), "raw_k": rng.integers(0, 40, size=n).astype(np.int32) * 5},
        raw=["raw", "raw_k"], inverted=["j"])


@pytest.mark.parametrize("n", [1, 4096, 50_003])
def test_filtered_aggregations_equal_oracle(oracle, ctx, pm, n):
    seg = _segment(oracle, n, 7 + n)
    dev = to_device(ctx, seg)
    try:
        for text in QUERIES:
            check_query(oracle, pm, seg, dev, sql.parse(text), f"n={n}: {text}")
    finally:
        dev.destroy()


def test_filtered_aggregations_over_merged_segments(oracle, ctx, pm):
    """Device-side combine per clause (PB200_Q_MERGE_SEGMENTS), then the alignment by key: three segments with different
    dictionaries bound to one domain == the oracle-side merge by value of the per-segment oracle results."""
    from pinot_b200.plan_maker import DictionaryDomain
    from reduce_util import combine
    segs = [_segment(oracle, 20_000 + 31 * i, 300 + i) for i in range(3)]
    devs = [to_device(ctx, s) for s in segs]
    dom = None
    try:
        dom = DictionaryDomain.build(ctx, devs, ["k", "j", "w"])
        for d in devs:
            d.bind_domain(dom)
        for text in ("SELECT SUM(v) FILTER(WHERE j = 1), COUNT(*) FILTER(WHERE j = 1), MIN(w) FILTER(WHERE j = 5), MAX(v), COUNT(*) FROM t WHERE v > -400 GROUP BY k",
                     "SELECT COUNT(*) FILTER(WHERE v > 490), SUM(f) FILTER(WHERE v > 490) FROM t WHERE k != 0 GROUP BY k, j",
                     "SELECT SUM(v) FILTER(WHERE v > 3), SUM(v) FILTER(WHERE v < 4), COUNT(*) FROM t WHERE v > -300"):
            q = sql.parse(text)
            block = pm.execute_segments(devs, q, merge=True)[0]
            want = combine([a.function for a in q.aggregations], [oracle_table(s, q, oracle.execute(s, q)) for s in segs])
            assert_tables_equal(q, gpu_table(segs[0], q, block, devs[0]), want, "merged: " + text)
            check_exact(oracle, segs, q, gpu_table(segs[0], q, block, devs[0]), "merged: " + text)
            assert block.stats.num_docs_scanned == sum(oracle.execute(s, q).stats[0] for s in segs), text
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()


def test_filtered_result_as_datatable(oracle, ctx, pm):
    """The aligned result is an ordinary result: its DataTableImplV4 bytes read back by the test-side reader."""
    from datatable_util import parse
    seg = _segment(oracle, 10_000, 99)
    dev = to_device(ctx, seg)
    try:
        q = sql.parse("SELECT SUM(v) FILTER(WHERE j = 1), COUNT(*) FROM t WHERE v > 0 GROUP BY k")
        block = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
        table = parse(pm.to_datatable(dev, q, block))
        want = oracle_table(seg, q, oracle.execute(seg, q))
        got = {(row[0],): [float(row[1]), int(row[2])] for row in table["rows"]}
        assert got == {k: [float(v[0]), int(v[1])] for k, v in want.items()}
        block.release(ctx)
    finally:
        dev.destroy()


def test_refusal_does_not_depend_on_function_order(oracle, ctx, pm):
    """A query with several functions that do not run next to FILTER clauses, or have no DataTable type, is refused for
    the same one whichever comes first in the query."""
    seg = _segment(oracle, 4096, 5)
    dev = to_device(ctx, seg)
    try:
        for fns, family in ((["VARPOP(v)", "PERCENTILE(v, 50)"], "PERCENTILE"),
                            (["DISTINCTCOUNTHLL(k)", "DISTINCTSUM(v)", "STDDEVSAMP(f)"], "VAR/STDDEV")):
            for order in (fns, fns[::-1]):
                q = sql.parse(f"SELECT {', '.join(order)}, COUNT(*) FILTER(WHERE j = 1) FROM t")
                with pytest.raises(UnsupportedQueryError, match=re.escape(f"{family} in a query with FILTER (WHERE ...) clauses")):
                    pm.execute_segments([dev], q)
        for order in (["VARPOP(v)", "DISTINCTCOUNTHLL(k)"], ["DISTINCTCOUNTHLL(k)", "VARPOP(v)"]):
            q = sql.parse(f"SELECT {', '.join(order)} FROM t")
            block = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
            with pytest.raises(UnsupportedQueryError, match="DISTINCTCOUNTHLL is not written as a server DataTable"):
                pm.to_datatable(dev, q, block)
            block.release(ctx)
    finally:
        dev.destroy()

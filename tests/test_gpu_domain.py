"""Merging segments whose dictionaries DIFFER: refused without a common id space, by value once bound to a domain.

The reference merges per-segment group-by / aggregation results through VALUES (GroupByCombineOperator.java:130-146 ->
IndexedTable.upsert, AggregationFunction.merge).  The device-side combine (PB200_Q_MERGE_SEGMENTS) and the cross-GPU
table reduce work on dictId-indexed state instead, which is only the same thing when every contributor shares one
dictionary: pb200_domain_* builds the sorted union of the segments' dictionaries and re-encodes bound segments into it.
Oracle side: each segment through the CPU oracle with its OWN dictionaries, merged by value with tests/reduce_util.combine.
"""
import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain, UnsupportedQueryError
from reduce_util import combine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def device_table(dev, q, block):
    """Value-space table of a block whose ids are decoded through the SEGMENT HANDLE (domain dictionary when bound)."""
    rows = 1 if block.num_groups < 0 else block.num_groups
    out = {}
    for g in range(rows):
        key = () if block.num_groups < 0 else tuple(dev.dictionary_value(c, int(block.keys[g, j])) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            if agg.function == "COUNT":
                vals.append(int(block.longs[a][g]))
            elif agg.function == "AVG":
                vals.append((float(block.doubles[a][g]), int(block.longs[a][g])))
            elif agg.function == "DISTINCTCOUNT":
                vals.append(frozenset(dev.dictionary_value(agg.column, int(d)) for d in block.distinct[(a, g)]))
            else:
                vals.append(float(block.doubles[a][g]))
        out[key] = vals
    return out


def _segments(oracle, rng, sizes):
    """Per-segment dictionaries: different value subsets (different and EQUAL cardinalities), every type, an inverted
    index column, a sorted column."""
    segs = []
    for i, n in enumerate(sizes):
        pool_k = rng.choice(500, size=40 + 7 * (i % 3), replace=False).astype(np.int32) * 3 - 100       # INT keys
        pool_l = rng.choice(10_000, size=25, replace=False).astype(np.int64) * 1_000_003                 # LONG, equal cardinality everywhere
        pool_s = np.array([b"alpha", b"be", b"gamma_long_entry", b"d", b"epsilon", b"zeta" * (1 + i % 2)])[rng.choice(6, size=3 + i % 3, replace=False)]
        pool_f = (rng.choice(300, size=20 + i, replace=False) / 8.0).astype(np.float64)
        pool_g = (rng.choice(64, size=12, replace=False).astype(np.float32) - 30.0) * 0.25               # negative floats too
        cols = {
            "k": pool_k[rng.integers(0, len(pool_k), size=n)],
            "l": pool_l[rng.integers(0, len(pool_l), size=n)],
            "s": pool_s[rng.integers(0, len(pool_s), size=n)],
            "f": pool_f[rng.integers(0, len(pool_f), size=n)],
            "g": pool_g[rng.integers(0, len(pool_g), size=n)],
            "v": rng.integers(-1000, 1000, size=n).astype(np.int32),
            "t": np.sort(rng.integers(i, i + 4, size=n)).astype(np.int32) * 10,                          # sorted, shifted per segment
        }
        segs.append(oracle.build_segment(f"dom{i}", cols, inverted=["k", "s"]))
    return segs


QUERIES = [
    "SELECT COUNT(*), SUM(v), MIN(k), MAX(k) FROM t WHERE v > -500",
    "SELECT MIN(l), MAX(l), MIN(f), MAX(g), DISTINCTCOUNT(k), DISTINCTCOUNT(s) FROM t WHERE v < 900",
    "SELECT COUNT(*), SUM(v) FROM t WHERE v > -900 GROUP BY k",
    "SELECT COUNT(*), SUM(v), MAX(l), MIN(f) FROM t GROUP BY s, k",
    "SELECT SUM(f), AVG(g), MAX(g) FROM t WHERE k > 50 GROUP BY l",
    "SELECT COUNT(*), MAX(v) FROM t WHERE k IN (-100, -97, 2, 50, 299, 1001) GROUP BY s",       # inverted index, ids absent in some segments
    "SELECT COUNT(*), SUM(v) FROM t WHERE s != 'be' AND k BETWEEN 0 AND 700 GROUP BY t",         # inverted NOT + scan range + sorted key
    "SELECT COUNT(*), DISTINCTCOUNT(l) FROM t WHERE t >= 20 GROUP BY g",                         # sorted-index filter, per-group bitsets
    "SELECT COUNT(*), MIN(k), MAX(l) FROM t WHERE l > 5000000000 OR f < 10.0 GROUP BY k",
]


def test_merge_refused_when_dictionaries_differ(oracle, ctx, pm):
    rng = np.random.default_rng(11)
    # equal cardinality, different values: round 1 only compared cardinalities and merged garbage
    a = oracle.build_segment("a", {"k": (rng.integers(0, 50, size=5000) * 2).astype(np.int32), "v": rng.integers(0, 9, size=5000).astype(np.int32)})
    b = oracle.build_segment("b", {"k": (rng.integers(0, 50, size=5000) * 2 + 1).astype(np.int32), "v": rng.integers(0, 9, size=5000).astype(np.int32)})
    assert a.column("k").cardinality == b.column("k").cardinality
    da, db = to_device(ctx, a), to_device(ctx, b)
    try:
        for text in ("SELECT SUM(v) FROM t GROUP BY k", "SELECT MIN(k), MAX(k) FROM t", "SELECT DISTINCTCOUNT(k) FROM t",
                     "SELECT COUNT(*), DISTINCTCOUNT(k) FROM t GROUP BY v"):
            with pytest.raises(UnsupportedQueryError):
                pm.execute_segments([da, db], sql.parse(text), merge=True)
        # functions that never leave value space may still be merged
        q = sql.parse("SELECT COUNT(*), SUM(k), AVG(v) FROM t WHERE k > 10")
        got = pm.execute_segments([da, db], q, merge=True)[0]
        want = combine([x.function for x in q.aggregations], [oracle_table(s, q, oracle.execute(s, q)) for s in (a, b)])
        assert_tables_equal(q, device_table(da, q, got), want, "value-space merge")
        check_exact(oracle, [a, b], q, device_table(da, q, got), "value-space merge")
    finally:
        da.destroy()
        db.destroy()


@pytest.mark.parametrize("sizes", [[3000, 1, 8193, 40_001], [20_000, 20_000]])
def test_domain_merge_equals_oracle_merge_by_value(oracle, ctx, pm, sizes):
    rng = np.random.default_rng(500 + len(sizes))
    segs = _segments(oracle, rng, sizes)
    devs = [to_device(ctx, s) for s in segs]
    dom = None
    try:
        unbound = [{c: d.column_info(c) for c in ("k", "l", "s", "f", "g", "t")} for d in devs]
        dom = DictionaryDomain.build(ctx, devs, ["k", "l", "s", "f", "g", "t", "v"])
        for c in ("k", "l", "f", "g", "t"):   # union == np.unique over the segments' dictionaries
            want = np.unique(np.concatenate([s.column(c).dict_values for s in segs]))
            assert dom.info(c)["cardinality"] == len(want), c
            be = {"k": ">i4", "t": ">i4", "l": ">i8", "f": ">f8", "g": ">f4"}[c]
            assert np.array_equal(np.frombuffer(dom.dictionary_bytes(c).tobytes(), dtype=be), want.astype(be)), c
        assert dom.info("s")["cardinality"] == len({v for s in segs for v in s.column("s").dict_values.tolist()})
        for d in devs:
            d.bind_domain(dom)
        for d, s, ub in zip(devs, segs, unbound):
            for c in ("k", "l", "s", "f", "g", "t"):
                assert d.column_info(c)["cardinality"] == dom.info(c)["cardinality"]
                ids = d.local_ids(c)
                assert len(ids) == ub[c]["cardinality"] and np.all(np.diff(ids) > 0)
                # the ids that occur decode to exactly the segment's own dictionary
                assert [d.dictionary_value(c, int(i)) for i in ids] == [s.value_of(c, j) for j in range(len(ids))], c
        for text in QUERIES:
            q = sql.parse(text, num_groups_limit=1_000_000)
            fns = [a.function for a in q.aggregations]
            want_blocks = [oracle_table(s, q, oracle.execute(s, q)) for s in segs]
            # a bound segment alone still answers like the reference (ids decode through the domain)
            for d, w, blk in zip(devs, want_blocks, pm.execute_segments(devs, q)):
                assert_tables_equal(q, device_table(d, q, blk), w, "bound, per segment: " + text)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            assert_tables_equal(q, device_table(devs[0], q, merged), combine(fns, want_blocks), "merged by value: " + text)
            check_exact(oracle, segs, q, device_table(devs[0], q, merged), "merged by value: " + text)
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()


def test_bind_rejects_a_domain_that_misses_values(oracle, ctx, pm):
    rng = np.random.default_rng(3)
    a = oracle.build_segment("a", {"k": rng.integers(0, 30, size=2000).astype(np.int32)})
    b = oracle.build_segment("b", {"k": rng.integers(20, 60, size=2000).astype(np.int32)})
    da, db = to_device(ctx, a), to_device(ctx, b)
    dom = DictionaryDomain.build(ctx, [da], ["k"])
    try:
        from pinot_b200._lib import Pb200Error
        with pytest.raises(Pb200Error):
            db.bind_domain(dom)
        # the failed bind left the segment untouched
        q = sql.parse("SELECT COUNT(*), MIN(k), MAX(k) FROM t WHERE k > 25")
        got = pm.execute_segments([db], q)[0]
        assert_tables_equal(q, device_table(db, q, got), oracle_table(b, q, oracle.execute(b, q)), "after failed bind")
        da.bind_domain(dom)
        with pytest.raises(Pb200Error):
            da.bind_domain(dom)   # already bound
    finally:
        da.destroy()
        db.destroy()
        dom.release()

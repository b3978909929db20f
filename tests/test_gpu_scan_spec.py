"""-m gpu: the group-by kernel specialised for the shared-table shape (pb200_scan.cuh SPEC) against the generic kernel and
the references.  Every shape the planner admits runs twice, with pb200_tuning_set("spec", 1) and ("spec", 0); the two
results must be bit-identical (group keys, sums, counts, execution statistics, count-carrier outcome) and equal the
oracle and the exact reference (tests/exact_ref.py)."""
import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker
from reduce_util import combine

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def assert_same_blocks(a, b, what):
    assert a.num_groups == b.num_groups, what
    assert np.array_equal(a.keys, b.keys), what
    for x, y in zip(a.longs, b.longs):
        assert np.array_equal(x, y), what
    for x, y in zip(a.doubles, b.doubles):
        assert np.array_equal(x, y, equal_nan=True), what
    assert a.stats == b.stats, what
    assert a.count_carrier == b.count_carrier, what


def both_routes(ctx, run):
    """run() on the specialised route (the default) and on the generic one; both results."""
    spec = run()
    try:
        ctx.set_tuning("spec", 0)
        generic = run()
    finally:
        ctx.set_tuning("spec", 1)
    return spec, generic


def check_one(oracle, ctx, pm, seg, dev, text, what):
    q = sql.parse(text, num_groups_limit=1_000_000)
    spec, generic = both_routes(ctx, lambda: pm.make_segment_plan_node(dev, q).run().next_block())
    assert_same_blocks(spec, generic, f"{what}: {text}")
    check_query(oracle, pm, seg, dev, q, f"{what}: {text}")   # the specialised route (the default) against the references
    return spec


def make_seg(oracle, rng, name, n, keys=1000, extremes=False):
    k = rng.integers(0, keys, size=n).astype(np.int32)
    v = rng.integers(-1_000_000, 1_000_000, size=n).astype(np.int32)
    if extremes:
        v[rng.random(n) < 0.3] = INT_MIN
        v[rng.random(n) < 0.3] = INT_MAX
    return oracle.build_segment(name, {
        "k": k, "k2": rng.integers(0, 7, size=n).astype(np.int32), "v": v,
        "v2": rng.integers(-50, 50, size=n).astype(np.int32), "w": rng.integers(0, 40, size=n).astype(np.int32),
        "x": rng.integers(0, 300, size=n).astype(np.int32)})


SHAPES = [
    "SELECT SUM(v), COUNT(*) FROM t WHERE w > 3 GROUP BY k",              # the headline's shape
    "SELECT COUNT(*) FROM t WHERE w < 30 GROUP BY k",                     # COUNT only
    "SELECT SUM(v) FROM t WHERE w BETWEEN 5 AND 20 GROUP BY k",           # SUM only (count as the group marker)
    "SELECT SUM(v), SUM(v2), COUNT(*) FROM t WHERE w != 7 GROUP BY k",    # two sums
    "SELECT AVG(v2), COUNT(*) FROM t GROUP BY k",                         # no filter
    "SELECT SUM(v), COUNT(*) FROM t WHERE w > 3 AND x < 200 GROUP BY k",  # two range leaves
    "SELECT SUM(v), COUNT(*) FROM t WHERE x BETWEEN 1 AND 298 AND w >= 39 GROUP BY k, k2",  # two key columns
]


@pytest.mark.parametrize("n", [1, 31, 33, 1023, 1025, 8193, 65_537, 196_609])
def test_segment_sizes_with_ragged_tails(oracle, ctx, pm, n):
    rng = np.random.default_rng(n)
    seg = make_seg(oracle, rng, f"n{n}", n)
    dev = to_device(ctx, seg)
    try:
        for text in SHAPES:
            check_one(oracle, ctx, pm, seg, dev, text, f"n={n}")
    finally:
        dev.destroy()


def test_comparison_shapes_at_both_dictionary_edges(oracle, ctx, pm):
    rng = np.random.default_rng(40)
    seg = make_seg(oracle, rng, "edges", 70_001)
    dev = to_device(ctx, seg)
    try:
        for cond in ("w < 1", "w < 39", "w <= 39", "w > 0", "w > 38", "w >= 0", "w = 0", "w = 39", "w != 0", "w != 39",
                     "w BETWEEN 1 AND 38", "w BETWEEN 0 AND 0", "w BETWEEN 39 AND 39", "w > 39", "w < 0",
                     "x > 298 AND w < 1", "x < 1 AND w > 38"):
            check_one(oracle, ctx, pm, seg, dev, f"SELECT SUM(v), COUNT(*) FROM t WHERE {cond} GROUP BY k", "edges")
    finally:
        dev.destroy()


@pytest.mark.parametrize("keys", [1000, 10_000], ids=["w6_replicated", "w8_large"])
def test_values_at_the_int_extremes(oracle, ctx, pm, keys):
    rng = np.random.default_rng(keys)
    seg = make_seg(oracle, rng, f"ext{keys}", 150_000, keys=keys, extremes=True)
    dev = to_device(ctx, seg)
    try:
        for text in SHAPES[:4]:
            check_one(oracle, ctx, pm, seg, dev, text, f"extremes, {keys} keys")
    finally:
        dev.destroy()


def test_forced_carrier_overflow_falls_back_on_both_routes(oracle, ctx, pm):
    rng = np.random.default_rng(60)
    n = 300_000
    seg = oracle.build_segment("few", {"k": rng.integers(0, 4, size=n).astype(np.int32),
                                       "v": rng.integers(0, 100, size=n).astype(np.int32),
                                       "w": rng.integers(0, 10, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        ctx.set_tuning("pack_shift", 60)   # count field = 4 bits: every CTA's entries overflow it
        block = check_one(oracle, ctx, pm, seg, dev, "SELECT SUM(v), COUNT(*) FROM t WHERE w > 2 GROUP BY k", "overflow")
        assert not block.count_carrier
    finally:
        ctx.set_tuning("pack_shift", 0)
        dev.destroy()


@pytest.mark.parametrize("keys", [1000, 10_000], ids=["w6_replicated", "w8_large"])
def test_17_segments_merged_and_per_segment(oracle, ctx, pm, keys):
    """17 segments: two launch chunks; the merged result flushes each CTA's table once per launch, the per-segment results
    at every segment change."""
    rng = np.random.default_rng(17 + keys)

    def seg(i, n):
        k = np.concatenate([np.arange(keys), rng.integers(0, keys, size=n - keys)]).astype(np.int32)
        rng.shuffle(k)   # every segment holds every key: one dictionary, so the segments merge by value
        return oracle.build_segment(f"s{keys}_{i}", {"k": k, "v": rng.integers(-1000, 100_000, size=n).astype(np.int32),
                                                   "v2": rng.integers(INT_MIN, INT_MAX, size=n, endpoint=True).astype(np.int32),
                                                   "w": rng.integers(0, 10, size=n).astype(np.int32)})
    segs = [seg(i, keys + 1 + 3_071 * i) for i in range(17)]
    devs = [to_device(ctx, s) for s in segs]
    try:
        for text in ("SELECT SUM(v), COUNT(*) FROM t WHERE w > 0 GROUP BY k",
                     "SELECT SUM(v), SUM(v2) FROM t WHERE w < 9 GROUP BY k"):
            q = sql.parse(text, num_groups_limit=1_000_000)
            fns = [a.function for a in q.aggregations]
            want = [oracle_table(s, q, oracle.execute(s, q)) for s in segs]
            per_seg = both_routes(ctx, lambda: pm.execute_segments(devs, q))
            for s, a, b, w in zip(segs, per_seg[0], per_seg[1], want):
                assert_same_blocks(a, b, f"per segment: {text}")
                assert_tables_equal(q, gpu_table(s, q, a), w, f"per segment: {text}")
            merged = both_routes(ctx, lambda: pm.execute_segments(devs, q, merge=True))
            assert len(merged[0]) == 1 and len(merged[1]) == 1
            assert_same_blocks(merged[0][0], merged[1][0], f"merged: {text}")
            got = gpu_table(segs[0], q, merged[0][0])
            assert_tables_equal(q, got, combine(fns, want), f"merged: {text}")
            check_exact(oracle, segs, q, got, f"merged: {text}")
    finally:
        for d in devs:
            d.destroy()

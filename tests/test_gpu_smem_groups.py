"""-m gpu: GROUP BY tables kept in a CTA-private shared-memory table (thousands of groups: one 8-warp CTA per SM, the count
carrier inside 8-byte entries, one flush per merged launch) against the oracle, and the same shapes with the global-table
route forced through pb200_tuning_set("smem_groups", 0)."""
import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker
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


@pytest.fixture
def smem_groups(ctx, request):
    ctx.set_tuning("smem_groups", request.param)
    yield request.param
    ctx.set_tuning("smem_groups", 1)


@pytest.mark.parametrize("smem_groups", [1, 0], indirect=True, ids=["shared", "global"])
def test_carrier_shapes_on_both_routes(oracle, ctx, pm, smem_groups):
    """5 000 keys: shared-memory table by default, global table with the route switched off; both carry the counts."""
    rng = np.random.default_rng(64)
    n = 90_000
    seg = oracle.build_segment("carrier", {
        "k": rng.integers(0, 5000, size=n).astype(np.int32),
        "big": rng.integers(-2_000_000_000, 2_000_000_000, size=n).astype(np.int32),
        "small": rng.integers(-50, 50, size=n).astype(np.int32),
        "w": rng.integers(0, 40, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        for text in ("SELECT SUM(big), COUNT(*) FROM t WHERE w > 3 GROUP BY k",
                     "SELECT AVG(small), SUM(big) FROM t GROUP BY k",
                     "SELECT SUM(small) FROM t WHERE w < 30 GROUP BY k",             # count only as the group-exists marker
                     "SELECT COUNT(*), SUM(small), SUM(big) FROM t WHERE w != 7 GROUP BY k"):
            _, block = check_query(oracle, pm, seg, dev, sql.parse(text, num_groups_limit=1_000_000), f"smem={smem_groups}: {text}")
            assert block.count_carrier, text
        ctx.set_tuning("pack_count", 0)   # no carrier: a count array in the shared table (12-byte entries)
        try:
            text = "SELECT SUM(small), COUNT(*) FROM t WHERE w > 3 GROUP BY k"
            _, block = check_query(oracle, pm, seg, dev, sql.parse(text, num_groups_limit=1_000_000), f"smem={smem_groups}, no carrier")
            assert not block.count_carrier
        finally:
            ctx.set_tuning("pack_count", 1)
    finally:
        dev.destroy()


@pytest.mark.parametrize("smem_groups", [1, 0], indirect=True, ids=["shared", "global"])
def test_10000_groups_merged_segments_with_ragged_tails(oracle, ctx, pm, smem_groups):
    """The headline's key space over several segments whose lengths are not multiples of a tile: the merged result (one
    flush of each CTA's table at exit) and the per-segment results (a flush at every segment change) equal the oracle."""
    rng = np.random.default_rng(10_000)

    def seg(i, n):
        k = np.concatenate([np.arange(10_000), rng.integers(0, 10_000, size=n - 10_000)]).astype(np.int32)
        rng.shuffle(k)   # every segment holds every key: one dictionary, so the segments merge by value
        return oracle.build_segment(f"m{i}", {"k": k,
                                              "v": rng.integers(-1000, 100_000, size=n).astype(np.int32),
                                              "w": rng.integers(0, 10, size=n).astype(np.int32)})
    segs = [seg(i, n) for i, n in enumerate([100_003, 10_001, 65_537, 24_575, 50_000, 8_193 + 10_000])]
    devs = [to_device(ctx, s) for s in segs]
    try:
        for text in ("SELECT SUM(v), COUNT(*) FROM t WHERE w > 0 GROUP BY k",
                     "SELECT COUNT(*), AVG(v) FROM t WHERE w < 9 GROUP BY k"):
            q = sql.parse(text, num_groups_limit=1_000_000)
            fns = [a.function for a in q.aggregations]
            want = [oracle_table(s, q, oracle.execute(s, q)) for s in segs]
            for s, b, w in zip(segs, pm.execute_segments(devs, q), want):
                assert_tables_equal(q, gpu_table(s, q, b), w, f"smem={smem_groups} per segment: {text}")
            merged = pm.execute_segments(devs, q, merge=True)
            assert len(merged) == 1 and merged[0].count_carrier, text
            assert_tables_equal(q, gpu_table(segs[0], q, merged[0]), combine(fns, want), f"smem={smem_groups} merged: {text}")
            check_exact(oracle, segs, q, gpu_table(segs[0], q, merged[0]), f"smem={smem_groups} merged: {text}")
    finally:
        for d in devs:
            d.destroy()


def test_carrier_count_overflow_inside_a_cta_table_falls_back(oracle, ctx, pm):
    """A few groups and many rows: with a 4-bit count field every CTA's shared entries overflow it.  The flushed table
    equals what global REDs would build, so the overflow is detected and the query reruns without the carrier."""
    rng = np.random.default_rng(4)
    n = 300_000
    seg = oracle.build_segment("few", {"k": rng.integers(0, 4, size=n).astype(np.int32),
                                       "v": rng.integers(0, 100, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    q = sql.parse("SELECT SUM(v), COUNT(*) FROM t GROUP BY k")
    try:
        _, block = check_query(oracle, pm, seg, dev, q, "carrier")
        assert block.count_carrier
        ctx.set_tuning("pack_shift", 60)   # count field = 4 bits: 16 rows per group
        _, block = check_query(oracle, pm, seg, dev, q, "count field overflow")
        assert not block.count_carrier
        merged = pm.execute_segments([dev, dev, dev], q, merge=True)[0]
        assert not merged.count_carrier
        assert_tables_equal(q, gpu_table(seg, q, merged), combine(["SUM", "COUNT"], [oracle_table(seg, q, oracle.execute(seg, q))] * 3), "merged overflow")
        check_exact(oracle, [seg] * 3, q, gpu_table(seg, q, merged), "merged overflow")
    finally:
        ctx.set_tuning("pack_shift", 0)
        dev.destroy()

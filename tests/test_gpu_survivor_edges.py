"""-m gpu: the scan kernel's survivor paths (pinot_b200/csrc/pb200_scan.cuh) on segments whose survivors are designed
slice by slice (tests/survivor_plan.py), held to the oracle and the exact reference (gpu_util.check_query).

Each slice has a chosen survivor count S at the queue's batch edges (0 .. 5, 31 .. 33, 127 .. 129, ..., 1023, 1024), packed,
spread over the lanes or in one lane, with decoy rows that pass the first filter leaf only (per-lane counts on both sides
of sparse_max before the second leaf).  Under `grid` 1 every non-zero S is followed in the same warp's next tile by a
non-zero S, by S = 0, by a bitmap-skipped slice, by the ragged last slice and by the segment's end, so the pipelined last
batch of the GROUP BY queue and the deferred gathers of the aggregation-only kernel are drained by each of them.  The
routes -- the shared table specialised or not, the 8-warp table, the global dense table, the hash table, without the
count carrier or the pipeline, every aggregation-only variant -- are forced with tuning knobs; which plan each one gets is
pinned by tests/test_survivor_plan_cpu.py.  Submissions of 24 segments (two launch chunks) run per segment and merged.
The hash table is held at exactly numGroupsLimit groups and one more, and with probe chains that wrap past its end."""
import pytest

import survivor_plan as sp
from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device, tuned
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, UnsupportedQueryError

pytestmark = pytest.mark.gpu

LIMIT = 1_000_000


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def _load(oracle, ctx, planned, name):
    seg = oracle.build_segment(name, planned.columns, inverted=["inv"], raw=["r"])
    with tuned(ctx, raw_dict_max=0):   # "r" stays a raw 32-bit column
        return seg, to_device(ctx, seg)


@pytest.fixture(scope="module")
def sets(oracle, ctx):
    """{"w6" | "w8" | "big": [(host segment, device segment)]}."""
    out = {}
    plans = {"w6": sp.hand_over_plans(6), "w8": sp.hand_over_plans(8),
             "big": [sp.long_plan("big0", 73, 77), sp.long_plan("big1", 72, 0, start=11)]}
    for name, ps in plans.items():
        out[name] = [_load(oracle, ctx, sp.build_columns(p, 7000 + k), p.name) for k, p in enumerate(ps)]
    yield out
    for segs in out.values():
        for _, dev in segs:
            dev.destroy()


# ---------------------------------------------------------------------------------------------------- every route, every segment
@pytest.mark.parametrize("rid, knobs, segset, queries", sp.ROUTES, ids=[r[0] for r in sp.ROUTES])
def test_route(oracle, ctx, pm, sets, rid, knobs, segset, queries):
    with tuned(ctx, **knobs):
        for text in queries:
            q = sql.parse(text, num_groups_limit=LIMIT)
            for seg, dev in sets[segset]:
                check_query(oracle, pm, seg, dev, q, f"{rid} {seg.name}: {text}")


# ---------------------------------------------------------------------------------------------------- submissions
SUBMISSION_KNOBS = [{}, {"grid": 1}, {"grid": 7}, {"grid": 1, "spec": 0}, {"grid": 1, "smem_groups": 0},
                    {"grid": 1, "pack_count": 0}, {"grid": 1, "warps": 8}]


@pytest.mark.parametrize("knobs", SUBMISSION_KNOBS, ids=[",".join(f"{k}={v}" for k, v in kn.items()) or "defaults"
                                                         for kn in SUBMISSION_KNOBS])
def test_per_segment_and_merged_submissions(oracle, ctx, pm, sets, knobs):
    """All 24 segments of a set in one submission (two launch chunks): per segment, a flush (and a shared-table flush) at
    every segment change -- under grid 1 the same CTA carries its warps' pending batches into the next segment; merged,
    one table for the submission, flushed once at exit.  Sizes: 1024 k + 1, 1024 k - 1, 12 x 1024, 16 x 1024, ..."""
    segset = "w8" if knobs.get("warps") == 8 else "w6"
    hs = [s for s, _ in sets[segset]]
    ds = [d for _, d in sets[segset]]
    with tuned(ctx, **knobs):
        for text in (sp.GB_SPEC, sp.GB_INV, sp.MIX4, sp.GB_KB, sp.AGG_SUM, sp.AGG_MIX):
            q = sql.parse(text, num_groups_limit=LIMIT)
            what = f"{knobs}: {text}"
            for s, b in zip(hs, pm.execute_segments(ds, q)):
                got = gpu_table(s, q, b)
                assert_tables_equal(q, got, oracle_table(s, q, oracle.execute(s, q)), "per segment " + what)
                check_exact(oracle, [s], q, got, "per segment " + what)
            if q.is_group_by and text != sp.MIX4:   # MIN / MAX: see MERGED_K70 below
                merged = pm.execute_segments(ds, q, merge=True)
                assert len(merged) == 1
                check_exact(oracle, hs, q, gpu_table(hs[0], q, merged[0]), "merged " + what)


# merged MIN / MAX compare dictIds, so they need one dictionary per column across the segments (or a domain): the merged
# cases aggregate sums, over values whose dictionaries differ from segment to segment
MERGED_K70 = f"SELECT SUM(v), SUM(f), AVG(l) FROM t WHERE {sp.F} GROUP BY k70"
MERGED_HASH = f"SELECT SUM(v), COUNT(*), SUM(f) FROM t WHERE {sp.F} GROUP BY ha, hb"


def test_merged_70000_keys(oracle, ctx, pm, sets):
    """Two long segments (73 805 and 73 728 rows) merged into one global dense table of 70 000 keys."""
    hs = [s for s, _ in sets["big"]]
    ds = [d for _, d in sets["big"]]
    for knobs in ({}, {"grid": 1}):
        with tuned(ctx, **knobs):
            for text in (sp.GB_K70, MERGED_K70):
                q = sql.parse(text, num_groups_limit=LIMIT)
                check_exact(oracle, hs, q, gpu_table(hs[0], q, pm.execute_segments(ds, q, merge=True)[0]), f"{knobs}: {text}")


# ---------------------------------------------------------------------------------------------------- the hash table
L = 300
CARD = 2048
HASH_QUERIES = [f"SELECT SUM(v), COUNT(*), MIN(v) FROM t WHERE {sp.F} GROUP BY ha, hb",
                f"SELECT SUM(f), MAX(v) FROM t WHERE {sp.F} GROUP BY ha, hb"]
HASH_KNOBS = [{"dense_max": 1}, {"dense_max": 1, "grid": 1}, {"dense_max": 1, "gb_defer": 0}]
HASH_IDS = ["defaults", "grid1", "no_gb_defer"]


@pytest.fixture(scope="module")
def pairs():
    """48 key pairs whose home slot is among the last 16 of the table (numGroupsLimit L: 2^16 slots), then more."""
    return sp.distinct_pairs(sp.keys_at_table_end(CARD, CARD, L, 48), CARD, L + 1)


@pytest.fixture(scope="module")
def hash_segs(oracle, ctx, pairs):
    """name -> (host, device): "exact" (L groups, the last two new in the pipelined batch), "over" (L + 1), "wrap" (only
    the 48 wrapping pairs), and "a" / "b" / "b_over" whose group sets overlap: a u b = L, a u b_over = L + 1."""
    specs = {"exact": pairs[:L], "over": pairs[:L + 1], "wrap": pairs[:48], "a": pairs[:L - 5], "b": pairs[5:L],
             "b_over": pairs[5:L + 1]}
    out = {name: _load(oracle, ctx, sp.hash_segment_columns(p, CARD, 100 + k), f"h_{name}")
           for k, (name, p) in enumerate(specs.items())}
    yield out
    for _, dev in out.values():
        dev.destroy()


def _refused_by_the_table(fn):
    with pytest.raises(UnsupportedQueryError) as e:
        fn()
    # the kernel's own cut-off (hash_slot stops admitting keys at numGroupsLimit), not the count after the scan
    assert "hash table saw more groups" in str(e.value), str(e.value)


@pytest.mark.parametrize("knobs", HASH_KNOBS, ids=HASH_IDS)
def test_hash_groups_limit_on_one_segment(oracle, ctx, pm, hash_segs, knobs):
    """Exactly L groups are answered exactly; L + 1 are refused (PB200_E_LIMIT), never truncated.  The L-th and
    (L + 1)-th new keys are the last two rows of the last slice: the pipelined last batch."""
    with tuned(ctx, **knobs):
        for text in HASH_QUERIES:
            q = sql.parse(text, num_groups_limit=L)
            seg, dev = hash_segs["exact"]
            _, block = check_query(oracle, pm, seg, dev, q, f"{knobs} exact: {text}")
            assert block.num_groups == L
            seg, dev = hash_segs["over"]
            _refused_by_the_table(lambda: pm.execute_segments([dev], q))


@pytest.mark.parametrize("knobs", HASH_KNOBS, ids=HASH_IDS)
def test_hash_groups_limit_merged(oracle, ctx, pm, hash_segs, knobs):
    """Merged over two segments whose group sets overlap, each under L: the union decides."""
    (ha, da), (hb, db), (_, dbo) = hash_segs["a"], hash_segs["b"], hash_segs["b_over"]
    with tuned(ctx, **knobs):
        q = sql.parse(MERGED_HASH, num_groups_limit=L)
        block = pm.execute_segments([da, db], q, merge=True)[0]
        assert block.num_groups == L
        check_exact(oracle, [ha, hb], q, gpu_table(ha, q, block), f"{knobs} merged")
        _refused_by_the_table(lambda: pm.execute_segments([da, dbo], q, merge=True))


@pytest.mark.parametrize("knobs", HASH_KNOBS, ids=HASH_IDS)
def test_hash_probe_chains_wrap_past_the_table_end(oracle, ctx, pm, hash_segs, knobs):
    """48 keys whose home slots are the table's last 16: their probe chains run past h_mask to slot 0 and back into the
    extraction."""
    seg, dev = hash_segs["wrap"]
    with tuned(ctx, **knobs):
        for text in HASH_QUERIES:
            _, block = check_query(oracle, pm, seg, dev, sql.parse(text, num_groups_limit=L), f"{knobs} wrap: {text}")
            assert block.num_groups == 48

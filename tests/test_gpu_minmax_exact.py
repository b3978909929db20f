"""-m gpu: MIN / MAX / DISTINCTCOUNT against the exact reference (tests/exact_ref.py) on every route of the scan kernel, with
values at the extremes of their types:

* INT {INT_MIN, -1, 0, 1, INT_MAX} as a dictionary column "i" and as a raw column "r" (loaded with raw_dict_max 0, so it
  stays a raw 32-bit stream, VAL_RAW_I32).  Groups k % 4 == 0 hold INT_MAX only, k % 4 == 1 INT_MIN only: a raw MAX at
  INT_MAX and a raw MIN at INT_MAX sit on the u32 values that mean "no row" for a dictionary entry.
* LONG at INT64_MIN / INT64_MAX and 2^53 - 1, 2^53, 2^53 + 1 (rounded to double to nearest); FLOAT / DOUBLE at +-inf,
  +-max and the smallest subnormals.  NaN and -0.0: tests/test_gpu_float_edges.py.
* DISTINCTCOUNT columns of cardinality exactly 2^5 and 2^5 + 1 (dictIds 0 and card - 1 present) over INT, LONG, FLOAT,
  DOUBLE and STRING: the group-by bitset has 1 and 2 words per group.
* "e" with "k": `k = 0 AND e = 1` matches rows of the large segments only.  The host cannot prove it empty (each leaf
  matches), so the kernel runs and the small segments come back without a row.

Each route is forced with pb200_tuning_set (tuned() restores the knob).  Every docstring names the host rule in
pinot_b200/csrc/pb200_plan.cpp (plan_scan) that picks the route.  Segment sizes cover ragged tails and the tile edges
of both CTA widths (6 x 1024 and 8 x 1024 rows).  For dictionary columns the C-ABI dictId of every MIN / MAX must be the
id of the reference's value."""
import numpy as np
import pytest

from exact_ref import check_exact, reference
from gpu_util import check_query, gpu_table, to_device, tuned
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 33, 6_145, 8_191, 20_000]
G = 24
BIG = 8_000       # segments of at least this many rows match `k = 0 AND e = 1`

FIVE = np.array([INT_MIN, -1, 0, 1, INT_MAX], dtype=np.int32)
LONGS = np.array([INT64_MIN, INT64_MAX, (1 << 53) - 1, 1 << 53, (1 << 53) + 1, -(1 << 53) - 1, 0], dtype=np.int64)
FLOATS = np.array([-np.inf, np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                   np.finfo(np.float32).smallest_subnormal, -np.finfo(np.float32).smallest_subnormal, 1.5], dtype=np.float32)
DOUBLES = np.array([-np.inf, np.inf, np.finfo(np.float64).max, -np.finfo(np.float64).max, 5e-324, -5e-324, 0.1],
                   dtype=np.float64)
DISTINCT = {"c32": np.arange(32, dtype=np.int32) * 7 - 100,
            "c33": np.arange(33, dtype=np.int32) * 65_537 + INT_MIN,
            "l32": np.linspace(-2.0 ** 62, 2.0 ** 62, 32).astype(np.int64),
            "f33": (np.arange(33, dtype=np.float32) - 16.0) * np.float32(0.375),
            "d32": np.arange(32, dtype=np.float64) * 1e300 - 1.5e301,
            "s33": np.array([f"v{i:03d}".encode() for i in range(33)])}

AGG_QUERIES = ["SELECT MIN(r), MAX(r), MIN(i), MAX(i), COUNT(*) FROM t WHERE w < 7",
               "SELECT MIN(l), MAX(l), MIN(f), MAX(f), MIN(d), MAX(d) FROM t",
               "SELECT MIN(r), MAX(r), MIN(i), MAX(i) FROM t WHERE i BETWEEN -1 AND 1",     # filtered-out rows hold the extremes
               "SELECT MIN(r), MAX(r), MAX(i), MAX(l), MIN(d) FROM t WHERE k = 0 AND e = 1",   # INT_MAX only, or no row
               "SELECT DISTINCTCOUNT(c32), DISTINCTCOUNT(c33), DISTINCTCOUNT(l32), DISTINCTCOUNT(f33), DISTINCTCOUNT(d32), "
               "DISTINCTCOUNT(s33) FROM t WHERE w < 7"]
GB_QUERIES = ["SELECT MIN(r), MAX(r) FROM t WHERE w < 7 GROUP BY k",          # both pipelined; the raw tables are no marker
              "SELECT MAX(r) FROM t GROUP BY k",
              "SELECT SUM(r), MIN(r) FROM t GROUP BY k",                      # a raw sum carries no count
              "SELECT MIN(i), MAX(i), MIN(l), MAX(f), MIN(d) FROM t WHERE w != 3 GROUP BY k",   # 2 pipelined, 3 at once
              "SELECT MAX(i), MIN(l), MAX(r), MIN(r) FROM t WHERE w < 9 GROUP BY k",  # the raw ones at once
              "SELECT DISTINCTCOUNT(c32), DISTINCTCOUNT(c33), DISTINCTCOUNT(s33), DISTINCTCOUNT(f33) FROM t WHERE w < 7 GROUP BY k",
              "SELECT DISTINCTCOUNT(l32), DISTINCTCOUNT(d32), MAX(r), MIN(i) FROM t WHERE k = 0 AND e = 1 GROUP BY k"]


def _segment(oracle, n, seed, pools=None):
    """`pools` {column: values} replaces the value pool of a column (the domain test's per-segment dictionaries)."""
    pools = {"i": FIVE, "l": LONGS, "f": FLOATS, "d": DOUBLES, **DISTINCT, **(pools or {})}
    rng = np.random.default_rng(seed)
    k = rng.integers(0, G, size=n)
    k[:min(n, G)] = np.arange(min(n, G))
    k[G:G + 33] = 2 + np.arange(len(k[G:G + 33])) % 2   # rows whose "i" keeps its pool value
    cols = {"k": k.astype(np.int32), "w": rng.integers(0, 10, size=n).astype(np.int32)}
    e = rng.integers(0, 2, size=n)
    if n < BIG:
        e = np.where(k == 0, 0, e)
    e[1:3] = [0, 1][:len(e[1:3])]   # k = 1, 2: both values in every dictionary of "e" (n >= 3)
    cols["e"] = e.astype(np.int32)
    for c, pool in pools.items():
        v = pool[rng.integers(0, len(pool), size=n)]
        if n >= G + len(pool):   # every value of the pool occurs: segments share one dictionary
            v[G:G + len(pool)] = pool
        cols[c] = v
    i = cols["i"]
    i[k % 4 == 0] = INT_MAX
    i[k % 4 == 1] = INT_MIN
    cols["r"] = i.copy()
    return oracle.build_segment(f"mm{n}_{seed}", cols, raw=["r"])


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
    """{rows: (host segment, device segment)}; "r" stays raw (raw_dict_max 0)."""
    out = {}
    with tuned(ctx, raw_dict_max=0):
        for n in SIZES:
            seg = _segment(oracle, n, n)
            out[n] = (seg, to_device(ctx, seg))
    yield out
    for _, dev in out.values():
        dev.destroy()


def check_ids(q, block, table, ref, value_of, raw, what):
    """block.dict_ids of every dictionary MIN / MAX: -1 for no row, else the dictId of the reference's (exact, unrounded)
    value -- +-inf too, when the column stores it.  `table` is the block's value-space table (gpu_table: one key per
    block row, in row order).  Only an aggregation-only result can lack a row here (no query has a FILTER clause)."""
    no_row = block.num_groups < 0 and block.stats.num_docs_scanned == 0
    for g, key in enumerate(table):
        for a, agg in enumerate(q.aggregations):
            if agg.function not in ("MIN", "MAX") or agg.column in raw:
                continue
            want, i = ref[key][a], int(block.dict_ids[a][g])
            if no_row:
                assert i == -1 and want == (float("inf") if agg.function == "MIN" else float("-inf")), (what, key, i, want)
            else:
                assert i >= 0 and value_of(agg.column, i) == want, (what, agg.function, agg.column, key, i, want)


def sweep(oracle, pm, segs, queries, what):
    """check_query (oracle parity + exact reference) and check_ids of every query over every segment."""
    for n, (seg, dev) in segs.items():
        for text in queries:
            q = sql.parse(text, num_groups_limit=1_000_000)
            _, block = check_query(oracle, pm, seg, dev, q, f"{what} n={n}: {text}")
            if any(a.function in ("MIN", "MAX") for a in q.aggregations):
                check_ids(q, block, gpu_table(seg, q, block, dev), reference(oracle, [seg], q), seg.value_of, ("r",),
                          f"{what} n={n}: {text}")


# ---------------------------------------------------------------------------------------------------- aggregation only
@pytest.mark.parametrize("knobs", [{}, {"sparse_max_agg": 32}, {"grid": 1}, {"grid": 7}],
                         ids=["dense", "per_row", "grid_1", "grid_7"])
def test_aggregation_only(oracle, ctx, pm, segs, knobs):
    """Defaults: dictionary MIN / MAX on the left-aligned form (MinMaxLeft, then >> sh), raw INT unpacked (unpack_group,
    then ^ 0x80000000), DISTINCTCOUNT bitsets; one warp_min / warp_max + atomicMin / atomicMax per warp (flush) and the
    host decode in pb200_execute.  `sparse_max_agg` 32: q.sparse_max_agg >= every warp's survivor count (wmax2), so every
    surviving row goes through process_row.  `grid` 1 / 7: every tile in one CTA, or tiles spread over 7 CTAs (more
    flushes per segment, fewer per CTA)."""
    with tuned(ctx, **knobs):
        sweep(oracle, pm, segs, AGG_QUERIES, str(knobs))


@pytest.mark.parametrize("defer", [1, 0], ids=["w8_agg", "w8_agg_nodefer"])
def test_aggregation_only_eight_warps(oracle, ctx, pm, segs, defer):
    """`warps` 8: cw = tune.warps, 8192-row tiles.  ScanVariant's DEFER is `!(cw == 8 && !tune.defer)`: with `defer` 0
    the w8_agg_nodefer kernel runs."""
    with tuned(ctx, warps=8, defer=defer):
        sweep(oracle, pm, segs, AGG_QUERIES, f"w8 defer={defer}")


# ---------------------------------------------------------------------------------------------------- group-by
@pytest.mark.parametrize("knobs", [{}, {"gb_defer": 0}, {"always_count": 1}],
                         ids=["pipelined_last_batch", "no_pipeline", "always_count"])
def test_group_by_global_table(oracle, ctx, pm, segs, knobs):
    """MIN / MAX rule out the shared-memory table, so every table is global.  Defaults: `tune.gb_defer` pipelines up to
    two MIN / MAX per query (drain_gb compares against an entry read one tile earlier); the others test, then
    atomicMin / atomicMax at once.  `gb_defer` 0: all at once.  Without COUNT / AVG a dictionary MIN / MAX table marks the
    groups that exist (exists_min / exists_max), a raw INT one cannot (seen flag); `always_count` 1 keeps the count
    array instead."""
    with tuned(ctx, **knobs):
        sweep(oracle, pm, segs, GB_QUERIES, str(knobs))


def test_group_by_hash_table(oracle, ctx, pm, segs):
    """`dense_max` 1: the key space exceeds d.dense_max, so the table is hashed; its keys mark the groups, the MIN / MAX /
    bitset tables are indexed by slot."""
    with tuned(ctx, dense_max=1):
        sweep(oracle, pm, segs, GB_QUERIES, "hash")


@pytest.mark.parametrize("stride", [1, 16])
def test_group_by_spread_table(oracle, ctx, pm, segs, stride):
    """`table_stride` 1 / 16: a dense global table without DISTINCTCOUNT holds raw key k at k * tune.table_stride, and the
    extraction skips the entries between (1: not spread)."""
    with tuned(ctx, table_stride=stride):
        sweep(oracle, pm, segs, [t for t in GB_QUERIES if "DISTINCTCOUNT" not in t], f"stride {stride}")


# ---------------------------------------------------------------------------------------------------- submissions
@pytest.mark.parametrize("gb_defer", [1, 0], ids=["pipelined_last_batch", "no_pipeline"])
def test_merged_and_per_segment_submissions(oracle, ctx, pm, segs, gb_defer):
    """execute_segments(..., merge=True) over segments that share their dictionaries (every pool value occurs in each):
    one AggAccum / one dense table for all of them; 18 segments exceed kMaxLaunchSegs (16), so the submission takes two
    launches.  merge=False: one result per segment from the same launches."""
    chosen = [(s, d) for n, (s, d) in segs.items() if n >= G + 33]
    hs, ds = [s for s, _ in chosen] * 6, [d for _, d in chosen] * 6
    with tuned(ctx, gb_defer=gb_defer):
        for text in AGG_QUERIES + GB_QUERIES:
            q = sql.parse(text, num_groups_limit=1_000_000)
            for s, b in zip(hs, pm.execute_segments(ds[:len(chosen)], q)):
                table = gpu_table(s, q, b)
                check_ids(q, b, table, check_exact(oracle, [s], q, table, "per segment: " + text), s.value_of, ("r",),
                          "per segment: " + text)
            merged = pm.execute_segments(ds, q, merge=True)
            assert len(merged) == 1
            table = gpu_table(hs[0], q, merged[0])
            ref = check_exact(oracle, hs, q, table, f"merged x{len(ds)}: {text}")
            check_ids(q, merged[0], table, ref, hs[0].value_of, ("r",), f"merged x{len(ds)}: {text}")


def test_merge_over_a_domain_of_different_dictionaries(oracle, ctx, pm):
    """Segments with different value subsets per column (so different dictionaries and dictIds) bound to one
    DictionaryDomain: merged MIN / MAX / DISTINCTCOUNT work on domain ids, which must decode to the reference's values."""
    rng = np.random.default_rng(77)
    hs, devs, dom = [], [], None
    try:
        for j, n in enumerate([40, 6_145, 20_000]):
            pools = {c: pool[np.sort(rng.choice(len(pool), size=len(pool) - 1 - j % 2, replace=False))]
                     for c, pool in [("i", FIVE), ("l", LONGS), ("f", FLOATS), ("d", DOUBLES), *DISTINCT.items()]}
            hs.append(_segment(oracle, n, 900 + j, pools))
        devs = [to_device(ctx, s) for s in hs]
        dom = DictionaryDomain.build(ctx, devs, ["k", "w", "e", "i", "l", "f", "d", *DISTINCT])
        for d in devs:
            d.bind_domain(dom)
        queries = [t for t in AGG_QUERIES + GB_QUERIES if "(r)" not in t]   # "r" is raw: no domain
        queries.append("SELECT MIN(i), MAX(i), MAX(l), MIN(f), DISTINCTCOUNT(i), DISTINCTCOUNT(l) FROM t WHERE w < 7")
        for text in queries:
            q = sql.parse(text, num_groups_limit=1_000_000)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            table = gpu_table(_DomainValues(devs[0]), q, merged)
            ref = check_exact(oracle, hs, q, table, "domain merge: " + text)
            check_ids(q, merged, table, ref, devs[0].dictionary_value, (), "domain merge: " + text)
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()


class _DomainValues:
    """id -> value through a bound segment's handle (the domain dictionary)."""

    def __init__(self, dev):
        self.dev = dev

    def value_of(self, column, dict_id):
        return self.dev.dictionary_value(column, dict_id)

"""-m gpu: SUM / AVG / COUNT against the exact reference (tests/exact_ref.py) on every accumulation route of the scan kernel,
with INT values at the extremes: INT_MAX / INT_MIN everywhere, the dictionary {INT_MIN, -1, 0, 1, INT_MAX}, one heavy group
whose shared-table low word wraps many times, mixed signs whose group totals land on 0 and on multiples of 2^32, sums
above 2^53, the count carrier with a negative minimum over the full 32-bit range, and a carrier entry that wraps to zero.

Each route is forced with pb200_tuning_set and the knob is restored in a `finally`.  Every docstring names the host rule in
pinot_b200/csrc/pb200_plan.cpp (plan_scan) that sends the query down that route.  Segment sizes cover ragged tails and
the tile edges of both CTA widths (6 x 1024 and 8 x 1024 rows)."""
import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import check_query, gpu_table, to_device, tuned
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
SIZES = [1, 31, 33, 6_143, 6_144, 6_145, 8_191, 8_192, 8_193, 16_385, 50_000]
VALUE_SETS = ["int_max", "int_min", "five", "heavy", "cancel"]
G = 24            # small key space "k": a replicated shared-memory table
GB = 10_000       # large key space "kb": one 8-warp CTA per SM with the table (segments of >= GB rows hold every key)

AGG_QUERIES = ["SELECT SUM(v), COUNT(*), AVG(v) FROM t WHERE w < 7",
               "SELECT SUM(v) FROM t"]
GB_QUERIES = ["SELECT SUM(v), COUNT(*) FROM t WHERE w < 7 GROUP BY {k}",
              "SELECT AVG(v) FROM t GROUP BY {k}",
              "SELECT SUM(v) FROM t WHERE w != 3 GROUP BY {k}"]           # the count only marks the groups that exist
RAW_QUERIES = ["SELECT SUM(r), COUNT(*), AVG(r) FROM t WHERE w < 7",
               "SELECT SUM(r), COUNT(*) FROM t WHERE w < 7 GROUP BY k",
               "SELECT AVG(r), SUM(v) FROM t GROUP BY k"]


def _values(vset, k, rng):
    n = len(k)
    if vset == "int_max":
        return np.full(n, INT_MAX, dtype=np.int32)
    if vset == "int_min":
        return np.full(n, INT_MIN, dtype=np.int32)
    if vset == "five":
        return rng.choice(np.array([INT_MIN, -1, 0, 1, INT_MAX], dtype=np.int32), size=n)
    if vset == "heavy":   # k was made 90 % zeros: about every second row of group 0 carries out of the low word
        return (INT_MAX - rng.integers(0, 1000, size=n)).astype(np.int32)
    # "cancel": per group, (x, -x) pairs, after a prefix that makes the total 0, -2^32 or +2^32
    v = np.zeros(n, dtype=np.int64)
    for g in range(G):
        idx = np.nonzero(k == g)[0]
        prefix = [[], [INT_MIN, INT_MIN], [INT_MAX, INT_MAX, 2]][g % 3]
        if len(idx) < len(prefix):
            prefix = []
        v[idx[:len(prefix)]] = prefix
        rest = idx[len(prefix):]
        x = rng.integers(-INT_MAX, INT_MAX + 1, size=len(rest) // 2)
        v[rest[0:2 * len(x):2]] = x
        v[rest[1:2 * len(x):2]] = -x
    return v.astype(np.int32)


def _segment(oracle, vset, n, seed):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, G, size=n)
    if vset == "heavy":
        k = np.where(rng.random(n) < 0.9, 0, k)
    k[:min(n, G)] = np.arange(min(n, G))          # every segment of >= G rows holds every key: they merge by dictId
    kb = rng.permutation(n) % GB
    v = _values(vset, k, rng)
    return oracle.build_segment(f"{vset}{n}", {"k": k.astype(np.int32), "kb": kb.astype(np.int32),
                                               "w": rng.integers(0, 10, size=n).astype(np.int32), "v": v, "r": v.copy()},
                                raw=["r"])


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
    """{(value set, rows): (host segment, device segment)}.  The raw column "r" is loaded with raw_dict_max 0, so it stays a
    raw 32-bit stream (VAL_RAW_I32) whatever its distinct count."""
    out = {}
    with tuned(ctx, raw_dict_max=0):
        for i, vset in enumerate(VALUE_SETS):
            for n in SIZES:
                seg = _segment(oracle, vset, n, 1000 * i + n)
                out[(vset, n)] = (seg, to_device(ctx, seg))
    yield out
    for _, dev in out.values():
        dev.destroy()


def sweep(oracle, pm, segs, queries, what, min_rows=1, carrier=None):
    """check_query (oracle parity + exact reference) of every query over every segment; `carrier`: expected count_carrier
    of every group-by that reaches the device (a filter the host proves empty is answered without a launch)."""
    for (vset, n), (seg, dev) in segs.items():
        if n < min_rows:
            continue
        for text in queries:
            q = sql.parse(text, num_groups_limit=1_000_000)
            _, block = check_query(oracle, pm, seg, dev, q, f"{what} {vset} n={n}: {text}")
            if carrier is not None and q.is_group_by and block.operator_kind != "EMPTY":
                assert block.count_carrier == carrier, (what, vset, n, text)


def _gb(key="k"):
    return [t.format(k=key) for t in GB_QUERIES]


# ---------------------------------------------------------------------------------------------------- aggregation only
def test_agg_deferred_gathers(oracle, ctx, pm, segs):
    """Defaults.  `!plan.group_by && tune.defer` makes the first INT-dictionary SUM / AVG q.defer_agg: dense tiles gather
    biased values (GatherBiasedU32) and drain() sums them one tile later, removing popc * 2^31."""
    sweep(oracle, pm, segs, AGG_QUERIES, "deferred")


def test_agg_immediate_sum(oracle, ctx, pm, segs):
    """`defer` 0: q.defer_agg stays -1, so dense tiles sum with SumBiasedU32 and remove pc << 31 in the same tile."""
    with tuned(ctx, defer=0):
        sweep(oracle, pm, segs, AGG_QUERIES, "immediate")


def test_agg_sparse_rows(oracle, ctx, pm, segs):
    """`sparse_max_agg` 32: q.sparse_max_agg = 32 >= every warp's survivor count (wmax2), so every surviving row goes
    through process_row (one read per row, signed 64-bit add)."""
    with tuned(ctx, sparse_max_agg=32):
        sweep(oracle, pm, segs, AGG_QUERIES, "sparse")


@pytest.mark.parametrize("defer", [1, 0], ids=["w8_agg", "w8_agg_nodefer"])
def test_agg_eight_warps(oracle, ctx, pm, segs, defer):
    """`warps` 8: cw = tune.warps, 8192-row tiles.  ScanVariant's DEFER is `!(cw == 8 && !tune.defer)`: with `defer` 0
    the w8_agg_nodefer kernel runs."""
    with tuned(ctx, warps=8, defer=defer):
        sweep(oracle, pm, segs, AGG_QUERIES, f"w8 defer={defer}")


def test_raw_int_column(oracle, ctx, pm, segs):
    """"r" was loaded with raw_dict_max 0: bits == 32 and no device dictionary, so val_kind = VAL_RAW_I32 (signed words
    summed as they stream; in a group-by, a shared-table sum with a count array: the carrier needs VAL_DICT_I32)."""
    sweep(oracle, pm, segs, RAW_QUERIES, "raw")
    with tuned(ctx, smem_groups=0):
        sweep(oracle, pm, segs, RAW_QUERIES[1:], "raw, global table")


# ---------------------------------------------------------------------------------------------------- group-by tables
@pytest.mark.parametrize("gb_defer", [1, 0], ids=["pipelined_last_batch", "no_pipeline"])
def test_gb_global_table(oracle, ctx, pm, segs, gb_defer):
    """`smem_groups` 0: q.smem_groups stays 0, every survivor is a red.add.u64 into the global table.  With gb_defer (the
    default) the INT sum of the last queue batch is software-pipelined (drain_gb); `gb_defer` 0 reduces it at once."""
    with tuned(ctx, smem_groups=0, gb_defer=gb_defer):
        sweep(oracle, pm, segs, _gb(), f"global gb_defer={gb_defer}", carrier=True)


@pytest.mark.parametrize("copies", [0, 1, 32], ids=["auto", "one_copy", "32_copies"])
def test_gb_shared_small_table(oracle, ctx, pm, segs, copies):
    """24 keys, only COUNT and INT sums: the table fits next to a 2-deep ring (room_for(cw, ctas_per_sm)), so each CTA keeps
    it in shared memory, replicated while copies x 2 fit in 64 KB; `smem_copies` 1 / 32 clamp the replication."""
    with tuned(ctx, smem_copies=copies):
        sweep(oracle, pm, segs, _gb(), f"shared copies={copies}", carrier=True)


def test_gb_shared_small_table_eight_warps(oracle, ctx, pm, segs):
    """`warps` 8: cw = tune.warps for the group-by kernel as well (8192-row tiles, w8_gb kernels), shared table."""
    with tuned(ctx, warps=8):
        sweep(oracle, pm, segs, _gb(), "shared w8", carrier=True)


def test_gb_shared_large_table(oracle, ctx, pm, segs):
    """10 000 keys: the 8-byte-entry table does not fit next to the rings of two 6-warp CTAs but room_for(8, 1) holds it,
    so pb200_execute switches to one 8-warp CTA per SM (cw = 8, ctas_per_sm = 1)."""
    sweep(oracle, pm, segs, _gb("kb"), "shared large", min_rows=GB, carrier=True)
    with tuned(ctx, pack_count=0):   # a count array too: 12-byte entries, still the 8-warp CTA
        sweep(oracle, pm, segs, _gb("kb")[:1], "shared large, no carrier", min_rows=GB, carrier=False)


def test_gb_count_carrier_off(oracle, ctx, pm, segs):
    """`pack_count` 0: count_carrier() returns no carrier, the table keeps a separate count (shared table: q.smem_count)."""
    with tuned(ctx, pack_count=0):
        sweep(oracle, pm, segs, _gb(), "no carrier", carrier=False)
        with tuned(ctx, smem_groups=0):
            sweep(oracle, pm, segs, _gb()[:1], "no carrier, global", carrier=False)


def test_gb_count_carrier_forced_overflow(oracle, ctx, pm, segs):
    """`pack_shift` 60: cr.shift = tune.pack_shift leaves a 4-bit count field.  Groups of 16+ rows overflow it, the
    verification (sum of carried counts != matched docs) reruns the submission without the carrier."""
    with tuned(ctx, pack_shift=60):
        sweep(oracle, pm, segs, _gb(), "pack_shift 60")
        with tuned(ctx, smem_groups=0):
            sweep(oracle, pm, segs, _gb()[:1], "pack_shift 60, global")


def test_gb_hash_table(oracle, ctx, pm, segs):
    """`dense_max` 1: the key space exceeds d.dense_max, so the table is hashed (and `gmax > tune.dense_max` rules out the
    shared table)."""
    with tuned(ctx, dense_max=1):
        sweep(oracle, pm, segs, _gb(), "hash")


@pytest.mark.parametrize("stride", [1, 16])
def test_gb_spread_table(oracle, ctx, pm, segs, stride):
    """`smem_groups` 0 and `table_stride` 1 / 16: a dense global table with q.smem_groups == 0 and no DISTINCTCOUNT holds raw
    key k at k * tune.table_stride (1: not spread)."""
    with tuned(ctx, smem_groups=0, table_stride=stride):
        sweep(oracle, pm, segs, _gb(), f"stride {stride}", carrier=True)


# ---------------------------------------------------------------------------------------------------- merged submissions
@pytest.mark.parametrize("smem_groups", [1, 0], ids=["shared", "global"])
def test_merged_and_per_segment_submissions(oracle, ctx, pm, segs, smem_groups):
    """execute_segments(..., merge=True): q.smem_merged = 1, each CTA flushes its shared table once, at exit; merge=False:
    a flush at every segment change.  20 and 37 segments exceed kMaxLaunchSegs (16): several launches per submission."""
    with tuned(ctx, smem_groups=smem_groups):
        for vset in VALUE_SETS:
            group = [(s, d) for (vs, n), (s, d) in segs.items() if vs == vset and n >= G]
            for key, rows in (("k", G), ("kb", GB)):
                chosen = [(s, d) for s, d in group if s.num_docs >= rows]
                hs, ds = [s for s, _ in chosen], [d for _, d in chosen]
                for text in [t for t in AGG_QUERIES] + _gb(key)[:2]:
                    q = sql.parse(text, num_groups_limit=1_000_000)
                    what = f"smem={smem_groups} {vset} {key}: {text}"
                    for s, b in zip(hs, pm.execute_segments(ds, q)):
                        check_exact(oracle, [s], q, gpu_table(s, q, b), "per segment " + what)
                    for copies in ((1,) if key == "kb" else (1, 2)):
                        merged = pm.execute_segments(ds * copies, q, merge=True)
                        assert len(merged) == 1
                        check_exact(oracle, hs * copies, q, gpu_table(hs[0], q, merged[0]), f"merged x{copies} " + what)
            s, d = group[-1]
            q = sql.parse(_gb()[0], num_groups_limit=1_000_000)
            check_exact(oracle, [s] * 37, q, gpu_table(s, q, pm.execute_segments([d] * 37, q, merge=True)[0]), f"x37 {vset}")


# ---------------------------------------------------------------------------------------------------- sums above 2^53
@pytest.fixture(scope="module")
def above_2_53(oracle, ctx):
    """2^22 + 2^20 rows of values within 3 of INT_MAX in one group: its sum is in [2^53, 2^54) and = 3 mod 4, so a
    truncating conversion to double differs from round-to-nearest.  Key 1 holds two rows whose sum is 0 mod 4, so the
    whole segment's sum is 3 mod 4 as well."""
    rng = np.random.default_rng(53)
    n = (1 << 22) + (1 << 20)
    k = np.zeros(n, dtype=np.int32)
    k[:2] = 1
    v = (INT_MAX - rng.integers(0, 4, size=n)).astype(np.int64)
    v[:2] = INT_MAX - 3
    v[2] = INT_MAX - 3
    v[2] += (3 - int(v[k == 0].sum())) % 4
    s0 = int(v[k == 0].sum())
    assert (1 << 53) < s0 < (1 << 54) and s0 % 4 == 3 and int(v.sum()) % 4 == 3
    seg = oracle.build_segment("above_2_53", {"k": k, "v": v.astype(np.int32), "w": rng.integers(0, 10, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    yield seg, dev
    dev.destroy()


@pytest.mark.parametrize("knobs", [{}, {"defer": 0}, {"sparse_max_agg": 32}, {"warps": 8}],
                         ids=["deferred", "immediate", "sparse", "w8"])
def test_sum_above_2_53_aggregation_only(oracle, ctx, pm, above_2_53, knobs):
    """The aggregation-only routes above (see their tests): the host's (double)acc.isum must round to nearest."""
    seg, dev = above_2_53
    with tuned(ctx, **knobs):
        for text in ("SELECT SUM(v), COUNT(*), AVG(v) FROM t", "SELECT SUM(v) FROM t WHERE w < 7"):
            check_query(oracle, pm, seg, dev, sql.parse(text), f"{knobs}: {text}")


@pytest.mark.parametrize("knobs,carrier", [({}, True), ({"pack_count": 0}, False), ({"smem_groups": 0}, True),
                                           ({"smem_groups": 0, "pack_count": 0}, False)],
                         ids=["shared_carrier", "shared_count", "global_carrier", "global_count"])
def test_sum_above_2_53_group_by(oracle, ctx, pm, above_2_53, knobs, carrier):
    """Group-by: extraction's (double)long long, and with the carrier (2-bit value range: shift 33, 31-bit count field) its
    decode sum = field + count * vmin, both rounded to nearest."""
    seg, dev = above_2_53
    with tuned(ctx, **knobs):
        for text in ("SELECT SUM(v), COUNT(*) FROM t GROUP BY k", "SELECT AVG(v) FROM t WHERE w < 7 GROUP BY k"):
            _, block = check_query(oracle, pm, seg, dev, sql.parse(text), f"{knobs}: {text}")
            assert block.count_carrier == carrier, (knobs, text)


# ---------------------------------------------------------------------------------------------------- count carrier edges
@pytest.mark.parametrize("heavy,carrier", [(False, True), (True, False)], ids=["fits_16_bit_count", "count_overflows"])
@pytest.mark.parametrize("smem_groups", [1, 0], ids=["shared", "global"])
def test_carrier_negative_minimum_full_32_bit_range(oracle, ctx, pm, heavy, carrier, smem_groups):
    """Values span INT_MIN .. INT_MAX: rbits = 32, so shift = (64 + 32 + 1) / 2 = 48 and the count field has 16 bits; the
    decode adds count * vmin with vmin = INT_MIN.  Every group under 65 535 rows keeps the carrier; a group of 80 000 rows
    (72 000 after the filter) overflows it, and the submission reruns without the carrier."""
    rng = np.random.default_rng(32)
    n = 200_000
    k = rng.integers(1, 60, size=n).astype(np.int32)
    if heavy:
        k[:80_000] = 0
    v = rng.integers(INT_MIN, INT_MAX + 1, size=n).astype(np.int32)
    v[:3] = [INT_MIN, INT_MAX, INT_MIN]
    seg = oracle.build_segment("full_range", {"k": k, "v": v, "w": rng.integers(0, 10, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        with tuned(ctx, smem_groups=smem_groups):
            for text in ("SELECT SUM(v), COUNT(*) FROM t GROUP BY k", "SELECT AVG(v) FROM t WHERE w < 9 GROUP BY k"):
                _, block = check_query(oracle, pm, seg, dev, sql.parse(text), text)
                assert block.count_carrier == carrier, text
    finally:
        dev.destroy()


@pytest.mark.parametrize("smem_groups", [1, 0], ids=["shared", "global"])
def test_carrier_entry_wrapping_to_zero_is_detected(oracle, ctx, pm, smem_groups):
    """`pack_shift` 60 (4-bit count field) and `grid` 1 (one CTA takes every row): group 0 has exactly 16 rows, all equal
    to vmin, so its entry is 16 * 2^60 = 0 mod 2^64 -- table_flush skips it as empty.  The verification still sees 16
    counts missing and reruns without the carrier."""
    k = np.concatenate([np.zeros(16), np.repeat(np.arange(1, 6), 10)]).astype(np.int32)
    v = np.concatenate([np.full(16, -7), np.tile(np.arange(10) * 11 - 6, 5)]).astype(np.int32)
    seg = oracle.build_segment("wrap0", {"k": k, "v": v})
    dev = to_device(ctx, seg)
    try:
        with tuned(ctx, pack_shift=60, grid=1, smem_groups=smem_groups):
            for text in ("SELECT SUM(v), COUNT(*) FROM t GROUP BY k", "SELECT SUM(v) FROM t GROUP BY k"):
                _, block = check_query(oracle, pm, seg, dev, sql.parse(text), text)
                assert not block.count_carrier, text
    finally:
        dev.destroy()


# ---------------------------------------------------------------------------------------------------- LONG / FLOAT / DOUBLE
@pytest.mark.parametrize("n", [33, 8_193, 50_000])
def test_long_float_double_within_gamma_bound(oracle, ctx, pm, n):
    """Sums in double (sum_in_double: LONG, FLOAT, DOUBLE dictionaries) with values that cancel (+-1e15 next to small ones)
    and of mixed magnitude, on the aggregation-only kernel, the global table and the hash table.  Held to |got - S| <=
    gamma_n * A only: the oracle's 1e-6-relative rule is not meaningful where the sum cancels."""
    rng = np.random.default_rng(n)
    k = rng.integers(0, 7, size=n).astype(np.int32)
    seg = oracle.build_segment(f"fp{n}", {
        "k": k, "w": rng.integers(0, 10, size=n).astype(np.int32),
        "l": rng.choice(np.array([10**15, -10**15, 1, 3, -2, 1 << 62, -(1 << 62), 123_456_789_012], dtype=np.int64), size=n),
        "f": rng.choice(np.array([1e7, -1e7, 0.5, 1e-3, 3.25, -0.125], dtype=np.float32), size=n),
        "d": rng.choice(np.array([1e15, -1e15, 0.1, 1e-8, 123.456, -7.0], dtype=np.float64), size=n)})
    dev = to_device(ctx, seg)
    try:
        for knobs in ({}, {"defer": 0}, {"dense_max": 1}):
            with tuned(ctx, **knobs):
                for text in ("SELECT SUM(l), SUM(f), SUM(d), AVG(d), COUNT(*) FROM t WHERE w < 7",
                             "SELECT SUM(l), AVG(f), SUM(d), COUNT(*) FROM t WHERE w < 7 GROUP BY k",
                             "SELECT AVG(l), SUM(f) FROM t GROUP BY k"):
                    q = sql.parse(text)
                    block = pm.execute_segments([dev], q)[0]
                    check_exact(oracle, [seg], q, gpu_table(seg, q, block, dev), f"{knobs}: {text}")
    finally:
        dev.destroy()


# ---------------------------------------------------------------------------------------------------- determinism
def test_int_sums_do_not_depend_on_the_launch_geometry(oracle, ctx, pm, segs):
    """Integer sums are exact 64-bit sums (modulo 2^64), so grid, warps and CTAs per SM must not change a bit."""
    seg, dev = segs[("five", 50_000)]
    for text in (AGG_QUERIES[0], _gb()[0], _gb()[1], "SELECT SUM(r), COUNT(*) FROM t GROUP BY k"):
        q = sql.parse(text)
        first = None
        for knobs in ({}, {"grid": 1}, {"grid": 7}, {"warps": 8}, {"ctas_per_sm": 1}, {"warps": 8, "grid": 3}):
            with tuned(ctx, **knobs):
                block = pm.execute_segments([dev], q)[0]
            got = (np.asarray(block.keys).tobytes(), [np.asarray(x).tobytes() for x in block.doubles],
                   [np.asarray(x).tobytes() for x in block.longs])
            if first is None:
                first = got
                check_exact(oracle, [seg], q, gpu_table(seg, q, block, dev), text)
            assert got == first, (text, knobs)

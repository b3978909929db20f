"""-m gpu: the CUDA path (through the C-ABI) against the oracle and the reference's golden vectors."""
import numpy as np
import pytest

import golden_cases as G
from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment, UnsupportedQueryError
from reduce_util import combine, reduce_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def sv_dev(ctx, sv_segment):
    s = to_device(ctx, sv_segment)
    yield s
    s.destroy()


# ---------------------------------------------------------------------------------------------- reference goldens
@pytest.mark.parametrize("query,stats,expected", G.INNER_SEGMENT_AGGREGATION)
def test_golden_inner_segment_aggregation(pm, sv_segment, sv_dev, query, stats, expected):
    q = sql.parse(query)
    op = pm.make_segment_plan_node(sv_dev, q).run()
    block = op.next_block()
    count, s, mx, mn, avg_sum, avg_cnt = expected
    assert block.get_results(q) == [count, float(s), float(mx), float(mn), (float(avg_sum), avg_cnt)]
    st = op.get_execution_statistics()
    assert (st.num_docs_scanned, st.num_entries_scanned_post_filter, st.num_total_docs) == (stats[0], stats[2], stats[3])


@pytest.mark.parametrize("query,regime,stats,key,expected", G.INNER_SEGMENT_GROUP_BY)
def test_golden_inner_segment_group_by(pm, sv_segment, sv_dev, query, regime, stats, key, expected):
    q = sql.parse(query)
    if regime == "ARRAY_MAP":
        # keys wider than 63 bits are not accelerated: the plan maker must refuse (-> Java operator), never guess
        with pytest.raises(UnsupportedQueryError):
            pm.make_segment_plan_node(sv_dev, q).run().next_block()
        return
    block = pm.make_segment_plan_node(sv_dev, q).run().next_block()
    assert block.regime == regime
    table = gpu_table(sv_segment, q, block)
    count, s, mx, mn, avg_sum, avg_cnt = expected
    assert table[tuple(key)] == [count, float(s), float(mx), float(mn), (float(avg_sum), avg_cnt)]
    assert (block.stats.num_docs_scanned, block.stats.num_entries_scanned_post_filter) == (stats[0], stats[2])


@pytest.mark.parametrize("select,ascending,expected", G.INTER_SEGMENT)
def test_golden_inter_segment(pm, sv_segment, sv_dev, select, ascending, expected):
    base = f"SELECT {select} FROM testTable"
    for i, (flt, gb) in enumerate([("", ""), (G.FILTER, ""), ("", G.INTER_GROUP_BY), (G.FILTER, G.INTER_GROUP_BY)]):
        q = sql.parse(base + flt + gb)
        fns = [a.function for a in q.aggregations]
        blocks = pm.execute_segments([sv_dev] * 4, q)  # 2 segments x 2 servers in the reference's harness
        rows = reduce_rows(fns, combine(fns, [gpu_table(sv_segment, q, b) for b in blocks]))
        if gb:
            sign = 1 if ascending else -1
            rows.sort(key=lambda kv: (sign * kv[1][0], sign * kv[1][1]))
        for g, e in zip(rows[0][1], expected[i]):
            assert g == pytest.approx(e, rel=1e-9), (select, i)


def test_golden_non_scan_and_empty_operators(pm, sv_dev):
    # InterSegmentAggregationSingleValueQueriesTest.testMax: no filter -> NonScanBasedAggregationOperator
    q = sql.parse("SELECT MAX(column1), MIN(column3), COUNT(*), DISTINCTCOUNT(column1) FROM testTable")
    b = pm.execute_segments([sv_dev], q)[0]
    assert b.operator_kind == "NON_SCAN_AGGREGATION"
    assert b.get_results(q) == [2146952047.0, 17891.0, 30000, 6582]
    assert pm.explain(sv_dev, q).startswith("AGGREGATE_NO_SCAN")
    q = sql.parse("SELECT COUNT(*), SUM(column1) FROM testTable WHERE column5 = 'nope'")
    b = pm.execute_segments([sv_dev], q)[0]
    assert b.operator_kind == "EMPTY" and b.get_results(q) == [0, 0.0]
    q = sql.parse(G.AGGREGATION_QUERY + G.FILTER)
    text = pm.explain(sv_dev, q)
    assert "FILTER_SORTED_INDEX(EQ,daysSinceEpoch)" in text and "FILTER_INVERTED_INDEX(NOT_IN,column11)" in text
    assert "FILTER_FULL_SCAN(RANGE,column1" in text


# ---------------------------------------------------------------------------------------------- oracle parity, seeded
def _random_segment(oracle, rng, n, name="rnd"):
    cols = {
        "a": rng.integers(0, 7, size=n).astype(np.int32) * 3 - 5,            # card <= 7   (3 bits)
        "b": rng.integers(0, 1000, size=n).astype(np.int32),                 # 10 bits
        "c": rng.integers(0, 70000, size=n).astype(np.int32) * 11,           # 17 bits
        "d": rng.integers(0, 200, size=n).astype(np.int32),                  # 8 bits (byte aligned)
        "e": rng.integers(0, 50000, size=n).astype(np.int64) * 100003,       # LONG dictionary
        "f": (rng.integers(0, 300, size=n) / 7.0).astype(np.float64),        # DOUBLE dictionary
        "s": np.array([b"x", b"yy", b"zzz", b"w"])[rng.integers(0, 4, size=n)],  # STRING dictionary
        "t": np.sort(rng.integers(0, 5, size=n)).astype(np.int32),           # sorted column
        "g": (rng.integers(0, 60, size=n)).astype(np.float32) * 0.5,         # FLOAT dictionary
    }
    return oracle.build_segment(name, cols, inverted=["a", "d", "s"])


QUERIES = [
    "SELECT COUNT(*) FROM t",
    "SELECT COUNT(*), SUM(b), MIN(c), MAX(c), AVG(b) FROM t WHERE b > 500",
    "SELECT SUM(c), COUNT(*) FROM t WHERE b BETWEEN 100 AND 300 AND c > 200000",
    "SELECT SUM(e), MIN(e), MAX(e), AVG(e) FROM t WHERE c < 500000",
    "SELECT SUM(f), MIN(f), MAX(f), AVG(g), SUM(g) FROM t WHERE d >= 100",
    "SELECT DISTINCTCOUNT(b), DISTINCTCOUNT(s), COUNT(*) FROM t WHERE c > 100000",
    "SELECT COUNT(*), SUM(b) FROM t WHERE a = 1 AND d = 17",
    "SELECT COUNT(*), SUM(b) FROM t WHERE a IN (1, 4, 7) AND s = 'yy'",
    "SELECT COUNT(*), SUM(b) FROM t WHERE a != 1 AND s NOT IN ('x', 'w') AND b < 900",
    "SELECT COUNT(*), MAX(b) FROM t WHERE b IN (1, 5, 9, 500, 999, 1234567) OR c < 1000",
    "SELECT COUNT(*), MAX(b) FROM t WHERE b NOT IN (1, 5, 9, 500, 999)",
    "SELECT COUNT(*), SUM(c) FROM t WHERE (b < 100 OR b > 900) AND NOT (d = 5 OR c > 700000)",
    "SELECT COUNT(*), SUM(c) FROM t WHERE NOT (b < 100 AND d < 100) OR (a = 4 AND t = 2)",
    "SELECT COUNT(*), SUM(b) FROM t WHERE t = 3",
    "SELECT COUNT(*), SUM(b) FROM t WHERE t != 0 AND t < 4 AND b > 10",
    "SELECT COUNT(*), SUM(b) FROM t WHERE t IN (1, 3) OR a = -5",
    "SELECT COUNT(*), SUM(b) FROM t WHERE b > 5000",                      # always false -> EMPTY
    "SELECT COUNT(*), SUM(b) FROM t WHERE b >= 0",                        # always true -> MATCH_ALL
    "SELECT COUNT(*), SUM(c), MIN(b), MAX(b), AVG(c) FROM t GROUP BY a",
    "SELECT COUNT(*), SUM(c) FROM t WHERE b > 800 GROUP BY d",
    "SELECT SUM(b), MAX(c), MIN(e) FROM t WHERE c > 300000 GROUP BY a, s",
    "SELECT COUNT(*), SUM(f), AVG(e) FROM t GROUP BY d, a",
    "SELECT COUNT(*), SUM(b) FROM t WHERE a = 1 AND d < 50 GROUP BY b",
    "SELECT MAX(g), MIN(f) FROM t WHERE s != 'x' GROUP BY t, a",
    "SELECT COUNT(*) FROM t WHERE b > 5000 GROUP BY a",                   # no groups
    "SELECT DISTINCTCOUNT(b), DISTINCTCOUNT(s), COUNT(*) FROM t WHERE c > 100000 GROUP BY a",
    "SELECT DISTINCTCOUNT(d) FROM t GROUP BY s, t",
    "SELECT SUM(c), SUM(a), COUNT(*) FROM t GROUP BY a",                  # shared-memory tables: carries and negative addends
    "SELECT SUM(a), AVG(c) FROM t WHERE b < 990 GROUP BY t, a",
]


@pytest.mark.parametrize("n", [1, 31, 33, 4096, 8191, 8193, 100_003])
def test_parity_vs_oracle_random_segments(oracle, ctx, pm, n):
    rng = np.random.default_rng(1000 + n)
    seg = _random_segment(oracle, rng, n)
    dev = to_device(ctx, seg)
    try:
        for text in QUERIES:
            check_query(oracle, pm, seg, dev, sql.parse(text), what=f"n={n}: {text}")
    finally:
        dev.destroy()


@pytest.mark.parametrize("bits", list(range(1, 17)))
def test_parity_every_bit_width(oracle, ctx, pm, bits):
    """FixedBitIntReaderTest's sweep, end to end: filter + sum + group-by on a column of every width 1..16
    (17..31 in test_parity_wide_columns)."""
    rng = np.random.default_rng(bits)
    n = 40_003
    card = 2 if bits == 1 else (1 << (bits - 1)) + 1  # smallest cardinality whose largest dictId needs `bits` bits
    ids = rng.integers(0, card, size=n)
    ids[:card] = np.arange(card)
    rng.shuffle(ids)
    vals = (ids * 3 + 1).astype(np.int32)
    seg = oracle.build_segment("w", {"x": vals, "k": rng.integers(0, 5, size=n).astype(np.int32)})
    assert seg.column("x").bits == bits
    dev = to_device(ctx, seg)
    try:
        span = int(vals.max()) - int(vals.min())
        lo, hi = int(vals.min()) + span // 4, int(vals.max()) - span // 4
        for text in (f"SELECT COUNT(*), SUM(x), MIN(x), MAX(x) FROM t WHERE x BETWEEN {lo} AND {hi}",
                     "SELECT COUNT(*), SUM(x), MAX(x) FROM t GROUP BY k",
                     "SELECT DISTINCTCOUNT(x) FROM t WHERE k = 2"):
            check_query(oracle, pm, seg, dev, sql.parse(text), what=f"bits={bits}: {text}")
    finally:
        dev.destroy()


@pytest.mark.parametrize("bits", [17, 20, 23, 24, 25, 26])
def test_parity_wide_columns(oracle, ctx, pm, bits):
    """Widths above 16 bits: dictionary with 2^(bits-1)+k entries would need that many rows; instead build the index
    buffers directly (dictIds written with the oracle's bit writer over a synthetic sorted dictionary)."""
    from oracle import segment_builder as sb
    rng = np.random.default_rng(bits)
    n = 30_000
    card = (1 << (bits - 1)) + 12345
    ids = rng.integers(0, card, size=n).astype(np.int64)
    ids[0], ids[1] = card - 1, 0
    # sparse "dictionary": only the first 70 000 entries are materialised; restrict SUM to dictIds below that
    lim = 70_000
    ids[2:n // 2] = rng.integers(0, lim, size=n // 2 - 2)
    fwd = sb.pack_fixed_bits(ids.astype(np.uint32), bits)
    dict_vals = (np.arange(lim, dtype=np.int64) * 2 + 7).astype(np.int32)
    k = rng.integers(0, 3, size=n).astype(np.int32)
    kcol = sb.build_column("k", k)
    xcol = sb.ColumnData("x", sb.INT, True, bits, card, False, 4, fwd, None, None)
    # registering needs card*4 dictionary bytes: allocate lazily-zero pages
    full = np.empty(card, dtype=">i4")
    full[:lim] = dict_vals
    full[lim:] = int(dict_vals[-1]) + 1 + np.arange(card - lim, dtype=np.int64)  # dictionaries are strictly sorted
    xcol.dict = np.frombuffer(full.tobytes(), dtype=np.uint8)
    xcol.dict_values = full.astype(np.int32)
    seg = sb.SegmentData("wide", n, [xcol, kcol])
    dev = to_device(ctx, seg)
    try:
        hi = int(dict_vals[-1])
        for text in (f"SELECT COUNT(*), SUM(x), MAX(x), MIN(x) FROM t WHERE x <= {hi}",
                     f"SELECT COUNT(*), SUM(x) FROM t WHERE x <= {hi} GROUP BY k",
                     "SELECT COUNT(*), MAX(x) FROM t WHERE k != 1"):
            check_query(oracle, pm, seg, dev, sql.parse(text), what=f"bits={bits}: {text}")
    finally:
        dev.destroy()


def test_multi_segment_single_submission_and_device_merge(oracle, ctx, pm):
    """8 segments in one launch (per-segment results) and the device-side combine against the oracle-side merge."""
    rng = np.random.default_rng(77)
    # shared dictionaries: every segment contains every value at least once
    def seg(i, n):
        b = np.concatenate([np.arange(100), rng.integers(0, 100, size=n - 100)]).astype(np.int32)
        a = np.concatenate([np.arange(100) % 8, rng.integers(0, 8, size=n - 100)]).astype(np.int32)
        c = np.concatenate([np.arange(100) * 50, rng.integers(0, 100, size=n - 100) * 50]).astype(np.int32)
        rng.shuffle(b)
        return oracle.build_segment(f"s{i}", {"a": a, "b": b, "c": c})
    segs = [seg(i, n) for i, n in enumerate([20_000, 9_000, 8192, 8193, 50_001, 333, 16_384, 12_345])]
    devs = [to_device(ctx, s) for s in segs]
    try:
        for text in ("SELECT COUNT(*), SUM(c), MIN(b), MAX(b) FROM t WHERE b > 40 AND c < 4000",
                     "SELECT COUNT(*), SUM(c), MAX(b), AVG(c) FROM t WHERE b > 40 GROUP BY a",
                     "SELECT SUM(b) FROM t GROUP BY a, b"):
            q = sql.parse(text)
            fns = [a.function for a in q.aggregations]
            want_blocks = [oracle_table(s, q, oracle.execute(s, q)) for s in segs]
            blocks = pm.execute_segments(devs, q)
            for s, b, w in zip(segs, blocks, want_blocks):
                assert_tables_equal(q, gpu_table(s, q, b), w, text)
                check_exact(oracle, [s], q, gpu_table(s, q, b), text)
            merged = pm.execute_segments(devs, q, merge=True)
            assert len(merged) == 1
            assert_tables_equal(q, gpu_table(segs[0], q, merged[0]), combine(fns, want_blocks), "merged " + text)
            check_exact(oracle, segs, q, gpu_table(segs[0], q, merged[0]), "merged " + text)
            if q.is_group_by:
                # deferred extraction (what a cross-GPU reduce of the dense tables sits between): tables first, groups later
                from pinot_b200 import _lib
                from pinot_b200.plan_maker import _read_result
                late = pm.execute_segments(devs, q, merge=True, keep_handle=True)[0]
                assert late.num_groups == 0 and late.handle is not None
                _lib.check(ctx.lib.pb200_result_finalize(ctx.handle, late.handle))
                late = _read_result(ctx, late.handle, q, 1, keep_handle=False)
                assert gpu_table(segs[0], q, late) == gpu_table(segs[0], q, merged[0]), "deferred " + text
    finally:
        for d in devs:
            d.destroy()


def test_more_segments_than_one_launch_holds(oracle, ctx, pm):
    """A submission of more than 16 segments is split into several launches (the TMA table of a launch holds 16): per-segment
    results and the device-side merge must not depend on where the chunk boundaries fall."""
    rng = np.random.default_rng(21)
    n = 9_000
    seg = oracle.build_segment("many", {"a": rng.integers(0, 6, size=n).astype(np.int32),
                                        "b": rng.integers(0, 300, size=n).astype(np.int32),
                                        "c": rng.integers(-50, 50, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        for text in ("SELECT COUNT(*), SUM(c), MIN(b), MAX(b) FROM t WHERE b > 100",
                     "SELECT COUNT(*), SUM(c) FROM t WHERE b < 250 GROUP BY a",            # shared-memory tables
                     "SELECT SUM(b), MAX(c), AVG(c) FROM t WHERE c > -40 GROUP BY b, a"):   # global tables
            q = sql.parse(text)
            want = oracle_table(seg, q, oracle.execute(seg, q))
            k = 37  # 16 + 16 + 5
            blocks = pm.execute_segments([dev] * k, q)
            assert len(blocks) == k
            for b in blocks:
                assert_tables_equal(q, gpu_table(seg, q, b), want, text)
            merged = gpu_table(seg, q, pm.execute_segments([dev] * k, q, merge=True)[0])
            fns = [a.function for a in q.aggregations]
            assert_tables_equal(q, merged, combine(fns, [want] * k), "merged x37 " + text)
            check_exact(oracle, [seg] * k, q, merged, "merged x37 " + text)
    finally:
        dev.destroy()


def test_num_groups_limit_forces_fallback(oracle, ctx, pm):
    rng = np.random.default_rng(5)
    seg = oracle.build_segment("lim", {"k": rng.integers(0, 5000, size=40_000).astype(np.int32),
                                       "v": rng.integers(0, 10, size=40_000).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        q = sql.parse("SELECT SUM(v) FROM t GROUP BY k", num_groups_limit=100, max_initial_result_holder_capacity=100)
        with pytest.raises(UnsupportedQueryError):
            pm.make_segment_plan_node(dev, q).run().next_block()
    finally:
        dev.destroy()


GROUP_BY_QUERIES = [t for t in QUERIES if "GROUP BY" in t] + [
    "SELECT COUNT(*), SUM(b), MIN(c), MAX(e), AVG(f) FROM t WHERE b < 700 GROUP BY a, d, s, t, g",   # 5 keys
    "SELECT SUM(c) FROM t GROUP BY c, b",                                                              # many groups
]


@pytest.mark.parametrize("n", [1, 33, 8193, 100_003])
def test_hash_group_table_parity(oracle, ctx, pm, n):
    """Key spaces beyond the dense limit (the reference's LONG_MAP regime) go through the device hash table; forcing the
    limit down to 1 sends every group-by shape through it."""
    ctx.set_tuning("dense_max", 1)
    rng = np.random.default_rng(2000 + n)
    seg = _random_segment(oracle, rng, n)
    dev = to_device(ctx, seg)
    try:
        for text in GROUP_BY_QUERIES:
            check_query(oracle, pm, seg, dev, sql.parse(text, num_groups_limit=200_000), what=f"hash n={n}: {text}")
        # device-side merge of several segments into ONE hash table
        q = sql.parse("SELECT COUNT(*), SUM(b), MAX(c) FROM t WHERE b > 100 GROUP BY d, a", num_groups_limit=200_000)
        merged = pm.execute_segments([dev, dev, dev], q, merge=True)[0]
        single = gpu_table(seg, q, pm.execute_segments([dev], q)[0])
        got = gpu_table(seg, q, merged)
        assert set(got) == set(single)
        for k, v in single.items():
            assert got[k] == [3 * v[0], 3 * v[1], v[2]], (k, got[k], v)
        # more groups than numGroupsLimit: explicit fallback, never a truncated table
        if n >= 8193:
            with pytest.raises(UnsupportedQueryError):
                pm.execute_segments([dev], sql.parse("SELECT SUM(c) FROM t GROUP BY c, b", num_groups_limit=1000))
    finally:
        ctx.set_tuning("dense_max", 1 << 24)
        dev.destroy()


def test_hash_group_table_natural_long_map(oracle, ctx, pm):
    """A key space that really needs 64-bit raw keys (product of cardinalities > 2^31)."""
    rng = np.random.default_rng(77)
    n = 60_000
    seg = oracle.build_segment("lm", {
        "k1": rng.integers(0, 50_000, size=n).astype(np.int32), "k2": rng.integers(0, 40_000, size=n).astype(np.int32),
        "k3": rng.integers(0, 300, size=n).astype(np.int32), "v": rng.integers(-1000, 1000, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        q = sql.parse("SELECT COUNT(*), SUM(v), MIN(v), MAX(v) FROM t WHERE v > -900 GROUP BY k1, k2, k3")
        r, block = check_query(oracle, pm, seg, dev, q, "natural LONG_MAP")
        assert block.regime == "LONG_MAP" and block.num_groups > 50_000
    finally:
        dev.destroy()


def test_raw_forward_index_column(oracle, ctx, pm):
    """No-dictionary INT metric (FixedByteChunkSVForwardIndexReader, PASS_THROUGH) as an aggregation argument."""
    rng = np.random.default_rng(9)
    n = 25_000
    seg = oracle.build_segment("raw", {"m": rng.integers(-10**9, 10**9, size=n).astype(np.int32),
                                       "k": rng.integers(0, 9, size=n).astype(np.int32)}, raw=["m"])
    ctx.set_tuning("raw_dict_max", 0)   # keep the column RAW on the device (default: dictionary synthesised at load, test_gpu_raw.py)
    try:
        dev = to_device(ctx, seg)
    finally:
        ctx.set_tuning("raw_dict_max", 1 << 20)
    try:
        for text in ("SELECT SUM(m), MIN(m), MAX(m), AVG(m), COUNT(*) FROM t WHERE k > 3",
                     "SELECT SUM(m), MAX(m), MIN(m) FROM t GROUP BY k",
                     # value-space predicates on the raw column itself (PB200_F_RAW_RANGE; IntRawValueBasedRangePredicateEvaluator)
                     "SELECT COUNT(*), SUM(m) FROM t WHERE m > 0",
                     "SELECT COUNT(*), SUM(m), MIN(m), MAX(m) FROM t WHERE m BETWEEN -500000000 AND 250000000 AND k < 7",
                     "SELECT COUNT(*) FROM t WHERE m >= -1000000000 AND m < -999000000",
                     f"SELECT COUNT(*), MAX(k) FROM t WHERE m = {int(seg.column('m').raw_values[17])} OR k = 2",
                     "SELECT COUNT(*), SUM(m) FROM t WHERE NOT (m > 5 AND m <= 700000000) GROUP BY k",
                     "SELECT COUNT(*) FROM t WHERE m > 2000000000"):                       # empty
            check_query(oracle, pm, seg, dev, sql.parse(text), text)
        with pytest.raises(UnsupportedQueryError):                                       # IN on a raw column: stock operator
            pm.execute_segments([dev], sql.parse("SELECT COUNT(*) FROM t WHERE m IN (1, 2, 3)"))
    finally:
        dev.destroy()


def test_errors_are_reported_not_swallowed(ctx, pm, sv_dev):
    from pinot_b200._lib import Pb200Error
    with pytest.raises(Pb200Error) as e:
        pm.execute_segments([sv_dev], sql.parse("SELECT SUM(nope) FROM t"))
    assert "nope" in str(e.value)
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([sv_dev], sql.parse("SELECT SUM(column11) FROM t WHERE column1 > 5"))


@pytest.mark.parametrize("bits", list(range(1, 32)))
def test_c_abi_dictid_space_every_width(ctx, bits):
    """Straight through include/pinot_b200.h (no host layer): SCAN_RANGE / SCAN_IN on dictIds + COUNT / MIN / MAX /
    DISTINCT-free aggregation for EVERY forward-index width 1..31, checked against numpy on the same dictIds."""
    import ctypes as C
    from oracle import segment_builder as sb
    from pinot_b200 import _lib
    L = ctx.lib
    rng = np.random.default_rng(500 + bits)
    n = 70_001
    top = (1 << bits) - 1
    ids = rng.integers(0, top + 1, size=n, dtype=np.int64)
    ids[:4] = [0, top, top // 2, 1]
    fwd = sb.pack_fixed_bits(ids.astype(np.uint32), bits)
    k = rng.integers(0, 4, size=n).astype(np.int64)
    kf = sb.pack_fixed_bits(k.astype(np.uint32), 2)
    cols = (_lib.ColDesc * 2)()
    # STRING stored type: no device dictionary needed; MIN/MAX come back as dictIds
    cols[0] = _lib.ColDesc(_lib.FWD_DICT_FIXEDBIT, _lib.STRING, bits, min(top + 1, 2**31 - 1), 0, 0,
                           fwd.ctypes.data_as(C.c_void_p), len(fwd), None, 0, None, 0)
    cols[1] = _lib.ColDesc(_lib.FWD_DICT_FIXEDBIT, _lib.STRING, 2, 4, 0, 0, kf.ctypes.data_as(C.c_void_p), len(kf),
                           None, 0, None, 0)
    seg = C.c_void_p()
    _lib.check(L.pb200_segment_register(ctx.handle, b"w", n, 2, cols, C.byref(seg)))
    try:
        lo, hi = top // 5, top - top // 7 + 1
        in_ids = np.unique(np.concatenate([ids[5:40], [0, top]])).astype(np.int32)
        in_ids = in_ids[in_ids >= 0]
        nodes = (_lib.FilterNode * 3)()
        nodes[0] = _lib.FilterNode(5, 0, 0, int(lo), int(min(hi, 2**31 - 1)), 0, None, 0, 0, 0, 0)       # SCAN_RANGE
        nodes[1] = _lib.FilterNode(7, 1, 0, 0, 0, 1, (C.c_int32 * 1)(2), 0, 0, 0, 0)                     # k NOT IN (2)
        nodes[2] = _lib.FilterNode(0, -1, 2, 0, 0, 0, None, 0, 0, 0, 0)                                  # AND
        aggs = (_lib.Agg * 3)(_lib.Agg(0, -1), _lib.Agg(2, 0), _lib.Agg(3, 0))
        q = _lib.Query(3, 0, 3, 100000, 10000, 0, nodes, None, aggs)
        segs = (C.c_void_p * 1)(seg)
        res = (C.c_void_p * 1)()
        _lib.check(L.pb200_execute(ctx.handle, C.byref(q), segs, 1, res))
        m = (ids >= lo) & (ids < hi) & (k != 2)
        d = np.zeros(1); l = np.zeros(1, dtype=np.int64); di = np.zeros(1, dtype=np.int32)
        _lib.check(L.pb200_result_agg(res[0], 0, d.ctypes.data_as(C.c_void_p), l.ctypes.data_as(C.c_void_p)))
        assert l[0] == int(m.sum())
        _lib.check(L.pb200_result_agg_dict_ids(res[0], 1, di.ctypes.data_as(C.c_void_p)))
        assert di[0] == (int(ids[m].min()) if m.any() else -1)
        _lib.check(L.pb200_result_agg_dict_ids(res[0], 2, di.ctypes.data_as(C.c_void_p)))
        assert di[0] == (int(ids[m].max()) if m.any() else -1)
        L.pb200_result_free(res[0])
        if bits <= 20:  # SCAN_IN through the dictId bitmap + group-by on the 2-bit key
            nodes2 = (_lib.FilterNode * 1)()
            arr = (C.c_int32 * len(in_ids))(*in_ids.tolist())
            nodes2[0] = _lib.FilterNode(6, 0, 0, 0, 0, len(in_ids), arr, 0, 0, 0, 0)
            gb = (C.c_int32 * 1)(1)
            aggs2 = (_lib.Agg * 2)(_lib.Agg(0, -1), _lib.Agg(3, 0))
            q2 = _lib.Query(1, 1, 2, 100000, 10000, 0, nodes2, gb, aggs2)
            _lib.check(L.pb200_execute(ctx.handle, C.byref(q2), segs, 1, res))
            meta = _lib.ResultMeta()
            _lib.check(L.pb200_result_meta_get(res[0], C.byref(meta)))
            m2 = np.isin(ids, in_ids)
            want = {int(g): (int((m2 & (k == g)).sum()), int(ids[m2 & (k == g)].max())) for g in np.unique(k[m2])}
            G_ = meta.num_groups
            keys = np.zeros((G_, 1), dtype=np.int32); cnt = np.zeros(G_, dtype=np.int64); dd = np.zeros(G_)
            mx = np.zeros(G_, dtype=np.int32)
            _lib.check(L.pb200_result_group_keys(res[0], keys.ctypes.data_as(C.c_void_p)))
            _lib.check(L.pb200_result_agg(res[0], 0, dd.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p)))
            _lib.check(L.pb200_result_agg_dict_ids(res[0], 1, mx.ctypes.data_as(C.c_void_p)))
            got = {int(keys[i, 0]): (int(cnt[i]), int(mx[i])) for i in range(G_)}
            assert got == want
            L.pb200_result_free(res[0])
    finally:
        L.pb200_segment_release(ctx.handle, seg)


def test_long_sum_does_not_wrap(oracle, ctx, pm):
    """SUM / AVG over a LONG dictionary accumulate in double like SumAggregationFunction.java:69-145: values whose sum
    passes 2^63 (epoch-millis-sized values x a few million rows, or a few ~1e18 values) must not wrap."""
    rng = np.random.default_rng(63)
    n = 70_000
    big = (rng.integers(1, 9, size=n).astype(np.int64) * 1_000_000_000_000_000_000) + rng.integers(0, 1000, size=n)   # ~1e18 .. 8e18
    seg = oracle.build_segment("long", {"e": big, "k": rng.integers(0, 5, size=n).astype(np.int32),
                                        "h": rng.integers(0, 3000, size=n).astype(np.int32)})
    assert float(big.astype(np.float64).sum()) > 2.0 ** 63
    dev = to_device(ctx, seg)
    try:
        for text in ("SELECT SUM(e), AVG(e), COUNT(*) FROM t", "SELECT SUM(e), AVG(e) FROM t WHERE k < 4",
                     "SELECT SUM(e), AVG(e), MAX(e) FROM t GROUP BY k",          # shared-memory-table sized key space
                     "SELECT SUM(e), COUNT(*) FROM t WHERE k > 0 GROUP BY h"):   # global tables, survivor queue
            r, block = check_query(oracle, pm, seg, dev, sql.parse(text), "LONG sum: " + text)
            assert all(v > 0 for v in block.doubles[0]), text
        merged = pm.execute_segments([dev, dev, dev], sql.parse("SELECT SUM(e) FROM t GROUP BY k"), merge=True)[0]
        single = pm.execute_segments([dev], sql.parse("SELECT SUM(e) FROM t GROUP BY k"))[0]
        assert np.allclose(merged.doubles[0], 3.0 * single.doubles[0], rtol=1e-12)
    finally:
        dev.destroy()


def test_count_carrier_and_its_overflow_fallback(oracle, ctx, pm):
    """Group-by COUNT / AVG counts ride in the upper bits of an INT sum's reductions (one L2 read-modify-write per row
    instead of two).  A sum field that overflows is detected exactly (sum of carried counts != matched docs) and the
    submission reruns with a separate COUNT table: results are exact either way."""
    rng = np.random.default_rng(64)
    n = 90_000
    seg = oracle.build_segment("carrier", {
        "k": rng.integers(0, 5000, size=n).astype(np.int32),                      # global tables (> shared-memory limit)
        "big": rng.integers(-2_000_000_000, 2_000_000_000, size=n).astype(np.int32),
        "small": rng.integers(-50, 50, size=n).astype(np.int32),
        "w": rng.integers(0, 40, size=n).astype(np.int32)})
    dev = to_device(ctx, seg)
    queries = ["SELECT SUM(big), COUNT(*) FROM t WHERE w > 3 GROUP BY k",
               "SELECT AVG(small), SUM(big), MAX(w) FROM t GROUP BY k",
               "SELECT SUM(small) FROM t WHERE w < 30 GROUP BY k",                 # count only as the group-exists marker
               "SELECT COUNT(*), SUM(small), SUM(big), AVG(big) FROM t WHERE w != 7 GROUP BY k, w"]
    try:
        for text in queries:
            q = sql.parse(text, num_groups_limit=1_000_000)
            _, block = check_query(oracle, pm, seg, dev, q, "carrier: " + text)
            assert block.count_carrier, text                                        # ~18 rows per group: neither field overflows
        ctx.set_tuning("pack_shift", 33)   # 33-bit sum field: groups of `big` overflow it (~18 rows x up to 4e9 each), `small` does not
        for text in queries:
            q = sql.parse(text, num_groups_limit=1_000_000)
            _, block = check_query(oracle, pm, seg, dev, q, "carrier, shift 33: " + text)
            carried_first = [a.column for a in q.aggregations if a.function in ("SUM", "AVG")][0]
            assert block.count_carrier == (carried_first == "small"), (text, block.count_carrier)
        ctx.set_tuning("pack_count", 0)
        _, block = check_query(oracle, pm, seg, dev, sql.parse(queries[0], num_groups_limit=1_000_000), "carrier off")
        assert not block.count_carrier
    finally:
        ctx.set_tuning("pack_shift", 0)
        ctx.set_tuning("pack_count", 1)
        dev.destroy()

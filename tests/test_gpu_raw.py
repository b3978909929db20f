"""-m gpu: raw (no-dictionary) columns -- every fixed-width type, every chunk compression the loader decodes, as aggregation
arguments, filter columns and GROUP BY keys.

What the product does (pinot_b200/csrc/host/raw_forward.cpp): chunks are decoded once at load; a raw column with at most
`raw_dict_max` distinct values gets a dictionary synthesised from its values and is an ordinary dictionary column on the
device from there on.  What the reference does: raw-value predicate evaluators, NoDictionary*GroupKeyGenerator (group keys
are VALUES, group ids in first-seen order), aggregation over the raw value block.  Both must give the same VALUES -- the
oracle restates the reference's side (oracle/pinot_oracle.cpp: raw predicates, NO_DICTIONARY regime; oracle/chunk_codecs.py)."""
import os

import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, check_query, gpu_table, oracle_table, to_device
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def _segment(oracle, n, seed, compression):
    rng = np.random.default_rng(seed)
    ri = (rng.integers(0, 300, size=n) * 7 - 1000).astype(np.int32)            # raw INT, 300 distinct values
    rl = (rng.integers(0, 50, size=n).astype(np.int64) * 3_000_000_007 - 5)     # raw LONG beyond 32 bits
    rf = (rng.integers(0, 64, size=n) / 4.0 - 3.0).astype(np.float32)           # raw FLOAT incl. negatives
    rd = (rng.integers(0, 1000, size=n) / 8.0 + 0.125).astype(np.float64)       # raw DOUBLE
    return oracle.build_segment(f"raw{seed}", {
        "ri": ri, "rl": rl, "rf": rf, "rd": rd,
        "k": rng.integers(0, 9, size=n).astype(np.int32), "v": rng.integers(-500, 500, size=n).astype(np.int32)},
        raw=["ri", "rl", "rf", "rd"], raw_compression={c: compression for c in ("ri", "rl", "rf", "rd")})


QUERIES = [
    # aggregation arguments of all four raw types, with and without GROUP BY on a dictionary column
    "SELECT SUM(ri), MIN(ri), MAX(ri), AVG(ri), COUNT(*) FROM t WHERE k > 3",
    "SELECT SUM(rl), MIN(rl), MAX(rl), AVG(rl) FROM t WHERE v < 100",
    "SELECT SUM(rf), MIN(rf), MAX(rf), SUM(rd), MIN(rd), MAX(rd) FROM t",
    "SELECT SUM(rd), MAX(rl), MIN(rf), COUNT(*) FROM t WHERE v BETWEEN -200 AND 300 GROUP BY k",
    # value predicates on raw columns (range, EQ, NEQ, IN, NOT IN; *RawValueBased*PredicateEvaluator)
    "SELECT COUNT(*), SUM(v) FROM t WHERE ri > 0 AND ri <= 700",
    "SELECT COUNT(*), SUM(v) FROM t WHERE rl >= 30000000065 AND k != 2",
    "SELECT COUNT(*), MAX(v) FROM t WHERE rf < -1.5 OR rd >= 100.125",
    "SELECT COUNT(*) FROM t WHERE rd = 3.125",
    "SELECT COUNT(*), SUM(ri) FROM t WHERE ri IN (-1000, -993, 1093, 12345) OR rf IN (0.25, 0.5)",
    "SELECT COUNT(*) FROM t WHERE rl NOT IN (-5, 2999999998) AND ri != -1000",
    "SELECT COUNT(*) FROM t WHERE rd > 1000000.0",                                            # matches nothing
    # GROUP BY raw columns: NoDictionarySingleColumnGroupKeyGenerator / NoDictionaryMultiColumnGroupKeyGenerator
    "SELECT COUNT(*), SUM(v) FROM t GROUP BY ri",
    "SELECT COUNT(*), MAX(v), MIN(rd) FROM t WHERE k < 5 GROUP BY rl",
    "SELECT SUM(v), COUNT(*) FROM t GROUP BY rf, k",
    "SELECT SUM(ri), AVG(rd) FROM t WHERE v > 0 GROUP BY rd, rl",
    "SELECT COUNT(*) FROM t GROUP BY k, ri, rf",
    # DISTINCTCOUNT over raw columns: value sets (DistinctCountAggregationFunction without a dictionary)
    "SELECT DISTINCTCOUNT(ri), DISTINCTCOUNT(rd), COUNT(*) FROM t WHERE k > 1",
    "SELECT DISTINCTCOUNT(rl), DISTINCTCOUNT(rf) FROM t WHERE v > 0 GROUP BY k",
    "SELECT DISTINCTCOUNT(rd) FROM t GROUP BY rf",
]


@pytest.mark.parametrize("compression", [0, 1, 3, 4], ids=["pass_through", "snappy", "lz4", "lz4_length_prefixed"])
def test_raw_columns_all_types_and_codecs(oracle, ctx, pm, compression):
    n = 6_001 if compression else 40_003
    seg = _segment(oracle, n, 40 + compression, compression)
    dev = to_device(ctx, seg)
    try:
        for c in ("ri", "rl", "rf", "rd"):   # the column became a dictionary column: sorted distinct values
            info = dev.column_info(c)
            uniq = np.unique(seg.column(c).raw_values)
            assert info["has_dictionary"] and info["cardinality"] == len(uniq)
            assert [dev.dictionary_value(c, i) for i in (0, len(uniq) - 1)] == [uniq[0].item(), uniq[-1].item()]
        for text in QUERIES:
            check_query(oracle, pm, seg, dev, sql.parse(text, num_groups_limit=1_000_000), text)
    finally:
        dev.destroy()


def test_raw_group_by_merged_over_segments_by_value(oracle, ctx, pm):
    """Three segments whose raw columns hold DIFFERENT value sets: per-segment synthesised dictionaries differ, so the
    device-side combine needs a dictionary domain -- built over the synthesised dictionaries like over stored ones."""
    from pinot_b200.plan_maker import DictionaryDomain
    from reduce_util import combine
    segs = [_segment(oracle, 9_000 + 17 * i, 90 + i, [0, 1, 3][i]) for i in range(3)]
    devs = [to_device(ctx, s) for s in segs]
    dom = None
    try:
        q = sql.parse("SELECT COUNT(*), SUM(v), MAX(rd) FROM t WHERE ri > -500 GROUP BY rl, rf", num_groups_limit=1_000_000)
        dom = DictionaryDomain.build(ctx, devs, ["rl", "rf", "rd"])
        for d in devs:
            d.bind_domain(dom)
        block = pm.execute_segments(devs, q, merge=True)[0]
        want = combine([a.function for a in q.aggregations], [oracle_table(s, q, oracle.execute(s, q)) for s in segs])
        assert_tables_equal(q, gpu_table(segs[0], q, block, devs[0]), want, "merged raw group-by")
        check_exact(oracle, segs, q, gpu_table(segs[0], q, block, devs[0]), "merged raw group-by")
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()


@pytest.mark.parametrize("name,num_docs,start", [("fixedByteRaw.v2", 2000, 100.2356), ("fixedByteCompressed.v2", 2000, 100.2356),
                                                 ("fixedByteSVRDoubles.v1", 10009, 0.0)])
def test_reference_written_raw_forward_index_through_the_device(oracle, ctx, pm, name, num_docs, start):
    """The reference's own raw DOUBLE forward-index files (FixedByteChunkSVForwardIndexTest.java:340-377: value i == i + start)
    as the metric column of a segment: SUM / MIN / MAX / COUNT by known answer, GROUP BY against the oracle."""
    from oracle import segment_builder as sb
    blob = np.fromfile(os.path.join(HERE, "golden", "raw_forward", name), dtype=np.uint8)
    k = (np.arange(num_docs) % 7).astype(np.int32)
    seg = oracle.build_segment("golden_raw", {"k": k})
    want_vals = np.arange(num_docs) + start
    from oracle import chunk_codecs as cc
    plain = cc.encode_fixed_byte_forward(want_vals.astype(">f8").tobytes(), 8, num_docs, cc.PASS_THROUGH)
    seg.columns.append(sb.ColumnData("m", sb.DOUBLE, False, 0, 0, False, 8, blob, None, None, raw_values=want_vals, oracle_fwd=plain))
    for dict_max in (1 << 20, 0):
        ctx.set_tuning("raw_dict_max", dict_max)
        try:
            if dict_max == 0:
                with pytest.raises(Exception):   # a raw DOUBLE column that stays raw is not accelerated: refused loudly
                    d2 = to_device(ctx, seg)
                    try:
                        pm.execute_segments([d2], sql.parse("SELECT SUM(m) FROM t"))
                    finally:
                        d2.destroy()
                continue
            dev = to_device(ctx, seg)
            try:
                b = pm.execute_segments([dev], sql.parse("SELECT SUM(m), MIN(m), MAX(m), COUNT(*) FROM t WHERE m >= 500.0"))[0]
                sel = want_vals[want_vals >= 500.0]
                assert int(b.longs[3][0]) == len(sel) and float(b.doubles[1][0]) == sel.min() and float(b.doubles[2][0]) == sel.max()
                assert abs(float(b.doubles[0][0]) - sel.sum()) <= 1e-9 * sel.sum()
                check_query(oracle, pm, seg, dev, sql.parse("SELECT SUM(m), MAX(m), COUNT(*) FROM t WHERE m < 1500.5 GROUP BY k"), name)
            finally:
                dev.destroy()
        finally:
            ctx.set_tuning("raw_dict_max", 1 << 20)


def test_high_cardinality_raw_int_stays_raw(oracle, ctx, pm):
    """More distinct values than raw_dict_max: the INT column stays a raw 4-byte stream (PB200_F_RAW_RANGE, raw aggregation)."""
    rng = np.random.default_rng(3)
    n = 30_000
    seg = oracle.build_segment("hc", {"m": rng.integers(-10**9, 10**9, size=n).astype(np.int32),
                                      "k": rng.integers(0, 9, size=n).astype(np.int32)}, raw=["m"], raw_compression={"m": 3})
    ctx.set_tuning("raw_dict_max", 1000)
    try:
        dev = to_device(ctx, seg)
        try:
            assert not dev.column_info("m")["has_dictionary"]
            for text in ("SELECT SUM(m), MIN(m), MAX(m), COUNT(*) FROM t WHERE k > 3",
                         "SELECT COUNT(*), SUM(m) FROM t WHERE m BETWEEN -500000000 AND 250000000 GROUP BY k"):
                check_query(oracle, pm, seg, dev, sql.parse(text), text)
        finally:
            dev.destroy()
    finally:
        ctx.set_tuning("raw_dict_max", 1 << 20)

"""-m gpu: BASELINE-sized parity.  One 100 M-row segment per workload shape (C2 aggregation, C3 bitmap filter -> GROUP BY
10 000, C3 range filter -> GROUP BY, C4 two-dimension GROUP BY with SUM / MAX) through the device library AND through the
CPU oracle on ALL rows -- not a property check.

The oracle's operator chain is single threaded per segment (as the reference's is); to finish in seconds the segment is
generated on the CPU by the oracle's twin of the device generator (identical bytes: test_gpu_synth.py) and cut into row
ranges at multiples of 32 rows (zero-copy views), one oracle call per range on every host core; ranges share the
dictionaries, so their tables merge by dictId with AggregationFunction.merge semantics (tests/reduce_util.combine).
"""
import os
import threading

import numpy as np
import pytest

from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, IndexSegment

pytestmark = pytest.mark.gpu

ROWS = 100_000_000
COLS = [("d1", 10, True), ("d2", 20, True), ("d3", 50, True), ("g", 10_000, False), ("m", 100_000, False),
        ("f", 10_000, False), ("g2", 100, False), ("h", 1_000_000, False)]


def _max_abs_value(spec):
    return max(abs(spec["value_base"]), abs(spec["value_base"] + spec["value_step"] * (spec["cardinality"] - 1)))


def specs(seed0):
    return [{"name": n, "cardinality": c, "value_base": 2, "value_step": 3, "inverted": inv, "seed": seed0 + i}
            for i, (n, c, inv) in enumerate(COLS)]


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def big(ctx, oracle):
    """(device segment with inverted indexes, the same segment's columns on the CPU split into row ranges)"""
    sp = specs(424242)
    dev = IndexSegment.synthetic(ctx, "full", ROWS, sp)
    host = oracle.synth_segment("full", ROWS, sp)
    parts = oracle.row_ranges(host, max(8, os.cpu_count() or 8))
    yield dev, host, parts
    dev.destroy()


def oracle_tables(oracle, parts, q):
    """{dictId key tuple: [per aggregation intermediate]} over all row ranges, merged like AggregationFunction.merge."""
    results = [None] * len(parts)
    nxt, lock = [0], threading.Lock()

    def work():
        while True:
            with lock:
                i = nxt[0]
                nxt[0] += 1
            if i >= len(parts):
                return
            results[i] = oracle.execute(parts[i], q)

    ts = [threading.Thread(target=work) for _ in range(min(len(parts), os.cpu_count() or 8))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    fns = [a.function for a in q.aggregations]
    out = {}
    for r in results:
        rows = 1 if r.num_groups < 0 else r.num_groups
        for g in range(rows):
            key = () if r.num_groups < 0 else tuple(int(x) for x in r.keys[g])
            vals = [int(r.longs[a][g]) if fn == "COUNT" else (float(r.doubles[a][g]), int(r.longs[a][g])) if fn == "AVG"
                    else float(r.doubles[a][g]) for a, fn in enumerate(fns)]
            cur = out.get(key)
            if cur is None:
                out[key] = vals
                continue
            for a, fn in enumerate(fns):
                if fn in ("COUNT", "SUM"):
                    cur[a] += vals[a]
                elif fn == "AVG":
                    cur[a] = (cur[a][0] + vals[a][0], cur[a][1] + vals[a][1])
                elif fn == "MIN":
                    cur[a] = min(cur[a], vals[a])
                else:
                    cur[a] = max(cur[a], vals[a])
    return out, sum(r.stats[0] for r in results)


def device_table(block, q):
    fns = [a.function for a in q.aggregations]
    rows = 1 if block.num_groups < 0 else block.num_groups
    out = {}
    for g in range(rows):
        key = () if block.num_groups < 0 else tuple(int(x) for x in block.keys[g])
        out[key] = [int(block.longs[a][g]) if fn == "COUNT" else (float(block.doubles[a][g]), int(block.longs[a][g])) if fn == "AVG"
                    else float(block.doubles[a][g]) for a, fn in enumerate(fns)]
    return out


FULL_QUERIES = [
    # C2: 2-predicate range filter + SUM / COUNT (BASELINE configs[1])
    ("c2", "SELECT SUM(m), COUNT(*), MIN(h), MAX(h) FROM t WHERE f BETWEEN 3002 AND 14999 AND h > 1500000"),
    # C3: inverted-index bitmap filter (3 EQ AND-ed) -> GROUP BY dim (card 10 000) SUM (configs[2]); dictIds 3, 5, 25
    ("c3_bitmap", "SELECT SUM(m), COUNT(*) FROM t WHERE d1 = 11 AND d2 = 17 AND d3 = 77 GROUP BY g"),
    # the bench headline's shape: range filter (10 %) -> GROUP BY 10 000 -> SUM, COUNT (per-thread sparse path)
    ("c3_range", "SELECT SUM(m), COUNT(*) FROM t WHERE f BETWEEN 3002 AND 5999 GROUP BY g"),
    # same through the survivor queue (50 % of the rows survive)
    ("c3_range_dense", "SELECT SUM(m), COUNT(*), AVG(m) FROM t WHERE f < 15002 GROUP BY g"),
    # C4: filter + GROUP BY 2 dims + SUM / MAX (configs[3]); 1 000 000-key space
    ("c4", "SELECT SUM(m), MAX(f), MIN(h) FROM t WHERE f BETWEEN 3002 AND 5999 GROUP BY g, g2"),
    # small key space: CTA-private shared-memory tables
    ("small_groups", "SELECT COUNT(*), SUM(m) FROM t WHERE h > 1000000 GROUP BY g2"),
]


@pytest.mark.parametrize("name,text", FULL_QUERIES)
def test_full_size_segment_equals_oracle(oracle, ctx, big, name, text):
    dev, host, parts = big
    q = sql.parse(text, num_groups_limit=2_000_000)
    # every partial sum of the oracle's Java-order double is an integer below rows x max|value| < 2^53, so it is exact:
    # the device's integer sums must equal it bit for bit
    for agg in q.aggregations:
        if agg.function in ("SUM", "AVG"):
            assert ROWS * _max_abs_value(next(s for s in specs(0) if s["name"] == agg.column)) < 2 ** 53, agg.column
    want, want_docs = oracle_tables(oracle, parts, q)
    block = B200PlanMaker(ctx).make_segment_plan_node(dev, q).run().next_block()
    got = device_table(block, q)
    assert block.stats.num_docs_scanned == want_docs, name
    assert set(got) == set(want), f"{name}: {len(got)} groups vs {len(want)}"
    for key, wv in want.items():
        gv = got[key]
        for a, agg in enumerate(q.aggregations):
            # SUM, AVG (sum and count), COUNT, MIN, MAX: bit exact
            assert gv[a] == wv[a], (name, key, agg.function, gv[a], wv[a])


def test_full_size_generators_agree(oracle, big):
    """The CPU table the oracle scanned IS the device table: forward-index bytes of a 100 M-row column, both generators."""
    dev, host, _ = big
    for cname in ("g", "h"):
        assert np.array_equal(dev.read_index(cname, "fwd"), host.column(cname).fwd), cname
        assert np.array_equal(dev.read_index(cname, "dict"), host.column(cname).dict), cname

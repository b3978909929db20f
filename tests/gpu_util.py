"""Helpers shared by the -m gpu tests: run one query through the product (C-ABI) and through the oracle, compare."""
from __future__ import annotations

import contextlib

from exact_ref import check_exact
from pinot_b200.plan_maker import IndexSegment
from reduce_util import normalise

# Parity with the oracle's Java-order double sums (BASELINE.json north_star): SUM / AVG within 1e-6 relative of the oracle,
# everything else equal.  It is not the exactness check: integer SUMs are held bit-exact, and floating sums to the gamma_n
# bound, by tests/exact_ref.py (check_query runs both).
SUM_REL_TOL = 1e-6

# pb200_tuning_set knobs at their library defaults: what tuned() restores
TUNING_DEFAULTS = {"warps": 6, "defer": 1, "gb_defer": 1, "sparse_max_agg": -1, "smem_groups": 1, "smem_copies": 0,
                   "pack_count": 1, "pack_shift": 0, "dense_max": 1 << 24, "table_stride": 0, "grid": 0, "ctas_per_sm": 2,
                   "raw_dict_max": 1 << 20, "always_count": 0,
                   "sparse_max": 4, "skip": 1, "stages": 0, "spec": 1}


@contextlib.contextmanager
def tuned(ctx, **knobs):
    """Sets tuning knobs for the body of a `with` and restores their defaults afterwards, also when the body fails."""
    try:
        for name, value in knobs.items():
            ctx.set_tuning(name, value)
        yield
    finally:
        for name in knobs:
            ctx.set_tuning(name, TUNING_DEFAULTS[name])


def to_device(ctx, seg_data) -> IndexSegment:
    """Registers oracle-built Pinot index buffers with the device library (host pointers -> HBM)."""
    return IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)


class _ProductValues:
    """id -> value for PRODUCT results: columns the segment stores raw got a dictionary at load (raw_forward.cpp), their ids
    are resolved through the product's own accessor (pb200h_dictionary_get), everything else through the oracle-built data."""

    def __init__(self, seg_data, dev_seg):
        self.seg_data, self.dev = seg_data, dev_seg
        self.cache = {}

    def value_of(self, column, dict_id):
        if self.seg_data.column(column).has_dictionary:
            return self.seg_data.value_of(column, dict_id)
        key = (column, dict_id)
        if key not in self.cache:
            self.cache[key] = self.dev.dictionary_value(column, dict_id)
        return self.cache[key]


class _OracleValues:
    """id -> value for ORACLE results: raw group-by keys are ids of the result's on-the-fly dictionary
    (NoDictionary*GroupKeyGenerator), see OracleResult.raw_key_values."""

    def __init__(self, seg_data, q, r):
        self.seg_data = seg_data
        self.raw = {q.group_by[j]: v for j, v in getattr(r, "raw_key_values", {}).items()}

    def value_of(self, column, dict_id):
        if column in self.raw:
            return self.raw[column][dict_id].item()
        return self.seg_data.value_of(column, dict_id)


def gpu_table(seg_data, q, block, dev_seg=None):
    values = seg_data if dev_seg is None else _ProductValues(seg_data, dev_seg)
    return normalise(values, q, block.num_groups, block.keys, block.doubles, block.longs, block.distinct)


def oracle_table(seg_data, q, r):
    table = normalise(_OracleValues(seg_data, q, r), q, r.num_groups, r.keys, r.doubles, r.longs,
                      {k: (v if k[0] not in getattr(r, "raw_distinct_values", {}) else ()) for k, v in r.distinct.items()})
    # DISTINCTCOUNT over a raw column: the oracle's sets hold numbers of its own value numbering (OracleResult.raw_distinct_values)
    raw = getattr(r, "raw_distinct_values", {})
    if raw:
        rows = 1 if r.num_groups < 0 else r.num_groups
        values = _OracleValues(seg_data, q, r)
        for g in range(rows):
            key = () if r.num_groups < 0 else tuple(values.value_of(c, int(r.keys[g, j])) for j, c in enumerate(q.group_by))
            for a, numbering in raw.items():
                table[key][a] = frozenset(numbering[int(i)].item() for i in r.distinct[(a, g)])
    return table


def assert_tables_equal(q, got, want, what=""):
    assert set(got.keys()) == set(want.keys()), f"{what}: group keys differ: {len(got)} vs {len(want)}"
    for key, wv in want.items():
        gv = got[key]
        for a, agg in enumerate(q.aggregations):
            fn = agg.function
            if fn in ("SUM",):
                assert gv[a] == wv[a] or abs(gv[a] - wv[a]) <= SUM_REL_TOL * abs(wv[a]), (what, key, fn, gv[a], wv[a])
            elif fn == "AVG":
                assert gv[a][1] == wv[a][1], (what, key, fn, gv[a], wv[a])
                assert gv[a][0] == wv[a][0] or abs(gv[a][0] - wv[a][0]) <= SUM_REL_TOL * abs(wv[a][0]), (what, key, fn)
            else:  # COUNT / MIN / MAX / DISTINCTCOUNT: bit exact
                assert gv[a] == wv[a], (what, key, fn, gv[a], wv[a])


def check_query(oracle, pm, seg_data, dev_seg, q, what=""):
    r = oracle.execute(seg_data, q)
    block = pm.make_segment_plan_node(dev_seg, q).run().next_block()
    got = gpu_table(seg_data, q, block, dev_seg)
    assert_tables_equal(q, got, oracle_table(seg_data, q, r), what)
    check_exact(oracle, [seg_data], q, got, what)
    assert block.stats.num_docs_scanned == r.stats[0], what
    assert block.stats.num_total_docs == r.stats[3], what
    return r, block

"""-m gpu: GROUP BY ... ORDER BY ... LIMIT -- rows ordered and trimmed by the library (pb200h_execute_ordered), against an
ordering of the exact reference (tests/exact_ref.py).

The reference takes the exact per-group table, computes final values (AVG = sum / count, DISTINCTCOUNT = set size),
orders the rows by the ORDER BY items and then by the group-key values ascending, and keeps the first K.  The device rows
must be those rows, in that order: keys equal, COUNT / MIN / MAX / DISTINCTCOUNT equal, INT SUM / AVG bit-exact.  The
matrix sums INT columns only; LONG / DOUBLE sums, which are exact only within a bound, have a test of their own.

Every order shape runs with every trim size (0 = sorted, not trimmed; 1; K inside a run of equal items; the group count;
above it) on every route: the table kinds of the scan kernel (forced with tuned()), merged, deferred and per-segment
submissions, FILTER-clause results (aligned and ordered on the host) and star-tree results (ordered on the host)."""
import ctypes as C
import math

import numpy as np
import pytest

import datatable_util
import golden_cases as G
from exact_ref import reference
from gpu_util import to_device, tuned
from oracle import startree_builder as stb
from pinot_b200 import _lib, sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, _marshal_query, _read_result, order_spec

pytestmark = pytest.mark.gpu

KG, K2, STRS, VALS, DIST = 37, 3, 12, 7, 40

SHAPES = {
    "count_desc": "SELECT COUNT(*), SUM(m) FROM t GROUP BY k ORDER BY COUNT(*) DESC",
    "sum_asc": "SELECT SUM(m), COUNT(*) FROM t GROUP BY k ORDER BY SUM(m)",
    "min_asc_max_desc": "SELECT MIN(m), MAX(m) FROM t GROUP BY k, k2 ORDER BY MIN(m), MAX(m) DESC",
    "avg": "SELECT AVG(m), COUNT(*) FROM t GROUP BY k ORDER BY AVG(m) DESC",
    "distinctcount": "SELECT DISTINCTCOUNT(c), COUNT(*) FROM t GROUP BY k ORDER BY DISTINCTCOUNT(c) DESC",
    "key_desc": "SELECT COUNT(*) FROM t GROUP BY k, k2 ORDER BY k DESC",
    "string_key": "SELECT SUM(m) FROM t GROUP BY s, k2 ORDER BY s DESC, SUM(m)",
    "two_items_tie_runs": "SELECT COUNT(*), MAX(t3), MIN(t3) FROM t GROUP BY k, k2 ORDER BY MAX(t3) DESC, MIN(t3)",
}
TRIMS = ["0", "1", "tie", "groups", "above"]
KNOB_ROUTES = {"global": {"smem_groups": 0}, "smem_carrier": {}, "carrier_off": {"pack_count": 0}, "hash": {"dense_max": 1},
               "stride_1": {"table_stride": 1}, "stride_16": {"table_stride": 16}}
ROUTES = list(KNOB_ROUTES) + ["merged_18", "deferred", "per_segment", "filter_clause"]


def _segment(oracle, n, seed):
    """Every value of every pool occurs in each segment (identical dictionaries: segments merge on the device)."""
    rng = np.random.default_rng(seed)
    pools = {"k": KG, "k2": K2, "s": STRS, "m": VALS, "c": DIST, "t3": 3, "w": 10}
    cols = {}
    for c, card in pools.items():
        v = rng.integers(0, card, size=n)
        v[:card] = np.arange(card)
        cols[c] = v
    cols["k"] = np.where(rng.random(n) < 0.3, cols["k"] % 5, cols["k"])    # skewed counts: some ties, some not
    cols["k"][:KG] = np.arange(KG)
    out = {c: v.astype(np.int32) for c, v in cols.items()}
    out["m"] = (out["m"] - 3) * 1000                                       # negative, zero and positive sums
    out["s"] = np.array([f"s{i:02d}".encode() for i in range(STRS)])[cols["s"]]
    out["x"] = rng.standard_normal(n) * 1e6                                # DOUBLE
    out["l"] = rng.integers(-(1 << 40), 1 << 40, size=n).astype(np.int64)  # LONG
    return oracle.build_segment(f"ob{n}_{seed}", out)


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def data(oracle, ctx):
    """18 segments of ragged sizes; segment 0 is the large one the single-segment routes use."""
    sizes = [9_001] + [1_000 + 113 * i for i in range(17)]
    hs = [_segment(oracle, n, 40 + i) for i, n in enumerate(sizes)]
    ds = [to_device(ctx, s) for s in hs]
    yield hs, ds
    for d in ds:
        d.destroy()


def _dbl_key(x: float):
    """Double.compare order (-0.0 before 0.0)."""
    return (x, math.copysign(1.0, x))


def _final(fn, v):
    if fn == "COUNT":
        return int(v)
    if fn == "SUM":
        return float(v.s)
    if fn == "AVG":
        return float(v.s) / v.n if v.n else float("-inf")
    if fn == "DISTINCTCOUNT":
        return len(v)
    return float(v)


def ordered_reference(oracle, segs, q):
    """[(key values, final values)] of the whole table in ORDER BY order, ties by the key values ascending."""
    ref = reference(oracle, segs, q)
    rows = sorted((key, [_final(a.function, v) for a, v in zip(q.aggregations, vals)]) for key, vals in ref.items())
    for kind, index, asc in reversed(sql.resolve_order_by(q)):
        if kind == "GROUP_BY":
            rows.sort(key=lambda r: r[0][index], reverse=not asc)
        else:
            rows.sort(key=lambda r: _dbl_key(float(r[1][index])), reverse=not asc)
    return rows


def items_of(q, row):
    return tuple(row[0][i] if kind == "GROUP_BY" else row[1][i] for kind, i, _ in sql.resolve_order_by(q))


def tie_trim(q, rows):
    """K that ends inside a run of rows equal on every item (the tie key decides which rows are kept)."""
    for i in range(1, len(rows)):
        if items_of(q, rows[i - 1]) == items_of(q, rows[i]) and i + 1 < len(rows) and items_of(q, rows[i]) == items_of(q, rows[i + 1]):
            return i
    for i in range(1, len(rows)):
        if items_of(q, rows[i - 1]) == items_of(q, rows[i]):
            return i
    return max(1, len(rows) // 2)


def trim_value(name, q, rows):
    return {"0": 0, "1": 1, "tie": tie_trim(q, rows), "groups": len(rows), "above": len(rows) + 7}[name]


def device_rows(seg, q, block):
    out = []
    for g in range(block.num_groups):
        key = tuple(seg.value_of(c, int(block.keys[g, j])) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            fn = agg.function
            if fn in ("COUNT", "DISTINCTCOUNT"):
                vals.append(int(block.longs[a][g]))
            elif fn == "AVG":
                n = int(block.longs[a][g])
                vals.append(float(block.doubles[a][g]) / n if n else float("-inf"))
            else:
                vals.append(float(block.doubles[a][g]))
        out.append((key, vals))
    return out


def execute_ordered(pm, devs, q, trim, merge=False, defer=False):
    """pb200h_execute_ordered with an explicit trim size (deferred: merge_segments 2, reduce_world 1, then finalize)."""
    L, ctx = pm.ctx.lib, pm.ctx
    spec = order_spec(q, merge)
    spec.trim_size = trim
    hq, _keep = _marshal_query(q, 2 if defer else merge, reduce_world=1 if defer else 0)
    n = len(devs)
    segs = (C.c_void_p * n)(*[d.handle for d in devs])
    nres = 1 if merge else n
    res, kinds = (C.c_void_p * nres)(), (C.c_int32 * n)()
    _lib.check(L.pb200h_execute_ordered(ctx.handle, C.byref(hq), C.byref(spec), segs, n, res, kinds))
    if defer:
        _lib.check(L.pb200_result_finalize(ctx.handle, res[0]))
    return [_read_result(ctx, C.c_void_p(res[i]), q, kinds[0 if merge else i], False) for i in range(nres)]


def assert_rows(got, want, trim, what):
    kept = min(trim, len(want)) if trim > 0 else len(want)
    assert len(got) == kept, f"{what}: {len(got)} rows, want {kept}"
    for i, (g, w) in enumerate(zip(got, want[:kept])):
        assert g[0] == w[0], (what, "row", i, "key", g[0], w[0])
        assert all(a == b and math.copysign(1, a) == math.copysign(1, b) if isinstance(b, float) else a == b
                   for a, b in zip(g[1], w[1])), (what, "row", i, g, w)


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_order_and_trim(oracle, pm, ctx, data, shape, route):
    hs, ds = data
    text = SHAPES[shape]
    if route == "filter_clause":
        text = text.replace(" FROM t", ", SUM(m) FILTER (WHERE w < 5) FROM t", 1)
    q = sql.parse(text, num_groups_limit=1_000_000)
    if route in KNOB_ROUTES:
        want = ordered_reference(oracle, [hs[0]], q)
        with tuned(ctx, **KNOB_ROUTES[route]):
            for t in TRIMS:
                trim = trim_value(t, q, want)
                block = execute_ordered(pm, [ds[0]], q, trim)[0]
                assert_rows(device_rows(hs[0], q, block), want, trim, f"{shape} {route} trim={t}")
    elif route in ("merged_18", "deferred"):
        segs = (hs, ds) if route == "merged_18" else (hs[:2], ds[:2])
        want = ordered_reference(oracle, segs[0], q)
        for t in TRIMS:
            trim = trim_value(t, q, want)
            block = execute_ordered(pm, segs[1], q, trim, merge=True, defer=route == "deferred")[0]
            assert_rows(device_rows(hs[0], q, block), want, trim, f"{shape} {route} trim={t}")
    elif route == "per_segment":
        wants = [ordered_reference(oracle, [h], q) for h in hs[1:4]]
        for t in TRIMS:
            trim = trim_value(t, q, wants[0])
            blocks = execute_ordered(pm, ds[1:4], q, trim)
            for h, b, w in zip(hs[1:4], blocks, wants):
                assert_rows(device_rows(h, q, b), w, trim, f"{shape} per segment {h.name} trim={t}")
    else:
        for merge in (False, True):
            segs = ([hs[0]], [ds[0]]) if not merge else (hs[:3], ds[:3])
            want = ordered_reference(oracle, segs[0], q)
            for t in TRIMS:
                trim = trim_value(t, q, want)
                block = execute_ordered(pm, segs[1], q, trim, merge=merge)[0]
                assert_rows(device_rows(hs[0], q, block), want, trim, f"{shape} FILTER merge={merge} trim={t}")


def test_star_tree_results_are_ordered_on_the_host(oracle, ctx, pm):
    rng = np.random.default_rng(5)
    n = 30_000
    seg = oracle.build_segment("obst", {"d1": rng.integers(0, 60, size=n).astype(np.int32),
                                        "d2": rng.integers(0, 4, size=n).astype(np.int32),
                                        "m": rng.integers(-5, 6, size=n).astype(np.int32) * 100})
    st = stb.build_star_tree(seg, ["d1", "d2"], [("COUNT", None), ("SUM", "m"), ("MAX", "m"), ("MIN", "m")], max_leaf_records=10)
    dev = to_device(ctx, seg)
    try:
        nd = len(st.dimensions)
        dev.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                             [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
        for order in ("COUNT(*) DESC", "SUM(m)", "MIN(m), MAX(m) DESC", "AVG(m) DESC", "d1 DESC", "MAX(m) DESC, d2"):
            q = sql.parse(f"SELECT COUNT(*), SUM(m), MIN(m), MAX(m), AVG(m) FROM t GROUP BY d1, d2 ORDER BY {order}")
            want = ordered_reference(oracle, [seg], q)
            for t in TRIMS:
                trim = trim_value(t, q, want)
                block = execute_ordered(pm, [dev], q, trim)[0]
                assert block.operator_kind == "STAR_TREE"
                assert_rows(device_rows(seg, q, block), want, trim, f"star-tree {order} trim={t}")
    finally:
        dev.destroy()


def test_approximate_sums_are_ordered_by_their_own_values(oracle, pm, data):
    """LONG / DOUBLE sums: exact only within exact_ref's bound.  The rows must be sorted by the device's own values, and
    every reference row clearly above the K-th value (beyond the bound) must be kept."""
    hs, ds = data
    for text in ("SELECT SUM(x), COUNT(*) FROM t GROUP BY k ORDER BY SUM(x) DESC",
                 "SELECT SUM(l) FROM t GROUP BY k, k2 ORDER BY SUM(l)",
                 "SELECT AVG(x) FROM t GROUP BY k ORDER BY AVG(x) DESC"):
        q = sql.parse(text, num_groups_limit=1_000_000)
        ref = reference(oracle, hs, q)
        (_, _, asc), = sql.resolve_order_by(q)
        trim = 9
        block = execute_ordered(pm, ds, q, trim, merge=True)[0]
        got = device_rows(hs[0], q, block)
        assert len(got) == trim
        vals = [r[1][0] for r in got]
        assert vals == sorted(vals, reverse=not asc), text
        exact = {key: (float(v[0].s) / (v[0].n or 1) if q.aggregations[0].function == "AVG" else float(v[0].s))
                 for key, v in ref.items()}
        bound = max(abs(float(v[0].a)) for v in ref.values()) * 1e-9
        kth = vals[-1]
        kept = {r[0] for r in got}
        for key, v in exact.items():
            beyond = v < kth - bound if asc else v > kth + bound
            if beyond:
                assert key in kept, (text, key, v, kth)


def test_golden_inter_segment_tops(pm, ctx, sv_segment):
    """InterSegmentAggregationSingleValueQueriesTest group-by tops: 4 copies of the reference fixture merged on the device
    with the trim; row 0 is the reference's answer."""
    dev = to_device(ctx, sv_segment)
    try:
        cases = [(sel, asc, exp[2], exp[3]) for sel, asc, exp in G.INTER_SEGMENT]
        cases.append(("COUNT(*)", False, (G.INTER_SEGMENT_COUNT[2],), (G.INTER_SEGMENT_COUNT[3],)))
        for select, ascending, top, top_filtered in cases:
            fns = [s.strip() for s in select.split(",")]
            order = ", ".join(f"{f} {'ASC' if ascending else 'DESC'}" for f in fns)
            for flt, expected in (("", top), (G.FILTER, top_filtered)):
                q = sql.parse(f"SELECT {select} FROM testTable{flt}{G.INTER_GROUP_BY} ORDER BY {order} LIMIT 1")
                block = pm.execute_segments([dev] * 4, q, merge=True)[0]
                assert block.num_groups == min(5000, block.num_groups) and block.num_groups >= 1
                row = device_rows(sv_segment, q, block)[0][1]
                for g, e in zip(row, expected):
                    assert g == pytest.approx(e, rel=1e-9), (select, flt, row, expected)
    finally:
        dev.destroy()


def test_datatable_of_a_trimmed_result(pm, data):
    hs, ds = data
    q = sql.parse("SELECT SUM(m), COUNT(*), AVG(m), s FROM t GROUP BY s, k ORDER BY SUM(m) DESC LIMIT 3",
                  min_server_group_trim_size=4)
    block = pm.execute_segments(ds[:3], q, merge=True, keep_handle=True, defer=False)[0]
    try:
        assert block.num_groups == 15   # max(5 * LIMIT, 4)
        dt = datatable_util.parse(pm.to_datatable(ds[0], q, block))
        rows = device_rows(hs[0], q, block)
        assert len(dt["rows"]) == len(rows)
        for r, (key, vals) in zip(dt["rows"], rows):
            assert tuple(r[:2]) == key
            assert r[2] == vals[0] and r[3] == vals[1] and r[4][1] == vals[1]
    finally:
        block.release(pm.ctx)


def test_refusals_and_aggregation_only(pm, ctx, data):
    hs, ds = data
    q = sql.parse("SELECT COUNT(*), SUM(m) FROM t GROUP BY k ORDER BY COUNT(*) DESC")
    hq, _keep = _marshal_query(q, False)
    segs = (C.c_void_p * 1)(ds[0].handle)
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * 1)()
    bad = []
    for kind, index in ((_lib.ORDER_AGG, 2), (_lib.ORDER_AGG, -1), (_lib.ORDER_GROUP_BY, 1), (7, 0)):
        spec = _lib.OrderBy(1, 0)
        spec.items[0] = _lib.OrderItem(kind, index, 0)
        bad.append(spec)
    for num in (0, 9):
        spec = _lib.OrderBy(num, 0)
        bad.append(spec)
    for spec in bad:
        assert ctx.lib.pb200h_execute_ordered(ctx.handle, C.byref(hq), C.byref(spec), segs, 1, res, kinds) == _lib.E_INVALID
    dq = _lib.Query()
    assert ctx.lib.pb200_execute_ordered(ctx.handle, C.byref(dq), C.byref(bad[-1]), None, 0, res) == _lib.E_INVALID
    for text in ("SELECT COUNT(*), SUM(m), MAX(m) FROM t WHERE w < 5", "SELECT AVG(m), DISTINCTCOUNT(c) FROM t"):
        plain = pm.execute_segments(ds[:3], sql.parse(text), merge=True)[0]
        spec = _lib.OrderBy(1, 1)
        spec.items[0] = _lib.OrderItem(_lib.ORDER_AGG, 0, 1)
        qa = sql.parse(text)
        hqa, _k = _marshal_query(qa, True)
        segs3 = (C.c_void_p * 3)(*[d.handle for d in ds[:3]])
        r1, k1 = (C.c_void_p * 1)(), (C.c_int32 * 3)()
        _lib.check(ctx.lib.pb200h_execute_ordered(ctx.handle, C.byref(hqa), C.byref(spec), segs3, 3, r1, k1))
        ordered = _read_result(ctx, C.c_void_p(r1[0]), qa, k1[0], False)
        assert ordered.num_groups == -1
        for a in range(len(qa.aggregations)):
            assert ordered.doubles[a][0] == plain.doubles[a][0] and ordered.longs[a][0] == plain.longs[a][0], text


def test_group_counts_with_and_without_order_by(pm, ctx):
    """A merged result of 100 000 groups: ORDER BY ... LIMIT 10 keeps max(5 * 10, 5000) rows, without ORDER BY all."""
    from pinot_b200.plan_maker import IndexSegment
    segs = [IndexSegment.synthetic(ctx, f"obc{i}", 2_000_000, [{"name": "g", "cardinality": 100_000, "seed": 11 + i},
                                                              {"name": "v", "cardinality": 1000, "seed": 99 + i}])
            for i in range(2)]
    try:
        names = ["g", "v"]
        base = f"SELECT SUM({names[1]}), COUNT(*) FROM t GROUP BY {names[0]}"
        full = pm.execute_segments(segs, sql.parse(base, num_groups_limit=1_000_000), merge=True)[0]
        assert full.num_groups == 100_000
        top = pm.execute_segments(segs, sql.parse(base + f" ORDER BY SUM({names[1]}) DESC LIMIT 10",
                                                  num_groups_limit=1_000_000), merge=True)[0]
        assert top.num_groups == 5000
        sums = full.doubles[0]
        order = sorted(range(100_000), key=lambda g: (-sums[g], int(full.keys[g, 0])))[:5000]
        assert [int(full.keys[g, 0]) for g in order] == [int(x) for x in top.keys[:, 0]]
        assert np.array_equal(np.asarray(top.doubles[0]), np.asarray(sums)[order])
    finally:
        for s in segs:
            s.destroy()

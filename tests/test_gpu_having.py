"""-m gpu: GROUP BY ... HAVING -- rows filtered by the library (pb200h_execute_having) before ORDER BY and its trim, against
the exact reference.

The reference takes the exact per-group table (tests/exact_ref.py; PERCENTILE and VAR / STDDEV computed exactly from the
same rows), applies HAVING with Python's float comparisons (Java's: a NaN matches only != and NOT IN, -0.0 == 0.0), then
ORDER BY (ties by the group-key values) and the trim.  Sums are over INT columns, so every value is exact and literals can
sit anywhere, equality included; the FLOAT / DOUBLE edge data sums quarters, which are exact too.  Literals are taken from
the reference's own values, so each condition keeps none, some or all of the groups as intended."""
import contextlib
import ctypes as C
import dataclasses
import math
from fractions import Fraction

import numpy as np
import pytest

import float_edges_ref as fr
from exact_ref import _key_value, column_values, reference
from gpu_util import to_device, tuned
from oracle import segment_builder as sb
from oracle import startree_builder as stb
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import (B200Context, B200PlanMaker, DictionaryDomain, IndexSegment, _marshal_query, _read_result,
                                   having_spec, order_spec)
from pinot_b200.query import Aggregation, Filter, moments_final, percentile_index
from test_gpu_float_edges import PATTERNS, edge_segment, product_table
from test_gpu_order_by import _segment, device_rows

pytestmark = pytest.mark.gpu

KNOB_ROUTES = {"smem": {}, "spec_off": {"spec": 0}, "global": {"smem_groups": 0}, "hash": {"dense_max": 1},
               "carrier_off": {"pack_count": 0}, "stride_16": {"table_stride": 16}}
LEAVES = ["COUNT(*)", "SUM(m)", "AVG(m)", "MIN(t3)", "MAX(m)", "DISTINCTCOUNT(c)", "PERCENTILE(m, 50)", "VAR_POP(m)",
          "VAR_SAMP(m)", "STDDEV_POP(m)", "STDDEV_SAMP(m)"]


@contextlib.contextmanager
def route(ctx, knobs):
    """gpu_util.tuned, plus the specialised-scan knob `spec` (default 1)."""
    knobs = dict(knobs)
    spec = knobs.pop("spec", None)
    try:
        if spec is not None:
            ctx.set_tuning("spec", spec)
        with tuned(ctx, **knobs):
            yield
    finally:
        if spec is not None:
            ctx.set_tuning("spec", 1)


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
    """Segment 0 (9 001 rows) for the single-segment routes; 17 more, bound to one domain, for the merged route."""
    sizes = [9_001] + [1_000 + 113 * i for i in range(17)]
    hs = [_segment(oracle, n, 70 + i) for i, n in enumerate(sizes)]
    ds = [to_device(ctx, s) for s in hs]
    domain = DictionaryDomain.build(ctx, ds[1:], ["k", "k2", "m", "c", "t3"])
    for d in ds[1:]:
        d.bind_domain(domain)
    yield hs, ds
    for d in ds:
        d.destroy()
    domain.release()


# ------------------------------------------------------------------------------------------------ reference
def _final(fn, v):
    if fn == "COUNT":
        return float(v)
    if fn == "SUM":
        return float(v.s)
    if fn == "AVG":
        return float(v.s) / v.n if v.n else -math.inf
    if fn == "DISTINCTCOUNT":
        return float(len(v))
    return float(v)


EXACT_REF_FUNCTIONS = ("COUNT", "SUM", "AVG", "MIN", "MAX", "DISTINCTCOUNT")


def _rows_values(oracle, segs, q, column):
    """{key: [values of `column` in the group's matched rows]} (q: a query the oracle can filter for)."""
    out = {}
    for s in segs:
        docs = oracle.filter_doc_ids(s, q)[0].astype(np.int64)
        keys = list(zip(*[[_key_value(x) for x in column_values(oracle, s, c, docs).tolist()] for c in q.group_by]))
        for key, x in zip(keys, column_values(oracle, s, column, docs).tolist()):
            out.setdefault(key, []).append(x)
    return out


def final_table(oracle, segs, original):
    """{key: [final value per aggregation]}: exact_ref for COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT, exact
    PERCENTILE and VAR / STDDEV from the rows."""
    # the oracle filters for the functions exact_ref knows: the others are placeholders there, computed below
    aggs = original.aggregations
    q = dataclasses.replace(original, having=None, aggregations=[a if a.function in EXACT_REF_FUNCTIONS else Aggregation("COUNT")
                                                                 for a in aggs])
    ref = reference(oracle, segs, q)
    out = {key: [_final(a.function, v) for a, v in zip(q.aggregations, vals)] for key, vals in ref.items()}
    for i, agg in enumerate(aggs):
        if agg.function == "PERCENTILE" or agg.function.startswith(("VAR", "STDDEV")):
            per = _rows_values(oracle, segs, q, agg.column)
            for key, xs in per.items():
                if agg.function == "PERCENTILE":
                    out[key][i] = float(sorted(xs)[percentile_index(len(xs), agg.arg)])
                else:
                    out[key][i] = moments_final(agg.function, (len(xs), Fraction(sum(xs)), Fraction(sum(x * x for x in xs))))
    return out


def having_ref(q, node, vals):
    if isinstance(node, Filter):
        outs = [having_ref(q, c, vals) for c in node.children]
        return all(outs) if node.type == "AND" else any(outs) if node.type == "OR" else not outs[0]
    a = next(i for i, agg in enumerate(q.aggregations) if agg.filter is None and sql.having_name(agg) == node.column)
    v, lits = vals[a], [float(x) for x in node.values]
    if node.type in ("EQ", "IN"):
        return any(v == x for x in lits)
    if node.type in ("NEQ", "NOT_IN"):
        return all(v != x for x in lits)
    return ((node.lower is None or (v >= float(node.lower) if node.lower_inclusive else v > float(node.lower))) and
            (node.upper is None or (v <= float(node.upper) if node.upper_inclusive else v < float(node.upper))))


def expected_rows(q, table, trim):
    """[(key, finals)] that pass HAVING, in ORDER BY order (ties by key values) and trimmed; unordered: by key."""
    rows = sorted((k, v) for k, v in table.items() if having_ref(q, q.having, v))
    for kind, index, asc in reversed(sql.resolve_order_by(q)):
        if kind == "GROUP_BY":
            rows.sort(key=lambda r: r[0][index], reverse=not asc)
        else:
            rows.sort(key=lambda r: fr.ORDER(r[1][index]), reverse=not asc)
    return rows[:trim] if (q.order_by and trim > 0) else rows


def got_rows(seg, q, block):
    out = []
    for key, vals in device_rows(seg, q, block):
        for a, agg in enumerate(q.aggregations):   # device_rows leaves DISTINCTCOUNT / COUNT as ints
            vals[a] = float(vals[a])
        out.append((key, vals))
    return out if q.order_by else sorted(out)


def assert_same(got, want, what):
    assert [g[0] for g in got] == [w[0] for w in want], (what, len(got), len(want))
    for g, w in zip(got, want):
        for x, y in zip(g[1], w[1]):
            assert x == y or (math.isnan(x) and math.isnan(y)), (what, g, w)


def execute(pm, devs, q, merge=False, trim=None):
    """pb200h_execute_having (with the ORDER BY spec and an explicit trim when given)."""
    ctx = pm.ctx
    spec = order_spec(q, merge)
    if spec is not None and trim is not None:
        spec.trim_size = trim
    hav = having_spec(q)
    hq, _keep = _marshal_query(q, merge)
    n = len(devs)
    segs = (C.c_void_p * n)(*[d.handle for d in devs])
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * n)()
    args = (C.c_double * len(q.aggregations))(*[a.arg or 0.0 for a in q.aggregations])
    _lib.check(ctx.lib.pb200h_execute_having(ctx.handle, C.byref(hq), C.byref(spec) if spec is not None else None, args,
                                             C.byref(hav) if hav is not None else None, segs, n, res, kinds))
    return _read_result(ctx, C.c_void_p(res[0]), q, kinds[0], False)


def _lit(x):
    return np.format_float_positional(float(x), unique=True, trim="0")


def conditions(leaf, values):
    """HAVING conditions on one leaf whose literals come from the groups' values: some, none, all, and each connective."""
    vs = sorted(set(values))
    lo, mid, hi = vs[0], vs[len(vs) // 2], vs[-1]
    return [f"{leaf} > {_lit(mid)}", f"{leaf} <= {_lit(mid)}", f"{leaf} = {_lit(mid)}", f"{leaf} <> {_lit(mid)}",
            f"{leaf} BETWEEN {_lit(lo)} AND {_lit(mid)}", f"{leaf} IN ({_lit(lo)}, {_lit(hi)}, 0.5)",
            f"{leaf} NOT IN ({_lit(hi)}, {_lit(mid)})", f"NOT {leaf} < {_lit(mid)}",
            f"{leaf} > {_lit(hi)}",                                           # none
            f"{leaf} >= {_lit(lo)}",                                          # all
            f"COUNT(*) > 3 AND ({leaf} < {_lit(mid)} OR {leaf} = {_lit(hi)})"]


def _all_finals(oracle, segs, group_by):
    """{leaf: {key: value}} for every leaf of LEAVES."""
    out = {}
    for leaf in LEAVES:
        q = sql.parse(f"SELECT {leaf} FROM t GROUP BY {group_by}", num_groups_limit=1_000_000)
        out[leaf] = {k: v[0] for k, v in final_table(oracle, segs, q).items()}
    return out


def _check_leaves(oracle, pm, hs_ref, devs, merge, what, group_by="k"):
    finals = _all_finals(oracle, hs_ref, group_by)
    cache = {}
    for leaf in LEAVES:
        for cond in conditions(leaf, finals[leaf].values()):
            text = f"SELECT {group_by}, COUNT(*), SUM(m) FROM t GROUP BY {group_by} HAVING {cond}"
            q = sql.parse(text, num_groups_limit=1_000_000)
            key = tuple((a.function, a.column, a.arg) for a in q.aggregations)
            if key not in cache:
                cache[key] = final_table(oracle, hs_ref, q)
            want = expected_rows(q, cache[key], max(5 * q.limit, 5000) if merge else 0)
            assert_same(got_rows(hs_ref[0], q, execute(pm, devs, q, merge)), want, f"{what}: {text}")


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("route_name", list(KNOB_ROUTES))
def test_every_leaf_function_on_every_table_route(oracle, ctx, pm, data, route_name):
    hs, ds = data
    with route(ctx, KNOB_ROUTES[route_name]):
        _check_leaves(oracle, pm, [hs[0]], [ds[0]], False, route_name)


def test_every_leaf_function_merged_over_17_segments(oracle, pm, data):
    hs, ds = data
    _check_leaves(oracle, pm, hs[1:], ds[1:], True, "merged 17", group_by="k, k2")


@pytest.mark.parametrize("order", ["SUM(m) DESC", "COUNT(*), k", "AVG(m) DESC, k DESC", "MAX(m) DESC"])
@pytest.mark.parametrize("trim", [0, 1, 4, 1000])
def test_having_before_order_and_trim(oracle, pm, data, order, trim):
    """HAVING -> ORDER BY -> trim: with a trim, only passing rows compete for it; AVG and MAX are hidden aggregations."""
    hs, ds = data
    for segs, devs, merge in (([hs[0]], [ds[0]], False), (hs[1:], ds[1:], True)):
        for cond in ("COUNT(*) > 200 AND AVG(m) > -5000 AND MAX(m) >= -3000", "SUM(m) < 0 OR AVG(m) > 100 OR MAX(m) < -3000",
                     "NOT MAX(m) = 3000 AND COUNT(*) BETWEEN 20 AND 10000 OR AVG(m) = 0"):
            q = sql.parse(f"SELECT k, k2, COUNT(*), SUM(m) FROM t GROUP BY k, k2 HAVING {cond} ORDER BY {order} LIMIT 3",
                          num_groups_limit=1_000_000)
            table = final_table(oracle, segs, q)
            want = expected_rows(q, table, trim)
            got = got_rows(segs[0], q, execute(pm, devs, q, merge, trim))
            assert_same(got, want, f"merge={merge} trim={trim} {cond} ORDER BY {order}")


def test_large_results_over_the_speculative_bound(pm, ctx):
    """A 1 M-key space (worst-case block far above 512 KB): HAVING keeping ~1 %, ~50 %, all and none of the groups, with and
    without ORDER BY ... LIMIT, against the same submission without HAVING filtered in Python."""
    segs = [IndexSegment.synthetic(ctx, f"hv{i}", 2_000_000, [{"name": "g", "cardinality": 1_000_000, "seed": 31 + i},
                                                             {"name": "v", "cardinality": 1000, "seed": 77 + i}])
            for i in range(2)]
    try:
        base = "SELECT SUM(v), COUNT(*) FROM t GROUP BY g"
        full = pm.execute_segments(segs, sql.parse(base, num_groups_limit=2_000_000), merge=True)[0]
        keys = np.asarray(full.keys[:, 0]).copy()
        counts = np.asarray(full.longs[1]).copy()
        sums = np.asarray(full.doubles[0]).copy()
        k99 = int(np.percentile(counts, 99))
        k50 = int(np.median(counts))
        for cond, sel in ((f"COUNT(*) > {k99}", counts > k99), (f"COUNT(*) > {k50}", counts > k50),
                          ("COUNT(*) >= 1", counts >= 1), ("COUNT(*) > 1000000", counts > 1_000_000)):
            q = sql.parse(f"{base} HAVING {cond}", num_groups_limit=2_000_000)
            got = pm.execute_segments(segs, q, merge=True)[0]
            assert got.num_groups == int(sel.sum()), cond
            assert np.array_equal(np.asarray(got.keys[:, 0]), keys[sel]), cond
            assert np.array_equal(np.asarray(got.doubles[0]), sums[sel]), cond
            q = sql.parse(f"{base} HAVING {cond} ORDER BY SUM(v) DESC LIMIT 10", num_groups_limit=2_000_000)
            top = pm.execute_segments(segs, q, merge=True)[0]
            idx = np.nonzero(sel)[0]
            order = sorted(idx.tolist(), key=lambda g: (-sums[g], int(keys[g])))[:5000]
            assert [int(keys[g]) for g in order] == [int(x) for x in top.keys[:, 0]], cond
    finally:
        for s in segs:
            s.destroy()


def test_filter_clause_results_are_filtered_after_alignment(oracle, pm, data):
    hs, ds = data
    texts = ["SELECT k, COUNT(*), SUM(m) FILTER (WHERE w < 5) FROM t GROUP BY k HAVING SUM(m) > 0",   # hidden unfiltered SUM
             "SELECT k, COUNT(*), SUM(m) FILTER (WHERE w < 5) FROM t GROUP BY k HAVING COUNT(*) > 250 ORDER BY COUNT(*) DESC LIMIT 2"]
    for text in texts:
        q = sql.parse(text, num_groups_limit=1_000_000)
        for segs, devs, merge in (([hs[0]], [ds[0]], False), (hs[1:4], ds[1:4], True)):
            want = expected_rows(q, final_table(oracle, segs, q), 5000 if merge else 0)
            got = got_rows(segs[0], q, execute(pm, devs, q, merge))
            assert 0 < len(want) < len(final_table(oracle, segs, q)), text
            assert_same(got, want, f"FILTER merge={merge}: {text}")


def test_star_tree_results_are_filtered_on_the_host(oracle, ctx, pm):
    rng = np.random.default_rng(6)
    n = 30_000
    seg = oracle.build_segment("hvst", {"d1": rng.integers(0, 60, size=n).astype(np.int32),
                                        "d2": rng.integers(0, 4, size=n).astype(np.int32),
                                        "m": rng.integers(-5, 6, size=n).astype(np.int32) * 100})
    st = stb.build_star_tree(seg, ["d1", "d2"], [("COUNT", None), ("SUM", "m"), ("MAX", "m"), ("MIN", "m")], max_leaf_records=10)
    dev = to_device(ctx, seg)
    try:
        nd = len(st.dimensions)
        dev.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                             [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
        for tail in ("HAVING COUNT(*) > 125", "HAVING SUM(m) < 0 AND NOT MAX(m) = 400",
                     "HAVING AVG(m) BETWEEN -10 AND 10 ORDER BY AVG(m) DESC LIMIT 2"):
            q = sql.parse(f"SELECT COUNT(*), SUM(m), MIN(m), MAX(m), AVG(m) FROM t GROUP BY d1, d2 {tail}")
            table = final_table(oracle, [seg], q)
            want = expected_rows(q, table, 0)
            assert 0 < len(want) < len(table), tail
            block = execute(pm, [dev], q)
            assert block.operator_kind == "STAR_TREE"
            assert_same(got_rows(seg, q, block), want, f"star-tree {tail}")
    finally:
        dev.destroy()


@pytest.mark.parametrize("dtype", [sb.DOUBLE, sb.FLOAT], ids=["DOUBLE", "FLOAT"])
def test_float_edge_values(oracle, ctx, pm, dtype):
    """NaN, -0.0 and +-inf in SUM / MIN / MAX / AVG / PERCENTILE: NaN passes only != and NOT IN, -0.0 equals 0."""
    pats = PATTERNS if dtype == sb.DOUBLE else [fr.F_NAN, fr.F_NEG_NAN, fr.F_PAYLOAD_NAN, fr.F_SIGNALLING_NAN]
    h = edge_segment(oracle, "hvfe", 20_001, 1, dtype, pats, pats[0])
    d = to_device(ctx, h)
    try:
        for cond in ("SUM(x) != 0", "SUM(x) = 0", "SUM(x) < 0", "SUM(x) NOT IN (0, 1.0e400)", "MIN(x) = 0", "MIN(x) >= -0.0",
                     "MAX(x) = 1.0e400", "MAX(x) < 1.0e400", "NOT MAX(x) > 0", "AVG(x) IN (0, 1.0e400)",
                     "PERCENTILE(x, 50) <> 0.25", "MIN(x) BETWEEN -2.5 AND 0 OR SUM(x) > 5"):
            q = sql.parse(f"SELECT g, COUNT(*) FROM t GROUP BY g HAVING {cond}", num_groups_limit=1_000_000)
            table = fr.reference(oracle, [h], q)
            finals = {k: [fr.final(a.function, v) for a, v in zip(q.aggregations, vals)] for k, vals in table.items()}
            want = sorted(k for k, v in finals.items() if having_ref(q, q.having, v))
            got = product_table(d, q, pm.execute_segments([d], q)[0])
            assert sorted(got) == want, (cond, sorted(got), want)
    finally:
        d.destroy()


def test_groups_limit_is_checked_before_having(pm, data):
    hs, ds = data
    q = sql.parse("SELECT k, COUNT(*) FROM t GROUP BY k, k2 HAVING COUNT(*) > 100000", num_groups_limit=10)
    for devs, merge in (([ds[0]], False), (ds[1:], True)):
        with pytest.raises(_lib.UnsupportedQueryError) as e:
            execute(pm, devs, q, merge)
        assert e.value.code == _lib.E_LIMIT


def test_refusals(pm, ctx, data):
    hs, ds = data
    q = sql.parse("SELECT k, COUNT(*), SUM(m) FROM t GROUP BY k HAVING COUNT(*) > 3")
    hav = having_spec(q)
    L = ctx.lib

    def call(qq, h, devs, merge=0, reduce_world=0):
        hq, _keep = _marshal_query(qq, merge, reduce_world=reduce_world)
        n = len(devs)
        segs = (C.c_void_p * n)(*[d.handle for d in devs])
        res, kinds = (C.c_void_p * n)(), (C.c_int32 * n)()
        rc = L.pb200h_execute_having(ctx.handle, C.byref(hq), None, None, C.byref(h), segs, n, res, kinds)
        assert rc != 0
        return rc

    assert call(q, hav, ds[1:3]) == _lib.E_INVALID                       # two per-segment results
    assert call(q, hav, ds[1:3], merge=2, reduce_world=1) == _lib.E_UNSUPPORTED
    assert call(q, hav, ds[1:3], merge=1, reduce_world=2) == _lib.E_UNSUPPORTED
    qa = sql.parse("SELECT COUNT(*), SUM(m) FROM t")
    assert call(qa, hav, [ds[0]]) == _lib.E_INVALID                       # no group-by
    bad = _lib.Having(1, 0)
    bad.nodes[0] = _lib.HavingNode(_lib.HAVING_CODES["EQ"], 0, 5, 0, 1.0, 0.0)
    assert call(q, bad, [ds[0]]) == _lib.E_INVALID                        # aggregation out of range
    bad.nodes[0] = _lib.HavingNode(_lib.HAVING_CODES["EQ"], 0, 0, 0, math.nan, 0.0)
    assert call(q, bad, [ds[0]]) == _lib.E_INVALID                        # NaN bound
    bad.num_nodes = 33
    assert call(q, bad, [ds[0]]) == _lib.E_INVALID
    # the device entry point: same checks
    dq = _lib.Query()
    dq.num_group_by, dq.num_aggs = 0, 1
    res = (C.c_void_p * 1)()
    assert L.pb200_execute_having(ctx.handle, C.byref(dq), None, None, C.byref(hav), None, 0, res) == _lib.E_INVALID
    # a result filtered by HAVING is final: it has no server DataTable
    block = pm.execute_segments(ds[1:4], q, merge=True, keep_handle=True, defer=False)[0]
    try:
        with pytest.raises(_lib.UnsupportedQueryError):
            pm.to_datatable(ds[1], q, block)
    finally:
        block.release(pm.ctx)
    # a merged deferred call with HAVING is refused, not silently unfiltered
    with pytest.raises(_lib.UnsupportedQueryError):
        pm.execute_segments(ds[1:3], q, merge=True, keep_handle=True)


def test_cli_host_merge_and_device_merge_agree(oracle, tmp_path, capsys):
    import segment_dir_util as sdu
    rng = np.random.default_rng(8)
    dirs = []
    for i in range(3):
        n = 20_000 + 1_000 * i
        cols = {"k": rng.integers(0, 300, size=n).astype(np.int32), "m": rng.integers(-50, 50, size=n).astype(np.int32)}
        seg = oracle.build_segment(f"hvcli{i}", cols)
        d = tmp_path / f"s{i}"
        sdu.write_segment_dir(str(d), seg)
        dirs.append(str(d))
    text = ("SELECT k, SUM(m) FROM t GROUP BY k HAVING COUNT(*) > 200 AND AVG(m) < 0 ORDER BY SUM(m) DESC, k LIMIT 15")
    args = ["--json"] + [x for d in dirs for x in ("--segment-dir", d)] + [text]
    import json
    outs = []
    for extra in ([], ["--merge-on-device"]):
        assert cli.main(extra + args) == 0
        outs.append(json.loads(capsys.readouterr().out))
    assert outs[0]["columns"] == outs[1]["columns"] == ["k", "sum(m)"]
    assert outs[0]["rows"] == outs[1]["rows"]
    assert 0 < len(outs[0]["rows"]) <= 15

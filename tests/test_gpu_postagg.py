"""-m gpu: GROUP BY ... ORDER BY arithmetic over aggregations (post-aggregation expressions such as SUM(m) / COUNT(*)),
ordered and trimmed by the library (pb200h_execute_post), against the exact reference.

The reference takes the exact per-group table (tests/exact_ref.py through test_gpu_having.final_table: sums of INT columns
are exact integers, rounded to a double once), computes each expression with Python floats (query.post_eval: one IEEE
operation per operator, Java's division by zero), orders the rows in Double.compare order with ties by the key values
ascending, and trims them.  Rows are compared key by key and value by value, bit for bit (all NaNs are one value)."""
import ctypes as C
import json
import math
import struct

import numpy as np
import pytest

import segment_dir_util as sdu
from gpu_util import to_device
from loopback_dist import run_ranks, values
from oracle import startree_builder as stb
from pinot_b200 import _lib, cli, sql
from pinot_b200.distributed import execute_and_combine
from pinot_b200.plan_maker import (B200Context, B200PlanMaker, DictionaryDomain, IndexSegment, _marshal_query, _read_result,
                                   order_spec, post_spec)
from pinot_b200.query import post_eval, value_order
from test_gpu_combine_loopback import Cluster, RecordingBackend
from test_gpu_combine_loopback import device_rows as combined_rows
from test_gpu_having import KNOB_ROUTES, final_table, got_rows, route
from test_gpu_order_by import _segment

pytestmark = pytest.mark.gpu

# m: multiples of 1000 around 0 (zero, negative and positive sums); t3 in 0..2; w in 0..9; c a DISTINCTCOUNT column
EXPRS = ["SUM(m) / COUNT(*)",
         "SUM(m) / SUM(t3)",
         "-SUM(m) * 0.5 + 3",
         "COUNT(*) * 100.0 / SUM(w)",
         "SUM(m) / (SUM(t3) - SUM(t3))",     # +inf, -inf and NaN (0 / 0)
         "-(SUM(m) * 0)",                    # -0.0 and 0.0
         "MAX(m) - MIN(t3) + AVG(m)",
         "DISTINCTCOUNT(c) / COUNT(*)"]


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
    hs = [_segment(oracle, n, 470 + i) for i, n in enumerate(sizes)]
    ds = [to_device(ctx, s) for s in hs]
    domain = DictionaryDomain.build(ctx, ds[1:], ["k", "k2", "m", "c", "t3"])
    for d in ds[1:]:
        d.bind_domain(domain)
    yield hs, ds
    for d in ds:
        d.destroy()
    domain.release()


# ------------------------------------------------------------------------------------------------ reference
def _same(x, y):
    return (math.isnan(x) and math.isnan(y)) or struct.pack("<d", x) == struct.pack("<d", y)


def expected_rows(q, table, trim):
    """[(key, finals)] in ORDER BY order (Double.compare, ties by the key values ascending), trimmed (trim <= 0: all)."""
    rows = sorted(table.items())
    for kind, index, asc in reversed(sql.resolve_order_by(q)):
        if kind == "GROUP_BY":
            rows.sort(key=lambda r: r[0][index], reverse=not asc)
        elif kind == "POST":
            program = q.post_aggregations[index].program
            rows.sort(key=lambda r: value_order(post_eval(program, lambda a: r[1][a])), reverse=not asc)
        else:
            rows.sort(key=lambda r: value_order(float(r[1][index])), reverse=not asc)
    return rows[:trim] if trim > 0 else rows


def assert_same(got, want, what):
    assert [g[0] for g in got] == [w[0] for w in want], (what, len(got), len(want))
    for g, w in zip(got, want):
        assert all(_same(x, y) for x, y in zip(g[1], w[1])), (what, g, w)


def execute(pm, devs, q, merge=False, trim=None, defer=False):
    """pb200h_execute_post with the query's ORDER BY (an explicit trim when given; deferred: merge_segments 2 and
    reduce_world 1, then pb200_result_finalize) -> one block per result."""
    ctx = pm.ctx
    spec, post = order_spec(q, merge), post_spec(q)
    if trim is not None:
        spec.trim_size = trim
    hq, _keep = _marshal_query(q, 2 if defer else merge, reduce_world=1 if defer else 0)
    n = len(devs)
    nres = 1 if merge else n
    segs = (C.c_void_p * n)(*[d.handle for d in devs])
    res, kinds = (C.c_void_p * nres)(), (C.c_int32 * n)()
    args = (_lib.HAggArg * len(q.aggregations))()
    _lib.check(ctx.lib.pb200h_execute_post(ctx.handle, C.byref(hq), C.byref(spec), args, None,
                                           C.byref(post) if post is not None else None, segs, n, res, kinds))
    if defer:
        _lib.check(ctx.lib.pb200_result_finalize(ctx.handle, res[0]))
    return [_read_result(ctx, C.c_void_p(res[i]), q, kinds[0 if merge else i], False) for i in range(nres)]


def parse(text, **kw):
    return sql.parse(text, num_groups_limit=1_000_000, **kw)


class Tables:
    """final_table per aggregation list, computed once per segment set."""

    def __init__(self, oracle):
        self.oracle, self.cache = oracle, {}

    def __call__(self, segs, q):
        key = (tuple(id(s) for s in segs), tuple((a.function, a.column, a.arg, repr(a.filter)) for a in q.aggregations))
        if key not in self.cache:
            self.cache[key] = final_table(self.oracle, segs, q)
        return self.cache[key]


@pytest.fixture(scope="module")
def tables(oracle):
    return Tables(oracle)


def check_exprs(pm, tables, segs, devs, merge, what, trim=0, group_by="k, k2"):
    for expr in EXPRS:
        for direction in ("", " DESC"):
            text = f"SELECT {group_by}, {expr} FROM t GROUP BY {group_by} ORDER BY {expr}{direction}, k LIMIT 3"
            q = parse(text)
            blocks = execute(pm, devs, q, merge, trim)
            if merge:
                assert_same(got_rows(segs[0], q, blocks[0]), expected_rows(q, tables(segs, q), trim), f"{what}: {text}")
            else:
                for s, b in zip(segs, blocks):
                    assert_same(got_rows(s, q, b), expected_rows(q, tables([s], q), trim), f"{what}: {text}")


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("route_name", list(KNOB_ROUTES))
def test_every_table_route(pm, ctx, tables, data, route_name):
    hs, ds = data
    with route(ctx, KNOB_ROUTES[route_name]):
        check_exprs(pm, tables, [hs[0]], [ds[0]], False, route_name)
        check_exprs(pm, tables, [hs[0]], [ds[0]], False, route_name + " trim 7", trim=7)


def test_merged_over_17_segments(pm, tables, data):
    hs, ds = data
    check_exprs(pm, tables, hs[1:], ds[1:], True, "merged 17", trim=5000)
    check_exprs(pm, tables, hs[1:], ds[1:], True, "merged 17 trim 4", trim=4)


def test_per_segment_results(pm, tables, data):
    hs, ds = data
    check_exprs(pm, tables, hs[1:4], ds[1:4], False, "per segment")


def test_deferred_result_is_ordered_when_finalized(pm, tables, data):
    hs, ds = data
    for expr in EXPRS[:4]:
        q = parse(f"SELECT k, k2, {expr} FROM t GROUP BY k, k2 ORDER BY {expr} DESC LIMIT 3")
        got = got_rows(hs[1], q, execute(pm, ds[1:], q, True, 9, defer=True)[0])
        assert_same(got, expected_rows(q, tables(hs[1:], q), 9), f"deferred {expr}")


def test_several_items_with_ties(pm, tables, data):
    """An expression item next to key and aggregation items; DISTINCTCOUNT / COUNT and COUNT / COUNT have many ties."""
    hs, ds = data
    for order in ("DISTINCTCOUNT(c) / COUNT(*) DESC, SUM(m) / COUNT(*), k2 DESC",
                  "COUNT(*) / COUNT(*), k DESC, SUM(t3) * 2 - COUNT(*)",
                  "MAX(m), SUM(m) / COUNT(*) DESC"):
        select = ", ".join(dict.fromkeys(x.strip().rsplit(" DESC", 1)[0] for x in order.split(",")))
        q = parse(f"SELECT k, k2, {select} FROM t GROUP BY k, k2 ORDER BY {order} LIMIT 2")
        for segs, devs, merge in (([hs[0]], [ds[0]], False), (hs[1:], ds[1:], True)):
            got = got_rows(segs[0], q, execute(pm, devs, q, merge, 11)[0])
            assert_same(got, expected_rows(q, tables(segs, q), 11), f"merge={merge} ORDER BY {order}")


def test_expression_orders_like_avg(pm, ctx, tables, data):
    """ORDER BY SUM(m) / COUNT(*) returns AVG(m)'s rows in AVG(m)'s order, on every route (m is INT: exact sums)."""
    hs, ds = data

    def keys(blocks, segs, q):
        return [[k for k, _ in got_rows(s, q, b)] for s, b in zip(segs, blocks)]
    for direction in ("", " DESC"):
        qe = parse(f"SELECT k, k2, SUM(m) / COUNT(*) FROM t GROUP BY k, k2 ORDER BY SUM(m) / COUNT(*){direction} LIMIT 3")
        qa = parse(f"SELECT k, k2, AVG(m) FROM t GROUP BY k, k2 ORDER BY AVG(m){direction} LIMIT 3")
        for name, knobs in KNOB_ROUTES.items():
            with route(ctx, knobs):
                for trim in (0, 5):
                    assert keys(execute(pm, [ds[0]], qe, False, trim), [hs[0]], qe) == \
                        keys(execute(pm, [ds[0]], qa, False, trim), [hs[0]], qa), (name, trim, direction)
        for devs, segs, merge in ((ds[1:], hs[1:], True), (ds[1:4], hs[1:4], False)):
            assert keys(execute(pm, devs, qe, merge, 15), segs[:1] if merge else segs, qe) == \
                keys(execute(pm, devs, qa, merge, 15), segs[:1] if merge else segs, qa), (merge, direction)


def test_filter_clause_operand(pm, tables, data):
    """FILTER-clause results are aligned on the host and ordered there by the same evaluator."""
    hs, ds = data
    for text in ["SELECT k, SUM(m) FILTER (WHERE w < 5) / COUNT(*) FROM t GROUP BY k "
                 "ORDER BY SUM(m) FILTER (WHERE w < 5) / COUNT(*) DESC LIMIT 2",
                 "SELECT k, COUNT(*), SUM(m) / SUM(m) FILTER (WHERE w < 5) FROM t GROUP BY k "
                 "ORDER BY SUM(m) / SUM(m) FILTER (WHERE w < 5), COUNT(*) LIMIT 2"]:
        q = parse(text)
        for segs, devs, merge in (([hs[0]], [ds[0]], False), (hs[1:4], ds[1:4], True)):
            got = got_rows(segs[0], q, execute(pm, devs, q, merge)[0])
            assert_same(got, expected_rows(q, tables(segs, q), 5000 if merge else 0), f"FILTER merge={merge}: {text}")


def test_star_tree_results_are_ordered_on_the_host(oracle, ctx, pm):
    rng = np.random.default_rng(16)
    n = 30_000
    seg = oracle.build_segment("past", {"d1": rng.integers(0, 60, size=n).astype(np.int32),
                                        "d2": rng.integers(0, 4, size=n).astype(np.int32),
                                        "m": rng.integers(-5, 6, size=n).astype(np.int32) * 100})
    st = stb.build_star_tree(seg, ["d1", "d2"], [("COUNT", None), ("SUM", "m"), ("MAX", "m"), ("MIN", "m")], max_leaf_records=10)
    dev = to_device(ctx, seg)
    try:
        nd = len(st.dimensions)
        dev.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                             [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
        for expr in ("SUM(m) / COUNT(*)", "(MAX(m) - MIN(m)) / SUM(m)", "-SUM(m) * 0"):
            for direction in ("", " DESC"):
                q = sql.parse(f"SELECT d1, d2, {expr} FROM t GROUP BY d1, d2 ORDER BY {expr}{direction} LIMIT 4")
                block = execute(pm, [dev], q, False, 20)[0]
                assert block.operator_kind == "STAR_TREE"
                assert_same(got_rows(seg, q, block), expected_rows(q, final_table(oracle, [seg], q), 20), f"star-tree {q.order_by}")
        # the same order as AVG on the star-tree route
        qe = sql.parse("SELECT d1, d2, SUM(m) / COUNT(*) FROM t GROUP BY d1, d2 ORDER BY SUM(m) / COUNT(*) DESC LIMIT 4")
        qa = sql.parse("SELECT d1, d2, AVG(m) FROM t GROUP BY d1, d2 ORDER BY AVG(m) DESC LIMIT 4")
        assert [k for k, _ in got_rows(seg, qe, execute(pm, [dev], qe)[0])] == [k for k, _ in got_rows(seg, qa, execute(pm, [dev], qa)[0])]
    finally:
        dev.destroy()


def test_edge_values(oracle, ctx, pm):
    """Groups whose expression is +inf, -inf, NaN, -0.0 and 0.0, in both directions and under a trim."""
    g = np.repeat(np.arange(12), 3).astype(np.int32)
    a = np.array([1, 2, 3,  -1, -2, 0,  0, 0, 0,  5, -5, 0,  7, 0, 0,  -7, 0, 0,
                  0, 0, 0,  4, 4, 4,  -3, 3, 0,  2, 0, 0,  -2, 0, 0,  9, 9, 9], dtype=np.int32)
    b = np.array([0, 0, 0,  0, 0, 0,  0, 0, 0,  1, 1, 0,  1, -1, 0,  2, 0, 0,
                  -1, 0, 0,  1, 1, 1,  0, 0, 0,  1, 0, 0,  -1, 0, 0,  3, 3, 3], dtype=np.int32)
    seg = oracle.build_segment("paedge", {"g": g, "a": a, "b": b})
    dev = to_device(ctx, seg)
    try:
        for expr in ("SUM(a) / SUM(b)", "-SUM(a) / SUM(b)", "SUM(a) * -1", "SUM(a) / SUM(b) * 0", "0 - SUM(a) * SUM(b)"):
            for direction in ("", " DESC"):
                q = sql.parse(f"SELECT g, {expr} FROM t GROUP BY g ORDER BY {expr}{direction} LIMIT 5")
                table = final_table(oracle, [seg], q)
                values = [post_eval(q.post_aggregations[0].program, lambda x: v[x]) for v in table.values()]
                if expr == "SUM(a) / SUM(b)":
                    assert {math.inf, -math.inf} <= set(values) and any(math.isnan(v) for v in values)
                if expr == "SUM(a) / SUM(b) * 0":
                    assert any(v == 0 and math.copysign(1, v) < 0 for v in values) and any(v == 0 and math.copysign(1, v) > 0 for v in values)
                for trim in (0, 5):
                    got = got_rows(seg, q, execute(pm, [dev], q, False, trim)[0])
                    assert_same(got, expected_rows(q, table, trim), f"{expr}{direction} trim {trim}")
    finally:
        dev.destroy()


def test_trimmed_100k_groups(pm, ctx):
    """100 000 groups, LIMIT 10: the 5 000 kept rows are the first 5 000 of the full sort by the expression."""
    segs = [IndexSegment.synthetic(ctx, f"pa{i}", 2_000_000, [{"name": "g", "cardinality": 100_000, "seed": 61 + i},
                                                              {"name": "v", "cardinality": 1000, "seed": 97 + i}])
            for i in range(2)]
    try:
        full = pm.execute_segments(segs, parse("SELECT SUM(v), COUNT(*) FROM t GROUP BY g"), merge=True, ordered=False)[0]
        keys = [int(x) for x in full.keys[:, 0]]
        ratio = [float(s) / int(c) for s, c in zip(full.doubles[0], full.longs[1])]
        assert len(keys) == 100_000
        for direction, sign in (("DESC", -1), ("ASC", 1)):
            q = parse(f"SELECT SUM(v) / COUNT(*) FROM t GROUP BY g ORDER BY SUM(v) / COUNT(*) {direction} LIMIT 10")
            top = pm.execute_segments(segs, q, merge=True)[0]
            want = sorted(range(len(keys)), key=lambda i: (sign * ratio[i], keys[i]))[:5000]
            assert top.num_groups == 5000
            assert [keys[i] for i in want] == [int(x) for x in top.keys[:, 0]], direction
    finally:
        for s in segs:
            s.destroy()


def test_loopback_combine(oracle):
    """A deferred result applies the programs when pb200_result_combine extracts it (world 2, dense route)."""
    cl = Cluster(oracle, 2)
    try:
        for expr, direction in (("SUM(v) / COUNT(*)", "DESC"), ("SUM(v) * 3 - MAX(t3)", ""), ("COUNT(*) / SUM(t3)", "DESC")):
            text = f"SELECT k, j, {expr} FROM t GROUP BY k, j ORDER BY {expr} {direction}, k LIMIT 7"
            backends = [RecordingBackend(p) for p in cl.pms]

            def body(dist):
                r = dist.get_rank()
                return execute_and_combine(backends[r], cl.devs[r], parse(text), dist, dst=0)
            got = values(run_ranks(cl.world, body))[0]
            q = parse(text)
            assert all(b.routes == ["dense"] for b in backends), [b.routes for b in backends]
            want = expected_rows(q, final_table(oracle, cl.all_hosts, q), order_spec(q, merge=True).trim_size)
            rows = [(k, [float(x) for x in v]) for k, v in combined_rows(cl, q, got)]
            assert_same(rows, want, f"loopback {text}")
    finally:
        cl.close()


def test_refusals(pm, ctx, data):
    hs, ds = data
    L = ctx.lib
    q = parse("SELECT k, SUM(m) / COUNT(*) FROM t GROUP BY k ORDER BY SUM(m) / COUNT(*)")
    hq, _keep = _marshal_query(q, False)
    segs = (C.c_void_p * 1)(ds[0].handle)
    res, kinds = (C.c_void_p * 1)(), (C.c_int32 * 1)()
    args = (_lib.HAggArg * 2)()

    def call(spec, post):
        return L.pb200h_execute_post(ctx.handle, C.byref(hq), C.byref(spec), args, None, C.byref(post) if post is not None else None,
                                     segs, 1, res, kinds)
    spec = order_spec(q, False)

    def program(*nodes):
        p = _lib.PostAggs(1, 0)
        p.programs[0].num_nodes = len(nodes)
        for i, n in enumerate(nodes):
            p.programs[0].nodes[i] = _lib.PostNode(*n)
        return p
    AGG, LIT, ADD, DIV = (_lib.POST_CODES[k] for k in ("AGG", "LIT", "ADD", "DIV"))
    assert call(spec, program((AGG, 0, 0.0), (AGG, 1, 0.0), (DIV, 0, 0.0))) == 0
    pb = _read_result(ctx, C.c_void_p(res[0]), q, kinds[0], False)
    assert pb.num_groups > 0
    for bad in (program((AGG, 2, 0.0)),                                   # aggregation out of range
                program((LIT, 0, math.nan)), program((LIT, 0, math.inf)),  # non-finite literal
                program((AGG, 0, 0.0), (AGG, 1, 0.0)),                    # two values left
                program((AGG, 0, 0.0), (ADD, 0, 0.0)),                    # an operator without its operands
                program((9, 0, 0.0)),                                      # unknown op
                program()):                                                # no node
        assert call(spec, bad) == _lib.E_INVALID
    many = program((AGG, 0, 0.0))
    many.num_programs = 9
    assert call(spec, many) == _lib.E_INVALID
    far = order_spec(q, False)
    far.items[0].index = 1                                                 # names a program past num_programs
    assert call(far, program((AGG, 0, 0.0))) == _lib.E_INVALID
    # a POST item without programs: every other entry point refuses it
    assert L.pb200h_execute_ordered(ctx.handle, C.byref(hq), C.byref(spec), segs, 1, res, kinds) == _lib.E_INVALID
    # more than 6 aggregations, hidden operands included: the stock operator runs
    q7 = parse("SELECT k, SUM(m) / COUNT(*) + MAX(m) - MIN(m) + AVG(t3) + SUM(w) + MAX(w) FROM t GROUP BY k "
               "ORDER BY SUM(m) / COUNT(*) + MAX(m) - MIN(m) + AVG(t3) + SUM(w) + MAX(w)")
    assert len(q7.aggregations) == 7
    with pytest.raises(_lib.UnsupportedQueryError):
        pm.execute_segments([ds[0]], q7)


def test_cli_host_merge_and_device_merge_agree(oracle, tmp_path, capsys):
    rng = np.random.default_rng(18)
    dirs = []
    for i in range(3):
        n = 20_000 + 1_000 * i
        cols = {"k": rng.integers(0, 300, size=n).astype(np.int32), "m": rng.integers(-50, 50, size=n).astype(np.int32),
                "n": rng.integers(0, 3, size=n).astype(np.int32)}
        seg = oracle.build_segment(f"pacli{i}", cols)
        d = tmp_path / f"s{i}"
        sdu.write_segment_dir(str(d), seg)
        dirs.append(str(d))
    text = "SELECT SUM(m) / SUM(n), k, COUNT(*) FROM t GROUP BY k ORDER BY SUM(m) / SUM(n) DESC, k LIMIT 15"
    args = ["--json"] + [x for d in dirs for x in ("--segment-dir", d)] + [text]
    outs = []
    for extra in ([], ["--merge-on-device"]):
        assert cli.main(extra + args) == 0
        outs.append(json.loads(capsys.readouterr().out))
    assert outs[0]["columns"] == outs[1]["columns"] == ["divide(sum(m),sum(n))", "k", "count(*)"]
    assert outs[0]["rows"] == outs[1]["rows"] and len(outs[0]["rows"]) == 15

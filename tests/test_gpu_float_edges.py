"""-m gpu: FLOAT / DOUBLE columns holding NaN (several bit patterns), -0.0, 0.0 and +-inf, against tests/float_edges_ref.py.

Columns: stored dictionaries (scan and inverted; a sorted one in a segment of its own) whose NaN entry has the sign bit
set in one segment and not in another, and raw columns (PASS_THROUGH and LZ4) holding every NaN pattern, which get a
dictionary at load.  Groups are built to hit each rule of the contract: only NaN, NaN with finite rows, only -0.0, both
zeros, +inf with -inf, one infinity, finite rows.  MIN / MAX / PERCENTILE are compared bit for bit (a NaN as any NaN),
SUM / AVG by float_edges_ref.check_sum."""
import math
from fractions import Fraction

import numpy as np
import pytest

import float_edges_ref as fr
from gpu_util import to_device, tuned
from oracle import segment_builder as sb
from pinot_b200 import cli, sql
from pinot_b200._lib import UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from test_gpu_order_by import execute_ordered

pytestmark = pytest.mark.gpu

LZ4 = 3
GROUPS = 12


def edge_rows(n, seed, data_type, nan_bits):
    """(g, x): per group g the values of one rule; NaN rows take the patterns in `nan_bits`."""
    rng = np.random.default_rng(seed)
    dt = np.float32 if data_type == sb.FLOAT else np.float64
    nans = [fr.float_of(b) if data_type == sb.FLOAT else fr.double_of(b) for b in nan_bits]
    g = rng.integers(0, GROUPS, size=n).astype(np.int32)
    g[:GROUPS] = np.arange(GROUPS)
    finite = (rng.integers(-40, 40, size=n) / 4.0).astype(dt)
    x = finite.copy()
    pick = rng.integers(0, len(nans), size=n)
    nan_col = np.array(nans, dtype=dt)[pick]
    x[g == 0] = nan_col[g == 0]                                                   # only NaN
    m1 = (g == 1) & (rng.random(n) < 0.3)
    x[m1] = nan_col[m1]                                                           # NaN with finite rows
    x[g == 2] = dt(-0.0)                                                          # only -0.0
    x[g == 3] = np.where(rng.random(int((g == 3).sum())) < 0.5, dt(-0.0), dt(0.0))  # both zeros
    x[g == 4] = np.where(rng.random(int((g == 4).sum())) < 0.5, dt(np.inf), dt(-np.inf))  # +inf with -inf
    m5 = (g == 5) & (rng.random(n) < 0.2)
    x[m5] = dt(np.inf)                                                            # one infinity with finite rows
    return g, x


def edge_segment(oracle, name, n, seed, data_type, nan_bits, stored_nan, sort=False):
    g, x = edge_rows(n, seed, data_type, nan_bits)
    # both zeros and both infinities in groups 3 / 4 of every segment, whatever the draw
    idx3, idx4 = np.nonzero(g == 3)[0], np.nonzero(g == 4)[0]
    dt = x.dtype.type
    if len(idx3) >= 2:
        x[idx3[0]], x[idx3[1]] = dt(-0.0), dt(0.0)
    if len(idx4) >= 2:
        x[idx4[0]], x[idx4[1]] = dt(np.inf), dt(-np.inf)
    if sort:
        order = sorted(range(n), key=lambda i: fr.ORDER(float(x[i])))
        g, x = g[order], x[order]
    rng = np.random.default_rng(seed + 1)
    m = rng.integers(0, 10, size=n).astype(np.int32)
    stored = x.copy()
    stored[np.isnan(stored)] = fr.float_of(stored_nan) if data_type == sb.FLOAT else fr.double_of(stored_nan)
    ext = np.array([1e-45, -1e-45, 3.4e38, -3.4e38] if data_type == sb.FLOAT else [5e-324, -5e-324, 1.7e308, -1.7e308],
                   dtype=x.dtype)[rng.integers(0, 4, size=n)]
    cols = [sb.build_column("g", g), sb.build_column("m", m),
            fr.build_dict_column("x", stored),
            fr.build_dict_column("xi", stored, inverted=not sort, lib=oracle),
            fr.build_dict_column("ext", ext),
            sb.build_raw_column("xr", x), sb.build_raw_column("xz", x, compression=LZ4)]
    return sb.SegmentData(name, n, cols)


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


PATTERNS = [fr.D_NAN, fr.D_NEG_NAN, fr.D_PAYLOAD_NAN, fr.D_SIGNALLING_NAN]
F_PATTERNS = [fr.F_NAN, fr.F_NEG_NAN, fr.F_PAYLOAD_NAN, fr.F_SIGNALLING_NAN]


@pytest.fixture(scope="module", params=[sb.DOUBLE, sb.FLOAT], ids=["DOUBLE", "FLOAT"])
def segs(request, oracle, ctx):
    """Three segments of ragged sizes: stored NaN entries 0x7ff8.. / 0xfff8.. / 0x7ff8..; the last one sorted on x."""
    dt = request.param
    pats = PATTERNS if dt == sb.DOUBLE else F_PATTERNS
    hs = [edge_segment(oracle, "fe0", 20_001, 1, dt, pats, pats[0]),
          edge_segment(oracle, "fe1", 3_333, 2, dt, pats, pats[1]),
          edge_segment(oracle, "fe2", 997, 3, dt, pats[:2], pats[1], sort=True)]
    assert hs[2].column("x").is_sorted
    ds = [to_device(ctx, h) for h in hs]
    yield hs, ds
    for d in ds:
        d.destroy()


class _Values:
    def __init__(self, dev):
        self.dev, self.cache = dev, {}

    def __call__(self, column, dict_id):
        k = (column, int(dict_id))
        if k not in self.cache:
            self.cache[k] = self.dev.dictionary_value(column, int(dict_id))
        return self.cache[k]


def product_table(dev, q, b):
    value = _Values(dev)
    rows = 1 if b.num_groups < 0 else b.num_groups
    out = {}
    for g in range(rows):
        key = () if b.num_groups < 0 else tuple(fr.Key(value(c, b.keys[g, j])) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            fn = agg.function
            if fn == "COUNT":
                vals.append(int(b.longs[a][g]))
            elif fn == "AVG":
                vals.append((float(b.doubles[a][g]), int(b.longs[a][g])))
            elif fn == "DISTINCTCOUNT":
                dt = sb.FLOAT if dev.column_info(agg.column)["data_type"] == sb.FLOAT else sb.DOUBLE
                vals.append(frozenset(fr.identity(value(agg.column, d), dt) for d in b.distinct[(a, g)]))
            else:
                vals.append(float(b.doubles[a][g]))
        assert key not in out, f"group key {key} twice"
        out[key] = vals
    return out


def assert_matches(q, got, want, what):
    assert set(got) == set(want), (what, sorted(got), sorted(want))
    for key, wv in want.items():
        gv = got[key]
        for a, agg in enumerate(q.aggregations):
            fn, g, w = agg.function, gv[a], wv[a]
            if fn in ("COUNT", "DISTINCTCOUNT"):
                assert g == w, (what, key, fn, g, w)
            elif fn == "SUM":
                assert fr.check_sum(g, w), (what, key, fn, g, w)
            elif fn == "AVG":
                assert g[1] == w[1] and fr.check_sum(g[0], w[0]), (what, key, fn, g, w)
            else:
                assert fr.check_value(g, w), (what, key, str(agg), float(g).hex(), float(w).hex())


_REFERENCE = {}


def reference(oracle, h, q, text):
    """fr.reference of one segment, once per (segment, query): the routes share it."""
    key = (h.name, h.column("x").data_type, text)
    if key not in _REFERENCE:
        _REFERENCE[key] = fr.reference(oracle, [h], q)
    return _REFERENCE[key]


def run(oracle, pm, h, d, text, what=""):
    q = sql.parse(text, num_groups_limit=1_000_000)
    b = pm.execute_segments([d], q)[0]
    assert_matches(q, product_table(d, q, b), reference(oracle, h, q, text), f"{what} {h.name}: {text}")
    return b


COLUMNS = ["x", "xi", "xr", "xz"]


@pytest.mark.parametrize("route", ["default", "global", "hash", "sparse_0", "per_row"])
def test_aggregations_per_rule(oracle, ctx, pm, segs, route):
    knobs = {"default": {}, "global": {"smem_groups": 0}, "hash": {"dense_max": 1}, "sparse_0": {"sparse_max": 0},
             "per_row": {"sparse_max_agg": 32}}[route]
    hs, ds = segs
    with tuned(ctx, **knobs):
        for h, d in zip(hs, ds):
            for c in COLUMNS:
                aggs = f"COUNT(*), SUM({c}), AVG({c}), MIN({c}), MAX({c}), DISTINCTCOUNT({c})"
                for tail in ("", " GROUP BY g", " WHERE m < 7 GROUP BY g"):
                    run(oracle, pm, h, d, f"SELECT {aggs} FROM t{tail}", route)
                run(oracle, pm, h, d, f"SELECT COUNT(*), SUM(m), MIN(ext), MAX(ext) FROM t GROUP BY {c}", route)
                for p in (0, 50, 100):
                    run(oracle, pm, h, d, f"SELECT PERCENTILE({c}, {p}), MIN({c}) FROM t GROUP BY g", route)
                    run(oracle, pm, h, d, f"SELECT PERCENTILE({c}, {p}) FROM t", route)
            run(oracle, pm, h, d, "SELECT MIN(ext), MAX(ext), COUNT(*) FROM t GROUP BY g", route)


def test_non_scan_shortcut(oracle, pm, segs):
    """MIN / MAX / DISTINCTCOUNT without a filter come from the dictionary: its first / last entry, its size."""
    hs, ds = segs
    for h, d in zip(hs, ds):
        for c in COLUMNS:
            b = run(oracle, pm, h, d, f"SELECT MIN({c}), MAX({c}), DISTINCTCOUNT({c}), COUNT(*) FROM t")
            assert math.isnan(float(b.doubles[1][0]))


def _pred_text(c, p):
    def lit(v):
        return repr(float(v)) if isinstance(v, float) else str(v)
    if p.type == "RANGE":
        parts = []
        if p.lower is not None:
            parts.append(f"{c} {'>=' if p.lower_inclusive else '>'} {lit(p.lower)}")
        if p.upper is not None:
            parts.append(f"{c} {'<=' if p.upper_inclusive else '<'} {lit(p.upper)}")
        return " AND ".join(parts)
    vs = ", ".join(lit(v) for v in p.values)
    return {"EQ": f"{c} = {vs}", "NEQ": f"{c} != {vs}", "IN": f"{c} IN ({vs})", "NOT_IN": f"{c} NOT IN ({vs})"}[p.type]


def test_filter_matrix(oracle, pm, segs):
    """Every predicate of the CPU matrix on stored (scan, inverted, sorted) and raw columns: the rows it selects are the
    reference's (the oracle's on a dictionary column, the value comparisons on a raw one)."""
    from pinot_b200.query import Predicate
    hs, ds = segs
    for h, d in zip(hs, ds):
        big = 1.7976931348623157e308 if h.column("x").data_type == sb.DOUBLE else 3.4028234663852886e38
        for c in COLUMNS:
            preds = [Predicate(t, c, [v]) for v in (0, -0.0, 1.5, big) for t in ("EQ", "NEQ")]
            preds += [Predicate("IN", c, [-0.0, 1.5]), Predicate("NOT_IN", c, [0, big])]
            preds += [Predicate("RANGE", c, [], lo, hi, li, ui) for lo, hi in ((-1.0, 1.0), (-0.0, 0.0), (0, None), (None, 0))
                      for li, ui in ((True, True), (False, False))]
            for p in preds:
                q = sql.parse(f"SELECT COUNT(*), SUM(m) FROM t WHERE {_pred_text(c, p)}")
                b = pm.execute_segments([d], q)[0]
                want = fr.reference(oracle, [h], q)
                assert_matches(q, product_table(d, q, b), want, f"{h.name} {_pred_text(c, p)}")


def _ordered_rows(dev, q, block):
    t = product_table(dev, q, block)
    value = _Values(dev)
    keys = [tuple(fr.Key(value(c, block.keys[g, j])) for j, c in enumerate(q.group_by)) for g in range(block.num_groups)]
    return [(k, t[k]) for k in keys]


@pytest.mark.parametrize("order", ["SUM(x)", "SUM(x) DESC", "AVG(xr)", "AVG(xr) DESC", "MIN(xz)", "MAX(x) DESC", "MAX(xi)"])
def test_order_by_aggregate_with_trim(oracle, pm, segs, order):
    """Rows ordered by a value that is NaN, +-inf or a zero in some groups; trims that end among them."""
    hs, ds = segs
    q = sql.parse(f"SELECT SUM(x), AVG(xr), MIN(xz), MAX(x), MAX(xi), COUNT(*) FROM t GROUP BY g ORDER BY {order} LIMIT 5")
    items = sql.resolve_order_by(q)
    for h, d in zip(hs, ds):
        want = fr.ordered(q, fr.reference(oracle, [h], q), items)
        for trim in (0, 1, 3, 5, 8):
            got = _ordered_rows(d, q, execute_ordered(pm, [d], q, trim)[0])
            kept = want if trim == 0 else want[:trim]
            assert [k for k, _ in got] == [k for k, _ in kept], (order, trim, h.name)


@pytest.mark.parametrize("order", ["x", "x DESC", "xr DESC", "xz"])
def test_order_by_float_key(oracle, pm, segs, order):
    hs, ds = segs
    col = order.split()[0]
    q = sql.parse(f"SELECT COUNT(*), SUM(m) FROM t GROUP BY {col} ORDER BY {order} LIMIT 5")
    items = sql.resolve_order_by(q)
    for h, d in zip(hs, ds):
        want = fr.ordered(q, fr.reference(oracle, [h], q), items)
        for trim in (0, 2, 4):
            got = _ordered_rows(d, q, execute_ordered(pm, [d], q, trim)[0])
            assert [k for k, _ in got] == [k for k, _ in (want if trim == 0 else want[:trim])], (order, trim, h.name)


def test_filter_clause_nan_sum_is_ordered_after_inf(oracle, pm, segs):
    """FILTER-clause results are aligned and ordered on the host: a NaN SUM is the largest value there too."""
    hs, ds = segs
    for desc in ("", " DESC"):
        q = sql.parse(f"SELECT SUM(x), SUM(x) FILTER (WHERE m < 5), COUNT(*) FROM t GROUP BY g ORDER BY SUM(x){desc}")
        items = sql.resolve_order_by(q)
        for h, d in zip(hs, ds):
            want = fr.ordered(q, fr.reference(oracle, [h], q), items)
            got = _ordered_rows(d, q, execute_ordered(pm, [d], q, 0)[0])
            assert [k for k, _ in got] == [k for k, _ in want], (desc, h.name)
            assert math.isnan(got[-1 if not desc else 0][1][0])


def test_domain_merge_and_cli(oracle, ctx, pm, segs):
    """Segments whose x dictionaries differ in their NaN bits, bound to one domain and merged on the device: the same
    groups and values as the reference over the union of their rows, and as the CLI's by-value merge."""
    hs, _ = segs
    texts = ["SELECT MIN(x), MAX(x), DISTINCTCOUNT(x), COUNT(*), SUM(x) FROM t GROUP BY g",
             "SELECT COUNT(*), SUM(m), MIN(ext) FROM t GROUP BY x",
             "SELECT MIN(xr), MAX(xr), DISTINCTCOUNT(xr), COUNT(*) FROM t"]
    for text in texts:
        q = sql.parse(text, num_groups_limit=1_000_000)
        want = fr.reference(oracle, hs, q)
        ds = [to_device(ctx, h) for h in hs]
        dom = None
        try:
            per_seg = pm.execute_segments(ds, q)
            table = cli.merge_blocks(q, ds, per_seg)
            got = {tuple(fr.Key(v) for v in k): vals for k, vals in table.items()}
            got = {k: [len(v) if a.function == "DISTINCTCOUNT" else v for a, v in zip(q.aggregations, vals)] for k, vals in got.items()}
            ref = {k: [len(v) if a.function == "DISTINCTCOUNT" else v for a, v in zip(q.aggregations, vals)] for k, vals in want.items()}
            assert_matches(q, got, ref, f"cli {text}")
            cols = [c for c in ("x", "xr", "ext") if c in text]
            dom = DictionaryDomain.build(ctx, ds, cols)
            for d in ds:
                d.bind_domain(dom)
            merged = pm.execute_segments(ds, q, merge=True)[0]
            assert_matches(q, product_table(ds[0], q, merged), want, f"domain {text}")
        finally:
            for d in ds:
                d.destroy()
            if dom is not None:
                dom.release()


def _matched_values(h, c, groups):
    g = fr.column_values(h, "g")
    return [float(v) for v in fr.column_values(h, c)[np.isin(g, groups)]]


def _assert_order(got, values, asc, limit, what):
    want = sorted(values, key=fr.ORDER, reverse=not asc)[:limit]
    assert [fr.identity(float(v)) for v in got] == [fr.identity(v) for v in want], what


def test_distinct_order(oracle, pm, segs):
    """SELECT DISTINCT x ORDER BY x, per segment and merged by value over segments whose NaN bits differ."""
    from pinot_b200.plan_maker import merge_distinct_blocks
    hs, ds = segs
    for c in ("x", "xr"):
        for asc in (True, False):
            q = sql.parse_distinct(f"SELECT DISTINCT {c} FROM t ORDER BY {c} {'ASC' if asc else 'DESC'} LIMIT 1000")
            for h, d in zip(hs, ds):
                b = pm.execute_distinct([d], q)[0]
                _assert_order(b.columns[0], fr.unique_values(fr.column_values(h, c), sb.DOUBLE), asc, 1000, (h.name, c, asc))
            union = np.concatenate([fr.column_values(h, c).astype(np.float64) for h in hs])
            merged = merge_distinct_blocks(pm.execute_distinct(ds, q), q.order_by, q.limit)
            _assert_order(merged.columns[0], fr.unique_values(union, sb.DOUBLE), asc, 1000, ("merged", c, asc))


def _selection_cases(hs, c):
    """(filter groups, LIMIT) pairs: one LIMIT ends inside the zeros, one inside the NaN rows (ASC) / the finite rows (DESC)."""
    zeros = [2, 3, 6]
    vals = [v for h in hs for v in _matched_values(h, c, zeros)]
    negatives = sum(1 for v in vals if v < 0 or fr.identity(v) == fr.identity(-0.0))
    edges = [0, 1, 4, 5]
    non_nan = sum(1 for h in hs for v in _matched_values(h, c, edges) if not math.isnan(v))
    return [(zeros, negatives + 7), (zeros, negatives - 7), (edges, non_nan + 5), (edges, 40)]


def _selection_check(pm, hs, ds, c, what):
    for groups, limit in _selection_cases(hs, c):
        for asc in (True, False):
            text = f"SELECT {c} FROM t WHERE g IN ({', '.join(map(str, groups))}) ORDER BY {c} {'ASC' if asc else 'DESC'} LIMIT {limit}"
            q = sql.parse_selection(text)
            merged = pm.execute_selection(ds, q, merge=True)
            _assert_order(merged.columns[0], [v for h in hs for v in _matched_values(h, c, groups)], asc, limit, (what, text))
            for h, d in zip(hs, ds):
                b = pm.execute_selection([d], q)[0]
                _assert_order(b.columns[0], _matched_values(h, c, groups), asc, limit, (what, h.name, text))


def test_selection_order(pm, segs):
    """SELECT x ... ORDER BY x LIMIT n, per segment and merged over the segments (the merge compares values on the
    host): -0.0 before 0.0, NaN after +inf, with LIMITs that end inside the zeros and inside the NaN rows."""
    hs, ds = segs
    for c in COLUMNS:
        _selection_check(pm, hs, ds, c, "dictionary")


def test_selection_order_raw_float_without_dictionary(ctx, pm, segs):
    """A raw FLOAT column loaded without a dictionary (raw_dict_max 0) is ordered by its 32-bit values: a NaN with the
    sign bit set must still sort after +inf."""
    hs, _ = segs
    if hs[0].column("xr").data_type != sb.FLOAT:
        pytest.skip("raw values are streamed for 4-byte columns only")
    with tuned(ctx, raw_dict_max=0):
        ds = [to_device(ctx, h) for h in hs]
    try:
        assert ds[0].column_info("xr")["has_dictionary"] == 0
        for c in ("xr", "xz"):
            _selection_check(pm, hs, ds, c, "raw")
    finally:
        for d in ds:
            d.destroy()


def _check_ordered(q, got_rows, want_rows, what):
    assert [k for k, _ in got_rows] == [k for k, _ in want_rows], what
    for (k, g), (_, w) in zip(got_rows, want_rows):
        for a, agg in enumerate(q.aggregations):
            if agg.function == "SUM":
                assert math.isnan(g[a]) if math.isnan(w[a]) else fr.same_double(g[a], w[a]), (what, k, g, w)
            elif agg.function == "COUNT":
                assert g[a] == w[a], (what, k, g, w)


def test_star_tree_nan_sum_is_ordered_on_the_host(oracle, ctx, pm, segs):
    """A star-tree result with a DOUBLE metric whose pre-aggregated SUMs are NaN (+inf with -inf, NaN rows), -0.0 and
    +-inf: its metric dictionary and the host ORDER BY follow Double.compare.  The finite values are quarters, so every
    sum is exact and compared bit for bit."""
    from oracle import startree_builder as stb
    hs, _ = segs
    h = hs[1]
    st = stb.build_star_tree(h, ["g", "m"], [("COUNT", None), ("SUM", "x")], max_leaf_records=10)
    dev = to_device(ctx, h)
    try:
        nd = len(st.dimensions)
        dev.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                             [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
        for order in ("SUM(x)", "SUM(x) DESC"):
            q = sql.parse(f"SELECT COUNT(*), SUM(x) FROM t GROUP BY g ORDER BY {order}")
            want = fr.ordered(q, fr.reference(oracle, [h], q), sql.resolve_order_by(q))
            for trim in (0, 3):
                block = execute_ordered(pm, [dev], q, trim)[0]
                assert block.operator_kind == "STAR_TREE"
                got = [(k, [v[0], v[1]]) for k, v in _ordered_rows(dev, q, block)]
                _check_ordered(q, got, want if trim == 0 else want[:trim], (order, trim))
    finally:
        dev.destroy()


@pytest.mark.parametrize("on_device", [False, True])
def test_cli_over_segment_directories(oracle, tmp_path, capsys, segs, on_device):
    """The command line over segment directories whose x dictionaries differ in their NaN bits: one row per value
    (one NaN, two zeros), in Double.compare order, with the reference's values."""
    import json

    from segment_dir_util import write_segment_dir
    hs, _ = segs
    dirs = [write_segment_dir(str(tmp_path / f"seg{i}"), h, "v1" if i == 0 else "v3") for i, h in enumerate(hs)]
    for order in ("x", "x DESC"):
        text = f"SELECT COUNT(*), SUM(x), MIN(xr), MAX(xr), DISTINCTCOUNT(xr) FROM t GROUP BY x ORDER BY {order} LIMIT 200"
        argv = [text, "--json"] + [a for d in dirs for a in ("--segment-dir", d)] + (["--merge-on-device"] if on_device else [])
        assert cli.main(argv) == 0
        out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
        q = sql.parse(text)
        want = fr.ordered(q, fr.reference(oracle, hs, q), sql.resolve_order_by(q))
        assert [fr.Key(float(r[0])) for r in out["rows"]] == [k[0] for k, _ in want], order
        for r, (k, w) in zip(out["rows"], want):
            assert r[1] == w[0], (k, r, w)
            assert math.isnan(r[2]) if math.isnan(w[1]) else fr.same_double(r[2], w[1]), (k, r, w)
            assert fr.check_value(r[3], w[2]) and fr.check_value(r[4], w[3]) and r[5] == w[4], (k, r, w)


def test_variance_refuses_non_finite_and_is_exact_at_zeros(oracle, ctx, pm, segs):
    hs, ds = segs
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([ds[0]], sql.parse("SELECT VAR_POP(x) FROM t"))
    n = 1000
    rng = np.random.default_rng(9)
    z = np.array([-0.0, 0.0, 1.0, 2.0, -0.0, 3.0], dtype=np.float64)[rng.integers(0, 6, size=n)]
    z[:2] = [-0.0, 0.0]
    seg = sb.SegmentData("zeros", n, [fr.build_dict_column("z", z)])
    dev = to_device(ctx, seg)
    try:
        b = pm.execute_segments([dev], sql.parse("SELECT VAR_POP(z) FROM t"))[0]
        xs = [Fraction(float(v)) for v in z]
        mean = sum(xs) / n
        assert float(b.doubles[0][0]) == float(sum((x - mean) ** 2 for x in xs) / n)
    finally:
        dev.destroy()

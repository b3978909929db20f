"""-m gpu: derived columns (single-column transforms) against an identity.  For an expression E over column c, the same
segment also stores a dictionary column `t` holding transform_ref(E, c) (tests/transform_ref.py, which shares no code
with the product), written by the oracle's segment writer without an inverted index.  Then:
  * the derived column IS `t`: its dictionary bytes and forward-index bytes equal t's byte for byte;
  * every query run with E returns exactly what the same query with `t` returns -- keys, every aggregate bit for bit
    (a SUM / AVG of doubles up to the order of its additions), group count and num_docs_scanned -- and the `t` query itself is held to the oracle and the exact references
    (gpu_util.check_query);
  * merged submissions over 17 segments (two launch chunks) with the source bound to a domain, and with the expression
    itself bound once the unbound dictionaries are refused; lazy and explicit derivation agree, a second query derives
    nothing, 12 threads deriving at once leave one column per segment; every refusal;
  * a source bound to a domain wider than the segment, DataTable bytes (the expression's name and result type), a
    star-tree segment answering an expression by the raw scan, and destroyed segments giving their derived memory back.
The expressions and data here produce no NaN and no -0.0: tests/test_gpu_transform_edges.py holds expressions that do
to a per-row reference."""
import threading

import numpy as np
import pytest

import transform_ref as ref
import datatable_util
from gpu_util import check_query, tuned
from oracle import startree_builder as stb
from pinot_b200 import sql
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED, Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain, IndexSegment
from pinot_b200.query import Aggregation, Predicate, QueryContext

pytestmark = pytest.mark.gpu

SIZES = [1, 31, 32, 8_193, 100_003]
TYPES = {"ts": "LONG", "i": "INT", "f": "FLOAT", "d": "DOUBLE", "r": "INT"}
# (expression, source): every function family, nested programs, non-monotone ones (mod, dayofweek, negative times)
EXPRS = [("datetrunc('HOUR',ts)", "ts"), ("datetrunc('WEEK',ts)", "ts"), ("datetrunc('MONTH',ts,'MILLISECONDS','UTC','DAYS')", "ts"),
         ("dayofweek(ts)", "ts"), ("year(ts)", "ts"), ("week(ts)", "ts"), ("hour(ts)", "ts"),
         ("timeconvert(ts,'MILLISECONDS','HOURS')", "ts"), ("toepochminutesbucket(ts,'15')", "ts"),
         ("mod(abs(ts),'10000')", "ts"), ("times(plus(i,'0.5'),'-3')", "i"), ("divide(i,'1000')", "i"),
         ("floor(divide(f,'100'))", "f"), ("plus(times(d,'0.1'),'0.7')", "d"), ("abs(r)", "r"), ("minute(i)", "i"),
         ("quarter(ts)", "ts"), ("month(ts)", "ts"), ("day(ts)", "ts"), ("dayofyear(ts)", "ts"), ("second(ts)", "ts"),
         ("millisecond(ts)", "ts"), ("datetrunc('MILLISECOND',i)", "i"), ("datetrunc('SECOND',ts)", "ts"),
         ("datetrunc('MINUTE',ts)", "ts"), ("datetrunc('DAY',ts)", "ts"), ("datetrunc('QUARTER',ts)", "ts"),
         ("datetrunc('YEAR',ts)", "ts"), ("toepochseconds(ts)", "ts"), ("toepochminutes(ts)", "ts"),
         ("toepochhours(ts)", "ts"), ("toepochdays(ts)", "ts"), ("toepochsecondsbucket(ts,'10')", "ts"),
         ("toepochhoursbucket(ts,'6')", "ts"), ("toepochdaysbucket(ts,'7')", "ts"), ("toepochsecondsrounded(ts,'10')", "ts"),
         ("toepochminutesrounded(ts,'5')", "ts"), ("toepochhoursrounded(ts,'3')", "ts"), ("toepochdaysrounded(ts,'7')", "ts"),
         ("ceil(divide(abs(d),'7'))", "d"), ("minus(i,'0.25')", "i"), ("minus('5',times(i,'3'))", "i"),
         ("mod(abs(f),'7')", "f"), ("year(timeconvert(i,'SECONDS','MILLISECONDS'))", "i")]


def _columns(n, seed):
    rng = np.random.default_rng(seed)
    return {"rid": np.arange(n, dtype=np.int32),
            "ts": rng.integers(-2_000_000_000, 1_800_000_000_000, size=n, dtype=np.int64),
            "i": rng.integers(-50_000_000, 50_000_000, size=n).astype(np.int32),
            "f": (rng.integers(-4000, 4000, size=n) / 8.0).astype(np.float32),
            "d": rng.integers(-6000, 6000, size=n) / 3.0,
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 7,
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "v": rng.integers(-1000, 1000, size=n).astype(np.int32),
            "s": np.array([b"a", b"ab", b"b"])[rng.integers(0, 3, size=n)]}


def _segment(oracle, cols, expr, src, name):
    cols = dict(cols)
    cols["t"] = ref.column(expr, cols[src], TYPES[src])
    return oracle.build_segment(name, cols, raw=["r"])


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def _block_bytes(b):
    """Everything of a block but its doubles, as bytes (the doubles: _assert_same)."""
    return (b.num_groups, b.stats.num_docs_scanned, np.asarray(b.keys).tobytes(), [np.asarray(x).tobytes() for x in b.longs],
            sorted((k, np.asarray(v).tobytes()) for k, v in b.distinct.items()))


def _assert_same(got, want, what):
    """Keys, counts, sets and statistics byte for byte; doubles too, except that a SUM / AVG of DOUBLE values may differ in
    its last bits between two runs of the same query (the device adds doubles in no fixed order; the `t` query is held to
    the gamma_n bound by check_query)."""
    assert _block_bytes(got) == _block_bytes(want), what
    for g, w in zip(got.doubles, want.doubles):
        g, w = np.asarray(g, dtype=np.float64), np.asarray(w, dtype=np.float64)
        assert g.tobytes() == w.tobytes() or np.allclose(g, w, rtol=1e-9, atol=0.0, equal_nan=True), what


def _swap(q: QueryContext, expr: str, name: str) -> QueryContext:
    """The same query with `name` in place of the expression wherever it appears."""
    sub = lambda c: name if c == expr else c  # noqa: E731
    def flt(f):
        if f is None:
            return None
        if isinstance(f, Predicate):
            return Predicate(f.type, sub(f.column), list(f.values), f.lower, f.upper, f.lower_inclusive, f.upper_inclusive)
        return type(f)(f.type, [flt(c) for c in f.children])
    aggs = [Aggregation(a.function, sub(a.column), arg=a.arg, filter=flt(a.filter)) for a in q.aggregations]
    return QueryContext(aggregations=aggs, filter=flt(q.filter), group_by=[sub(g) for g in q.group_by],
                        order_by=[(sub(e) if e == expr else e.replace(expr, name), asc) for e, asc in q.order_by], limit=q.limit)


def _queries(expr, t_values):
    mid = float(np.median(t_values)) if len(t_values) else 0.0
    if t_values.dtype.kind in "iu":
        mid = int(mid)
    where = Predicate("RANGE", expr, [], mid, None, True, True)
    return [
        QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v")], group_by=[expr]),
        QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("MAX", "v")], group_by=["g", expr], filter=where),
        QueryContext(aggregations=[Aggregation("SUM", expr), Aggregation("AVG", expr), Aggregation("MIN", expr),
                                   Aggregation("MAX", expr), Aggregation("DISTINCTCOUNT", expr)], group_by=["g"]),
        QueryContext(aggregations=[Aggregation("SUM", expr), Aggregation("MIN", expr), Aggregation("COUNT", None)], filter=where),
        QueryContext(aggregations=[Aggregation("PERCENTILE", expr, arg=90.0), Aggregation("COUNT", None)], group_by=["g"]),
        QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v", filter=where)], group_by=["g"]),
        QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v")], group_by=[expr],
                     order_by=[(expr, False)], limit=5),
    ]


@pytest.mark.parametrize("n", SIZES)
def test_identity(oracle, ctx, pm, n):
    base = _columns(n, n)
    for k, (expr, src) in enumerate(EXPRS):
        seg_data = _segment(oracle, base, expr, src, f"tr{n}_{k}")
        seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
        try:
            before = seg.device_bytes()
            col = seg.derive(expr)
            assert col == len(seg.column_names)                       # the first derived column, after the stored ones
            assert seg.column_info(expr)["bits"] == seg.column_info("t")["bits"], expr
            for which in ("dict", "fwd"):
                assert seg.read_index(expr, which).tobytes() == seg.read_index("t", which).tobytes(), (expr, n, which)
            assert seg.device_bytes() > before
            for q in _queries(expr, ref.column(expr, base[src], TYPES[src])):
                tq = _swap(q, expr, "t")
                got = pm.execute_segments([seg], q)[0]
                want = pm.execute_segments([seg], tq)[0]
                _assert_same(got, want, (expr, n, q))
                assert got.operator_kind == want.operator_kind or want.operator_kind == "NON_SCAN_AGGREGATION", (expr, n)
            check_query(oracle, pm, seg_data, seg, _swap(_queries(expr, base[src])[0], expr, "t"), f"{expr} n={n}")
            # selection and DISTINCT: the same rows and values
            sel = sql.SelectionQuery(columns=[expr, "rid"], order_by=[(expr, False), ("rid", True)], limit=50)
            tsel = sql.SelectionQuery(columns=["t", "rid"], order_by=[("t", False), ("rid", True)], limit=50)
            a, b = pm.execute_selection([seg], sel)[0], pm.execute_selection([seg], tsel)[0]
            assert [np.asarray(x).tobytes() for x in a.columns] == [np.asarray(x).tobytes() for x in b.columns], expr
            dq = sql.DistinctQuery(columns=[expr], order_by=[(expr, True)], limit=20)
            tdq = sql.DistinctQuery(columns=["t"], order_by=[("t", True)], limit=20)
            a, b = pm.execute_distinct([seg], dq)[0], pm.execute_distinct([seg], tdq)[0]
            assert [np.asarray(x).tobytes() for x in a.columns] == [np.asarray(x).tobytes() for x in b.columns], expr
            # a second query derives nothing
            again = seg.device_bytes()
            pm.execute_segments([seg], _queries(expr, base[src])[0])
            assert seg.device_bytes() == again and seg.derive(expr) == col and seg.column_index(expr) == col
        finally:
            seg.destroy()


def test_routes(oracle, ctx, pm):
    """The specialised shared-table route and the hash table (dense_max 1) serve a derived key unchanged."""
    base = _columns(100_003, 5)
    expr, src = "dayofweek(ts)", "ts"
    seg_data = _segment(oracle, base, expr, src, "routes")
    seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
    try:
        q = QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v")], group_by=[expr],
                         filter=Predicate("RANGE", "g", [], 2, None, True, True))
        for knobs in ({}, {"dense_max": 1}, {"smem_groups": 0}):
            with tuned(ctx, **knobs):
                _assert_same(pm.execute_segments([seg], q)[0], pm.execute_segments([seg], _swap(q, expr, "t"))[0], knobs)
        # two spellings, one derived column
        assert seg.column_index("DOW(ts)") == seg.column_index(expr) == len(seg.column_names)
    finally:
        seg.destroy()


def test_merged(oracle, ctx, pm):
    """17 segments in one merged call: source bound to a domain; unbound sources refused until the expression is bound."""
    expr, src = "datetrunc('DAY',ts)", "ts"
    datas = [_segment(oracle, _columns(3_001 + 97 * s, 100 + s), expr, src, f"m{s}") for s in range(17)]
    q = QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v"), Aggregation("DISTINCTCOUNT", "g")],
                     group_by=[expr])
    tq = _swap(q, expr, "t")

    def load():
        return [IndexSegment.from_columns(ctx, d.name, d.num_docs, d.columns) for d in datas]

    segs = load()
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments(segs, q, merge=True)
        dom = DictionaryDomain.build(ctx, segs, [expr, "t"])
        for s in segs:
            s.bind_domain(dom)
        dom.release()
        _assert_same(pm.execute_segments(segs, q, merge=True)[0], pm.execute_segments(segs, tq, merge=True)[0], "expression bound")
    finally:
        for s in segs:
            s.destroy()
    segs = load()
    try:
        dom = DictionaryDomain.build(ctx, segs, [src, "t"])
        for s in segs:
            s.bind_domain(dom)
        dom.release()
        got = pm.execute_segments(segs, q, merge=True)[0]
        _assert_same(got, pm.execute_segments(segs, tq, merge=True)[0], "source bound")
        assert all(s.local_ids(expr).tolist() == s.local_ids("t").tolist() for s in segs)
    finally:
        for s in segs:
            s.destroy()


def test_concurrent_first_queries(oracle, ctx, pm):
    expr, src = "hour(ts)", "ts"
    datas = [_segment(oracle, _columns(20_011, 300 + s), expr, src, f"c{s}") for s in range(3)]
    segs = [IndexSegment.from_columns(ctx, d.name, d.num_docs, d.columns) for d in datas]
    try:
        q = QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v")], group_by=[expr])
        full = lambda b: (_block_bytes(b), [np.asarray(x).tobytes() for x in b.doubles])  # noqa: E731  (SUM of INT: exact)
        want = [full(b) for b in pm.execute_segments(segs, _swap(q, expr, "t"))]
        out, errors = [None] * 12, []

        def run(k):
            try:
                out[k] = [full(b) for b in pm.execute_segments(segs, q)]
            except Exception as e:  # noqa: BLE001
                errors.append(e)
        threads = [threading.Thread(target=run, args=(k,)) for k in range(12)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert all(o == want for o in out)
        for s in segs:   # one derived column each: the next expression takes the next id
            assert s.column_index(expr) == len(s.column_names)
            assert s.derive("minute(ts)") == len(s.column_names) + 1
    finally:
        for s in segs:
            s.destroy()


def test_refusals(oracle, ctx, pm):
    cols = _columns(1_000, 9)
    cols["big"] = np.array([0, (1 << 53) + 1] * 500, dtype=np.int64)
    seg_data = oracle.build_segment("refuse", cols, raw=["r"])
    seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
    with tuned(ctx, raw_dict_max=0):
        raw = IndexSegment.from_columns(ctx, "refuse_raw", seg_data.num_docs, seg_data.columns)
    try:
        for expr, code in [("plus(i,v)", E_UNSUPPORTED), ("year(s)", E_UNSUPPORTED), ("upper(i)", E_UNSUPPORTED),
                           ("datetrunc('DAY',ts,'MILLISECONDS','Europe/Paris')", E_UNSUPPORTED), ("year(big)", E_UNSUPPORTED),
                           ("datetrunc('DAY',big)", E_UNSUPPORTED), ("year(d)", E_UNSUPPORTED), ("plus(i,'1'", E_INVALID),
                           ("plus(nosuch,'1')", E_INVALID), ("timeconvert(ts,'SECONDS')", E_UNSUPPORTED)]:
            with pytest.raises(Pb200Error) as e:
                seg.derive(expr)
            assert e.value.code == code, (expr, e.value)
        e17 = "x"
        for _ in range(17):
            e17 = f"abs({e17})"
        with pytest.raises(UnsupportedQueryError):
            seg.derive(e17.replace("x", "i"))
        with pytest.raises(UnsupportedQueryError):
            raw.derive("abs(r)")
        q = QueryContext(aggregations=[Aggregation("COUNT", None)], group_by=["plus(i,v)"])
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([seg], q)
        for k in range(32):                    # 32 derived columns per segment, not one more
            seg.derive(f"plus(i,'{k}')")
        with pytest.raises(UnsupportedQueryError):
            seg.derive("plus(i,'100')")
        assert seg.derive("plus(i,'3')") == len(seg.column_names) + 3
    finally:
        seg.destroy()
        raw.destroy()


def test_domain_bound_source(oracle, ctx, pm):
    """The identity over a source bound to a domain wider than the segment's own dictionary: the program runs over the
    domain's dictionary, so the derived dictionary is f(domain), exactly the domain dictionary of the stored `t`."""
    for expr, src in [("datetrunc('DAY',ts)", "ts"), ("dayofweek(ts)", "ts"), ("mod(abs(f),'7')", "f"), ("divide(i,'1000')", "i")]:
        datas = [_segment(oracle, _columns(5_003 + 17 * s, 900 + s), expr, src, f"dom{s}") for s in range(2)]
        segs = [IndexSegment.from_columns(ctx, d.name, d.num_docs, d.columns) for d in datas]
        try:
            dom = DictionaryDomain.build(ctx, segs, [src, "t"])
            for s in segs:
                s.bind_domain(dom)
            dom.release()
            for s in segs:
                s.derive(expr)
                for which in ("dict", "fwd"):
                    assert s.read_index(expr, which).tobytes() == s.read_index("t", which).tobytes(), (expr, which)
                assert s.local_ids(expr).tolist() == s.local_ids("t").tolist(), expr
                for q in _queries(expr, ref.column(expr, _columns(5_003, 900)[src], TYPES[src])):
                    _assert_same(pm.execute_segments([s], q)[0], pm.execute_segments([s], _swap(q, expr, "t"))[0], (expr, q))
        finally:
            for s in segs:
                s.destroy()


def test_datatable(oracle, ctx, pm):
    """DataTable bytes: the expression's column is written under its canonical text with its result type."""
    base = _columns(20_011, 41)
    for expr, src, typ in [("datetrunc('HOUR',ts)", "ts", "LONG"), ("dayofweek(ts)", "ts", "INT"), ("divide(i,'1000')", "i", "DOUBLE")]:
        seg_data = _segment(oracle, base, expr, src, "dt")
        seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
        try:
            tables = []
            for key in (expr, "t"):
                q = QueryContext(aggregations=[Aggregation("COUNT", None), Aggregation("SUM", "v"), Aggregation("MAX", "v")],
                                 group_by=[key], num_groups_limit=1_000_000)
                block = pm.execute_segments([seg], q, keep_handle=True, defer=False)[0]
                try:
                    tables.append(datatable_util.parse(pm.to_datatable(seg, q, block)))
                finally:
                    block.release(ctx)
            e, t = tables
            assert e["column_names"] == [expr, "count(*)", "sum(v)", "max(v)"]
            assert e["column_types"] == t["column_types"] == [typ, "LONG", "DOUBLE", "DOUBLE"]
            assert sorted(map(tuple, e["rows"])) == sorted(map(tuple, t["rows"]))
            for k in ("numDocsScanned", "totalDocs", "numGroupsLimitReached"):
                assert e["metadata"][k] == t["metadata"][k], k
        finally:
            seg.destroy()


def test_star_tree_segment_scans(oracle, ctx, pm):
    """An expression is no star-tree dimension: a star-tree segment answers it by the raw scan, with the identity."""
    rng = np.random.default_rng(8)
    n = 30_000
    cols = {"d1": rng.integers(0, 50, size=n).astype(np.int32), "d2": rng.integers(0, 7, size=n).astype(np.int32),
            "m": rng.integers(0, 1000, size=n).astype(np.int32)}
    expr = "mod(d1,'7')"
    cols["t"] = ref.column(expr, cols["d1"], "INT")
    seg_data = oracle.build_segment("stx", cols)
    st = stb.build_star_tree(seg_data, ["d1", "d2"], [("COUNT", None), ("SUM", "m")], max_leaf_records=10)
    seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
    try:
        nd = len(st.dimensions)
        seg.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                             [(fn, c, st.segment.columns[nd + i].fwd) for i, (fn, c) in enumerate(st.function_pairs)])
        for q in (sql.parse(f"SELECT {expr}, COUNT(*), SUM(m) FROM t GROUP BY {expr}"),
                  sql.parse(f"SELECT d2, COUNT(*), SUM(m) FROM t WHERE {expr} > 2 GROUP BY d2")):
            got = pm.execute_segments([seg], q)[0]
            assert got.operator_kind == "GROUP_BY", got.operator_kind
            _assert_same(got, pm.execute_segments([seg], _swap(q, expr, "t"))[0], q)
        assert pm.execute_segments([seg], sql.parse("SELECT d2, COUNT(*), SUM(m) FROM t GROUP BY d2"))[0].operator_kind == "STAR_TREE"
    finally:
        seg.destroy()


def test_destroy_frees_derived_memory(oracle, ctx, pm):
    """Destroying a segment gives its derived columns back: load, derive and destroy cycles do not grow the device's use."""
    seg_data = _segment(oracle, _columns(200_003, 12), "datetrunc('MINUTE',ts)", "ts", "free")

    def cycle():
        seg = IndexSegment.from_columns(ctx, seg_data.name, seg_data.num_docs, seg_data.columns)
        for e in ("datetrunc('MINUTE',ts)", "dayofweek(ts)", "divide(i,'7')"):
            seg.derive(e)
        derived = seg.device_bytes()
        seg.destroy()
        return derived, ctx.device_info()["free_mem_mb"]

    cycle()
    first = cycle()
    for _ in range(3):
        assert cycle() == first   # every block of a cycle came back to the pool and was reused by the next one

"""REGEXP_LIKE and LIKE on STRING dictionary columns on the device (DESIGN.md section 3.12).

Every pattern result is held to two independent answers: the doc set tests/pattern_ref.py builds from the column's
values, and the same query with each pattern leaf replaced by an IN over the values pattern_ref matches (answered by the
oracle on one segment, and by the already-verified IN path for merged, selection and DISTINCT calls).  Columns: plain,
inverted, sorted and domain-bound, with dictionaries of 1 to 100 000 entries."""
import dataclasses
import threading

import numpy as np
import pytest

import pattern_ref as R
from gpu_util import assert_tables_equal, gpu_table, oracle_table, to_device
from pinot_b200 import _lib, sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Filter, Predicate

pytestmark = pytest.mark.gpu

EDGE = ["", "a", "\n", "a\n", "a\r\n", "x ", "é", "日本", "😀x", "/api/v1/users", "HTTP/1.1", "a.b"]


def _urls(rng, n):
    paths = ["api", "v1", "v2", "users", "orders", "img", "static", "login", "search", "é", "日本"]
    out = []
    for _ in range(n):
        depth = rng.integers(1, 5)
        out.append("/" + "/".join(paths[rng.integers(0, len(paths))] for _ in range(depth)) + f"/{rng.integers(0, 10**6)}")
    return out


def _column(values, rng, n):
    ids = rng.integers(0, len(values), size=n)
    return np.array([v.encode() for v in values], dtype=object)[ids].astype("S")


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
    rng = np.random.default_rng(11)
    n = 20_000
    url_values = _urls(rng, 3000) + EDGE
    cols = {
        "u": _column(url_values, rng, n),                                        # plain STRING dictionary
        "h": _column([f"host{i}.example.com" for i in range(40)] + ["é.fr"], rng, n),  # inverted
        "s": np.sort(_column([f"s{i:03d}" for i in range(200)], rng, n)),        # sorted
        "k": rng.integers(0, 13, size=n).astype(np.int32),
        "m": rng.integers(-1000, 1000, size=n).astype(np.int32),
    }
    cols["u"][:3] = [b"a\xffb", b"\xe2\x82a", b"a\n"]   # invalid UTF-8 in the dictionary
    seg = oracle.build_segment("p0", cols, inverted=["h"])
    dev = to_device(ctx, seg)
    yield seg, dev, cols
    dev.destroy()


def _values(seg, col):
    return [bytes(v) for v in seg.column(col).dict_values]


def _to_in(node, segs):
    """The filter with every REGEXP_LIKE leaf replaced by an IN over the dictionary values pattern_ref matches."""
    if node is None:
        return None
    if isinstance(node, Filter):
        return Filter(node.type, [_to_in(c, segs) for c in node.children])
    if node.type != "REGEXP_LIKE":
        return node
    vals = sorted({v for s in segs for v in _values(s, node.column) if R.matches(node.values[0], v)})
    if not vals:
        return Predicate("EQ", node.column, [b"\x01no such value"])
    return Predicate("IN", node.column, vals)


def _in_query(q, segs):
    return dataclasses.replace(q, filter=_to_in(q.filter, segs),
                               aggregations=[dataclasses.replace(a, filter=_to_in(a.filter, segs)) for a in q.aggregations])


def _docs(cols, node):
    """The docs of a filter tree, from the column values (pattern leaves through pattern_ref)."""
    if isinstance(node, Filter):
        kids = [_docs(cols, c) for c in node.children]
        if node.type == "NOT":
            return ~kids[0]
        return np.logical_and.reduce(kids) if node.type == "AND" else np.logical_or.reduce(kids)
    vals = cols[node.column]
    if node.type == "REGEXP_LIKE":
        uniq, inv = np.unique(vals, return_inverse=True)
        return np.array([R.matches(node.values[0], bytes(v)) for v in uniq])[inv]
    assert node.type == "EQ"
    return vals == node.values[0]


PATTERNS = ["api", "^/api/", "users/\\d+$", "^/(?:v1|v2)/", "[0-9]{6}$", "é", "日本", "\\.", "^$", "", "^a",
            "zzz-no-match", ".", "\\n$", "[^a-z/0-9]", "^/[a-z]+/[a-z]+/\\d{1,3}$", "a.b"]


@pytest.mark.parametrize("pattern", PATTERNS)
def test_count_and_sum_match_the_doc_set(oracle, pm, data, pattern):
    seg, dev, cols = data
    for col in ("u", "h", "s"):
        q = sql.parse(f"SELECT COUNT(*), SUM(m) FROM t WHERE REGEXP_LIKE({col}, '{pattern}')")
        docs = _docs(cols, q.filter)
        block = pm.make_segment_plan_node(dev, q).run().next_block()
        assert int(block.longs[0][0]) == int(docs.sum()), (col, pattern)
        assert int(block.doubles[1][0]) == int(cols["m"][docs].sum()), (col, pattern)
        want = oracle.execute(seg, _in_query(q, [seg]))
        assert_tables_equal(q, gpu_table(seg, q, block, dev), oracle_table(seg, q, want), f"{col} {pattern}")
        assert block.stats.num_docs_scanned == want.stats[0]


QUERIES = [
    "SELECT k, COUNT(*), SUM(m), MIN(m), MAX(m) FROM t WHERE u LIKE '%/users/%' GROUP BY k",
    "SELECT k, COUNT(*) FROM t WHERE u NOT LIKE '/api%' AND REGEXP_LIKE(h, '^host1') GROUP BY k",
    "SELECT k, SUM(m) FROM t WHERE REGEXP_LIKE(u, 'v1') OR s LIKE 's01_' GROUP BY k ORDER BY SUM(m) DESC LIMIT 3",
    "SELECT k, COUNT(*) FROM t WHERE NOT (REGEXP_LIKE(u, 'é') OR REGEXP_LIKE(h, '\\.fr$')) GROUP BY k HAVING COUNT(*) > 1400",
    "SELECT h, COUNT(*), DISTINCTCOUNT(u) FROM t WHERE REGEXP_LIKE(u, '^/(?:img|static)/') GROUP BY h",
    "SELECT k, COUNT(*) FILTER (WHERE u LIKE '%login%'), SUM(m) FILTER (WHERE REGEXP_LIKE(h, '[13]\\.')), COUNT(*) FROM t GROUP BY k",
    "SELECT COUNT(*) FILTER (WHERE REGEXP_LIKE(s, '9$')), SUM(m) FROM t WHERE k < 7",
    "SELECT s, MAX(m) FROM t WHERE REGEXP_LIKE(s, '^s1') AND REGEXP_LIKE(s, '5') GROUP BY s",
]


@pytest.mark.parametrize("text", QUERIES)
def test_queries_match_the_in_equivalent(oracle, pm, data, text):
    seg, dev, _cols = data
    q = sql.parse(text)
    block = pm.execute_segments([dev], q)[0]
    q_in = _in_query(q, [seg])
    want = oracle.execute(seg, q_in) if q.having is None and not q.order_by else None
    got = gpu_table(seg, q, block, dev)
    ref = pm.execute_segments([dev], q_in)[0]
    assert_tables_equal(q, got, gpu_table(seg, q_in, ref, dev), text)
    if want is not None:
        assert_tables_equal(q, got, oracle_table(seg, q, want), text)


def test_explain_and_folding(pm, data):
    seg, dev, _cols = data
    ex = lambda t: pm.explain(dev, sql.parse(t))
    assert ex("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 'api')") == "AGGREGATE(FILTER_FULL_SCAN(REGEXP_LIKE,u))"
    assert ex("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(h, '^host1')") == "AGGREGATE(FILTER_INVERTED_INDEX(REGEXP_LIKE,h))"
    assert ex("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(s, '^s1')") == "AGGREGATE(FILTER_SORTED_INDEX(REGEXP_LIKE,s))"
    assert ex("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 'zzz')") == "EMPTY(FILTER_EMPTY)"
    assert ex("SELECT COUNT(*) FROM t WHERE u LIKE '%'") == "AGGREGATE_NO_SCAN(FILTER_MATCH_ENTIRE_SEGMENT)"
    assert ex("SELECT COUNT(*) FROM t WHERE NOT REGEXP_LIKE(h, 'example|é')") == "EMPTY(FILTER_EMPTY)"
    q = sql.parse("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 'zzz')")
    assert pm.execute_segments([dev], q)[0].operator_kind == "EMPTY"
    q = sql.parse("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(s, '^s')")
    b = pm.execute_segments([dev], q)[0]
    assert b.operator_kind == "NON_SCAN_AGGREGATION" and int(b.longs[0][0]) == seg.num_docs


def test_datatable_bytes_match_the_in_equivalent(pm, data):
    seg, dev, _cols = data
    q = sql.parse("SELECT h, COUNT(*), SUM(m) FROM t WHERE REGEXP_LIKE(u, 'users') GROUP BY h")
    q_in = _in_query(q, [seg])
    a = pm.execute_segments([dev], q, keep_handle=True)[0]
    b = pm.execute_segments([dev], q_in, keep_handle=True)[0]
    assert pm.to_datatable(dev, q, a) == pm.to_datatable(dev, q_in, b)


def test_selection_and_distinct(pm, data):
    seg, dev, cols = data
    s = sql.parse_selection("SELECT u, m FROM t WHERE u LIKE '/login%' AND k = 3 LIMIT 100000")
    got = pm.execute_selection([dev], s)[0]
    docs = np.nonzero(_docs(cols, s.filter.children[0]) & (cols["k"] == 3))[0]
    assert sorted(got.doc_ids.tolist()) == docs.tolist()
    d = sql.parse_distinct("SELECT DISTINCT h FROM t WHERE REGEXP_LIKE(u, '日本') ORDER BY h LIMIT 1000")
    want = sorted({cols["h"][i].decode() for i in np.nonzero(_docs(cols, d.filter))[0]})
    got = pm.execute_distinct([dev], d)[0]
    assert [str(v) for v in got.columns[0]] == want
    d_in = dataclasses.replace(d, filter=_to_in(d.filter, [seg]))
    assert list(pm.execute_distinct([dev], d_in)[0].columns[0]) == list(got.columns[0])


def test_merged_domain_bound_segments(oracle, ctx, pm):
    """Segments with different dictionaries, bound to one domain: ids are resolved against each segment's own
    dictionary and translated; the merged result equals the IN equivalent and the doc-set count."""
    rng = np.random.default_rng(5)
    segs, devs, all_cols = [], [], []
    for i, n in enumerate([3000, 1, 4500, 777]):
        cols = {"u": _column(_urls(rng, 50 + 400 * i) + EDGE[: 3 + i], rng, n),
                "k": rng.integers(0, 5, size=n).astype(np.int32), "m": rng.integers(0, 100, size=n).astype(np.int32)}
        seg = oracle.build_segment(f"pm{i}", cols)
        segs.append(seg); all_cols.append(cols); devs.append(to_device(ctx, seg))
    dom = DictionaryDomain.build(ctx, devs, ["u", "k"])
    try:
        for d in devs:
            d.bind_domain(dom)
        for text in ("SELECT u, COUNT(*) FROM t WHERE REGEXP_LIKE(u, '^/api/') GROUP BY u",
                     "SELECT k, COUNT(*), SUM(m) FROM t WHERE u NOT LIKE '%users%' GROUP BY k",
                     "SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, '\\n$')"):
            q = sql.parse(text)
            got = pm.execute_segments(devs, q, merge=True)[0]
            q_in = _in_query(q, segs)
            ref = pm.execute_segments(devs, q_in, merge=True)[0]
            assert _rows(got) == _rows(ref), text   # both in the domain's id space
            assert got.stats.num_docs_scanned == sum(int(_docs(c, q.filter).sum()) for c in all_cols), text
            per = pm.execute_segments(devs, q)
            assert [b.stats.num_docs_scanned for b in per] == [int(_docs(c, q.filter).sum()) for c in all_cols]
    finally:
        for d in devs:
            d.destroy()
        dom.release()


def _rows(block):
    n = max(block.num_groups, 1)
    return sorted((tuple(block.keys[g].tolist()) if block.num_groups >= 0 else (),
                   tuple(float(d[g]) for d in block.doubles), tuple(int(v[g]) for v in block.longs)) for g in range(n))


@pytest.mark.parametrize("card", [1, 2, 31, 32, 33, 1000, 100_000])
def test_dictionary_sizes(oracle, ctx, pm, card):
    rng = np.random.default_rng(card)
    n = max(card, 5000)
    values = [f"v{i}/{'é' if i % 7 == 0 else 'x'}{i % 97}" for i in range(card)]
    ids = np.concatenate([np.arange(card), rng.integers(0, card, size=n - card)])
    cols = {"u": np.array([v.encode() for v in values], dtype=object)[ids].astype("S"), "m": rng.integers(0, 9, size=n).astype(np.int32)}
    seg = oracle.build_segment(f"card{card}", cols)
    dev = to_device(ctx, seg)
    try:
        for pattern in ("é", "3$", "^v1", "/x[0-9]{2}$"):
            q = sql.parse(f"SELECT COUNT(*), SUM(m) FROM t WHERE REGEXP_LIKE(u, '{pattern}')")
            b = pm.execute_segments([dev], q)[0]
            docs = _docs(cols, q.filter)
            assert int(b.longs[0][0]) == int(docs.sum()) and int(b.doubles[1][0]) == int(cols["m"][docs].sum()), (card, pattern)
    finally:
        dev.destroy()


def test_star_tree_equals_the_raw_scan(oracle, ctx, pm):
    rng = np.random.default_rng(3)
    n = 30_000
    cols = {"h": _column([f"host{i}.example.com" for i in range(30)], rng, n), "k": rng.integers(0, 6, size=n).astype(np.int32),
            "m": rng.integers(0, 1000, size=n).astype(np.int32)}
    seg = oracle.build_segment("st", cols)
    dev = to_device(ctx, seg)
    try:
        dev.build_star_tree(["h", "k"], [("COUNT", None), ("SUM", "m")])
        for text in ("SELECT k, COUNT(*), SUM(m) FROM t WHERE REGEXP_LIKE(h, '^host1') GROUP BY k",
                     "SELECT COUNT(*), SUM(m) FROM t WHERE h LIKE '%2.example%' AND k = 3",
                     "SELECT h, SUM(m) FROM t WHERE REGEXP_LIKE(h, 'zz') GROUP BY h"):
            q = sql.parse(text)
            star = pm.execute_segments([dev], q)[0]
            raw_q = dataclasses.replace(q, use_star_tree=False)
            raw = pm.execute_segments([dev], raw_q)[0]
            assert star.operator_kind in ("STAR_TREE", "EMPTY"), text
            assert_tables_equal(q, gpu_table(seg, q, star, dev), gpu_table(seg, q, raw, dev), text)
            want = oracle.execute(seg, _in_query(q, [seg]))
            assert_tables_equal(q, gpu_table(seg, q, raw, dev), oracle_table(seg, q, want), text)
    finally:
        dev.destroy()


@pytest.mark.parametrize("text,code", [
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(k, '1')", "unsupported"),            # INT column
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(k + 1, '1')", "unsupported"),        # derived column
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(r, '1')", "unsupported"),            # no dictionary
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, '\\bapi')", "unsupported"),       # outside the subset
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, '(a)\\1')", "unsupported"),
    ("SELECT COUNT(*) FILTER (WHERE REGEXP_LIKE(u, 'a{99}')) FROM t", "unsupported"),
    ("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, '\udcff')", "invalid"),           # not UTF-8
])
def test_refusals(oracle, ctx, pm, text, code):
    rng = np.random.default_rng(1)
    cols = {"u": _column(["/a", "/b"], rng, 100), "k": rng.integers(0, 3, size=100).astype(np.int32),
            "r": rng.integers(0, 10**9, size=100).astype(np.int32)}
    seg = oracle.build_segment("ref", cols, raw=["r"])
    ctx.set_tuning("raw_dict_max", 0)   # r stays a raw column without a dictionary
    try:
        dev = to_device(ctx, seg)
    finally:
        ctx.set_tuning("raw_dict_max", 1 << 20)
    try:
        q = sql.parse(text.replace("\udcff", "X"))
        if code == "invalid":
            q.filter.values[0] = b"a\xff"
        with pytest.raises(_lib.Pb200Error) as e:
            pm.execute_segments([dev], q)
        assert isinstance(e.value, _lib.UnsupportedQueryError) == (code == "unsupported"), e.value
    finally:
        dev.destroy()


def test_concurrent_first_queries_upload_once(oracle, ctx, pm):
    rng = np.random.default_rng(9)
    n = 50_000
    cols = {"u": _column(_urls(rng, 20_000), rng, n), "m": rng.integers(0, 9, size=n).astype(np.int32)}
    seg = oracle.build_segment("cc", cols)
    a, b = to_device(ctx, seg), to_device(ctx, seg)
    try:
        before = a.device_bytes()
        q = sql.parse("SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(u, 'users/\\d+$')")
        want = int(_docs(cols, q.filter).sum())
        pm.execute_segments([b], q)
        one_upload = b.device_bytes() - before
        assert one_upload > 0
        results, errors = [], []

        def run():
            try:
                results.append(int(B200PlanMaker(ctx).execute_segments([a], q)[0].longs[0][0]))
            except Exception as e:  # noqa: BLE001
                errors.append(e)
        threads = [threading.Thread(target=run) for _ in range(12)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors and results == [want] * 12
        assert a.device_bytes() - before == one_upload   # built once
    finally:
        a.destroy()
        b.destroy()

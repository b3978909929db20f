"""-m gpu: predicates on expressions over two or more columns (DESIGN.md section 3.16) against the value-space reference
tests/expr_filter_ref.py (tests/filter_ref.py for ordinary leaves, expr_ref.evaluate + float_edges_ref.raw_matches for
expression leaves).

Segments of 1 .. 100 003 rows hold INT leaves at the INT ends, LONG leaves at the int64 ends and 2^53 + 1, FLOAT and DOUBLE
leaves with NaN, -0.0 and +-inf, raw INT / DOUBLE leaves (dictionaries synthesised at load, or the raw INT / FLOAT
streamed as 32-bit values with raw_dict_max=0), a sorted and an inverted column and group-by keys.  Doc sets are checked
exactly through selection (doc ids) for every predicate type, alone and under AND / OR / NOT next to scan, sorted and
inverted leaves, with two expression leaves in one tree; aggregation-only and group-by on the shared-memory, dense and hash
tables with the count carrier on and off; the same expression in WHERE and in SUM; ORDER BY ... LIMIT, HAVING, a FILTER
clause, DISTINCT, 17 merged segments with per-segment operand dictionaries and bound group keys, DataTable bytes, the
CLI, a loopback 2-rank combine, a star-tree segment, the statistics and the refusals."""
import json

import numpy as np
import pytest

from exact_ref import column_values
from expr_filter_ref import expression_values, matching_docs
from expr_ref import check_value
from gpu_util import to_device, tuned
from pinot_b200 import cli, sql
from pinot_b200._lib import E_INVALID, E_UNSUPPORTED, Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Filter, QueryContext
from pinot_b200.sql import SelectionQuery

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 33, 4096, 8193, 100_003]


def _segment(oracle, n, seed, name=None, edges=True, raw_double=True):
    rng = np.random.default_rng(seed)
    i = (rng.integers(-300, 300, size=n) * 7).astype(np.int32)
    j = rng.integers(-5, 6, size=n).astype(np.int32)
    lv = rng.integers(-10_000, 10_000, size=n).astype(np.int64)
    f = (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32)
    d = rng.integers(-600, 600, size=n) / 3.0
    if edges:
        i[rng.integers(0, n, size=max(1, n // 60))] = INT_MAX
        i[rng.integers(0, n, size=max(1, n // 60))] = INT_MIN
        longs = np.array([INT64_MIN, INT64_MAX, (1 << 53) + 1, -(1 << 53) - 1, 0], dtype=np.int64)
        lv[rng.integers(0, n, size=max(1, n // 40))] = longs[rng.integers(0, len(longs), size=max(1, n // 40))]
        f[rng.integers(0, n, size=max(1, n // 50))] = -0.0
        d[rng.integers(0, n, size=max(1, n // 50))] = -0.0
        d[rng.integers(0, n, size=max(1, n // 70))] = np.nan
        f[rng.integers(0, n, size=max(1, n // 90))] = np.inf
        d[rng.integers(0, n, size=max(1, n // 90))] = -np.inf
    cols = {"rid": np.arange(n, dtype=np.int32), "i": i, "j": j, "l": lv, "f": f, "d": d,
            "ri": rng.integers(-1_000, 1_000, size=n).astype(np.int32),
            "rd": rng.integers(-50, 50, size=n) / 4.0 if raw_double else rng.integers(-50, 50, size=n).astype(np.int32),
            "rf": (rng.integers(-50, 50, size=n) / 4.0).astype(np.float32),
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 3000, size=n).astype(np.int32),
            "srt": np.sort(rng.integers(0, 12, size=n)).astype(np.int32),
            "inv": rng.integers(0, 20, size=n).astype(np.int32),
            "s": np.array([b"a", b"bb", b"c"])[rng.integers(0, 3, size=n)]}
    return oracle.build_segment(name or f"ef{n}_{seed}", cols, raw=["ri", "rd", "rf"], inverted=["inv"])


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def segs(oracle, ctx):
    out = [(s, to_device(ctx, s)) for s in (_segment(oracle, n, n) for n in SIZES)]
    yield out
    for _, dev in out:
        dev.destroy()


# every predicate type on every leaf kind, and trees mixing them with scan, sorted and inverted leaves
WHERE = ["i > j", "l - i <= 100", "f * d >= 0", "d / f < 1", "i * j = 0", "ri - rd <> 0", "i + j IN (0, 7, 14, 14)",
         "mod(l, j) NOT IN (0, 1)", "d - f BETWEEN -3 AND 3", "5 < ri + j", "l * j > 9007199254740993", "d + f = -0.0",
         "abs(d - i) IN (0, 1.0e400)", "floor(d / j) <> 2",
         "i > j AND srt = 3", "i > j OR inv IN (1, 2)", "NOT (f * d >= 0)", "i > j AND d - f BETWEEN -3 AND 3",
         "rid > 10 AND (i * j = 0 OR g = 2)", "NOT (i > j) OR (inv = 4 AND ri - rd <> 0)", "srt IN (2, 5) AND NOT i + j IN (0, 7)"]


def _where(text):
    return sql.parse(f"SELECT COUNT(*) FROM t WHERE {text}").filter


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _doc_set(pm, dev, flt, n):
    got = pm.execute_selection([dev], SelectionQuery(columns=["rid"], filter=flt, limit=max(n, 1)))[0]
    return np.sort(np.asarray(got.doc_ids, dtype=np.int64)), got


def test_doc_sets(oracle, pm, segs):
    """Exact doc ids of every tree on every size, through selection."""
    for seg, dev in segs:
        for text in WHERE:
            flt = _where(text)
            want = np.nonzero(matching_docs(oracle, seg, flt))[0]
            got, _ = _doc_set(pm, dev, flt, seg.num_docs)
            assert np.array_equal(got, want), (seg.num_docs, text, len(got), len(want))


def test_streamed_raw_leaves(oracle, ctx, pm):
    """Raw INT and FLOAT leaves streamed as 32-bit values (raw_dict_max=0)."""
    with tuned(ctx, raw_dict_max=0):
        for n in (4096, 100_003):
            seg = _segment(oracle, n, 31 + n, raw_double=False)   # a raw DOUBLE only loads with a synthesised dictionary
            dev = to_device(ctx, seg)
            try:
                for text in ("ri > rf", "ri * rf <= 12.5", "rf - i IN (0, 3.25)", "NOT (ri + rf BETWEEN -10 AND 10) AND g = 3",
                             "ri / rf <> 1"):
                    flt = _where(text)
                    want = np.nonzero(matching_docs(oracle, seg, flt))[0]
                    assert np.array_equal(_doc_set(pm, dev, flt, n)[0], want), (n, text)
                    b = pm.execute_segments([dev], _query([Aggregation("COUNT")], flt))[0]
                    assert int(b.longs[0][0]) == len(want), (n, text)
            finally:
                dev.destroy()


def _query(aggs, flt=None, group_by=(), **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), limit=kw.pop("limit", 100_000), **kw)


def _ref_groups(oracle, data, flt, group_by):
    """{key: (COUNT(*), SUM(i))} over the matched docs of the segments `data`."""
    out = {} if group_by else {(): (0, 0)}
    for seg in data:
        docs = np.nonzero(matching_docs(oracle, seg, flt))[0]
        if not len(docs):
            continue
        keys = [column_values(oracle, seg, g, docs) for g in group_by]
        iv = column_values(oracle, seg, "i", docs)
        for k in range(len(docs)):
            key = tuple(_py(x[k]) for x in keys)
            c, s = out.get(key, (0, 0))
            out[key] = (c + 1, s + int(iv[k]))
    return out


def _check_groups(oracle, data, dev, q, b, what):
    ref = _ref_groups(oracle, data, q.filter, q.group_by)
    if not q.group_by:
        assert (int(b.longs[0][0]), float(b.doubles[1][0])) == (ref[()][0], float(ref[()][1])), what
        return
    got = {}
    for r in range(b.num_groups):
        key = tuple(_py(dev.dictionary_value(c, int(b.keys[r, k]))) for k, c in enumerate(q.group_by))
        got[key] = (int(b.longs[0][r]), int(round(float(b.doubles[1][r]))))
    assert got == ref, what


@pytest.mark.parametrize("knobs", [dict(), dict(dense_max=1), dict(pack_count=0), dict(pack_count=1)],
                         ids=["default", "hash", "carrier_off", "carrier_on"])
def test_aggregations_and_group_by(oracle, ctx, pm, segs, knobs):
    """COUNT(*) and SUM(i) under expression filters: aggregation only, and group-by on the shared-memory (g), dense (h)
    and hash (dense_max=1) tables, with the count carrier on and off."""
    with tuned(ctx, **knobs):
        for seg, dev in segs[2:]:
            for text in ("i > j", "i > j AND d - f BETWEEN -3 AND 3", "NOT (f * d >= 0) OR inv IN (1, 2)", "mod(l, j) NOT IN (0, 1)"):
                for gb in ([], ["g"], ["h"], ["g", "h"]):
                    q = _query([Aggregation("COUNT"), Aggregation("SUM", "i")], _where(text), group_by=gb)
                    _check_groups(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"{knobs} n={seg.num_docs} {text} {gb}")


def test_same_expression_in_where_and_sum(oracle, pm, segs):
    seg, dev = segs[5]
    for text in ("SELECT SUM(i * j), MAX(i * j), COUNT(*) FROM t WHERE i * j > 0",
                 "SELECT g, SUM(d - f), MIN(d - f), COUNT(*) FROM t WHERE d - f BETWEEN -3 AND 3 GROUP BY g"):
        q = sql.parse(text)
        b = pm.execute_segments([dev], q, merge=True)[0]
        docs = np.nonzero(matching_docs(oracle, seg, q.filter))[0]
        xs = expression_values(oracle, seg, q.filter.column)
        keys = column_values(oracle, seg, "g", docs) if q.group_by else None
        groups = {}
        for n, doc in enumerate(docs):
            groups.setdefault((_py(keys[n]),) if q.group_by else (), []).append(xs[doc])
        rows = 1 if b.num_groups < 0 else b.num_groups
        assert rows == len(groups)
        for r in range(rows):
            key = (_py(dev.dictionary_value("g", int(b.keys[r, 0]))),) if q.group_by else ()
            vals = groups[key]
            assert check_value("SUM", float(b.doubles[0][r]), 0, vals), (text, key)
            assert check_value(q.aggregations[1].function, float(b.doubles[1][r]), 0, vals), (text, key)
            assert int(b.longs[2][r]) == len(vals)


def test_order_by_having_filter_clause_distinct(oracle, pm, segs):
    seg, dev = segs[5]
    flt = _where("i > j")
    ref = _ref_groups(oracle, [seg], flt, ["h"])
    q = sql.parse("SELECT h, COUNT(*), SUM(i) FROM t WHERE i > j GROUP BY h ORDER BY COUNT(*) DESC, h LIMIT 5")
    b = pm.execute_segments([dev], q, merge=True)[0]
    want = sorted(ref.items(), key=lambda kv: (-kv[1][0], kv[0][0]))[:5]
    got = [((_py(dev.dictionary_value("h", int(b.keys[r, 0]))),), (int(b.longs[0][r]), int(round(float(b.doubles[1][r]))))) for r in range(5)]
    assert got == want
    q = sql.parse("SELECT h, COUNT(*), SUM(i) FROM t WHERE i > j GROUP BY h HAVING COUNT(*) > 20")
    b = pm.execute_segments([dev], q, merge=True)[0]
    assert b.num_groups == sum(1 for c, _ in ref.values() if c > 20)
    # a FILTER clause on an expression, next to one on a column, over an expression WHERE
    q = sql.parse("SELECT g, COUNT(*) FILTER (WHERE i * j > 0), SUM(i) FILTER (WHERE f * d >= 0), COUNT(*) FROM t WHERE l - i <= 100 GROUP BY g")
    b = pm.execute_segments([dev], q)[0]
    main = q.filter
    for k, sub in ((0, _where("i * j > 0")), (1, _where("f * d >= 0"))):
        r_sub = _ref_groups(oracle, [seg], Filter("AND", [main, sub]), ["g"])
        for r in range(b.num_groups):
            key = (_py(dev.dictionary_value("g", int(b.keys[r, 0]))),)
            c, s = r_sub.get(key, (0, 0))
            assert (int(b.longs[0][r]) if k == 0 else int(round(float(b.doubles[1][r])))) == (c if k == 0 else s), (k, key)
    r_main = _ref_groups(oracle, [seg], main, ["g"])
    assert b.num_groups == len(r_main)
    # DISTINCT
    q = sql.parse_distinct("SELECT DISTINCT g, srt FROM t WHERE i + j IN (0, 7, 14) LIMIT 1000")
    got = pm.execute_distinct([dev], q)[0]
    docs = np.nonzero(matching_docs(oracle, seg, q.filter))[0]
    want = {(int(a), int(c)) for a, c in zip(column_values(oracle, seg, "g", docs), column_values(oracle, seg, "srt", docs))}
    assert {(int(a), int(c)) for a, c in zip(got.columns[0], got.columns[1])} == want


def test_seventeen_segments_merged_and_bound(oracle, ctx, pm):
    """Merged on the device: the group-by keys bound to a domain, the leaf columns each with their own dictionary (and
    bound too: a bound leaf reads the domain's dictionary)."""
    data = [_segment(oracle, 3000 + 37 * k, 300 + k, name=f"ef17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = DictionaryDomain.build(ctx, devs, ["g", "h", "j"])
    try:
        for d in devs:
            d.bind_domain(domain)
        for text in ("i > j", "d / f < 1 AND inv IN (1, 2)", "NOT l - j IN (0, 7)"):
            for gb in ([], ["g"], ["g", "h"]):
                q = _query([Aggregation("COUNT"), Aggregation("SUM", "i")], _where(text), group_by=gb)
                _check_groups(oracle, data, devs[0], q, pm.execute_segments(devs, q, merge=True)[0], f"merged {text} {gb}")
                blocks = pm.execute_segments(devs, q)
                for seg, dev, b in zip(data, devs, blocks):
                    _check_groups(oracle, [seg], dev, q, b, f"per segment {text} {gb}")
            got = pm.execute_selection(devs, SelectionQuery(columns=["rid"], filter=_where(text), limit=1_000_000), merge=True)
            want = sum(int(np.count_nonzero(matching_docs(oracle, s, _where(text)))) for s in data)
            assert got.num_rows == want
    finally:
        for d in devs:
            d.destroy()
        domain.release()


def test_statistics(oracle, pm, segs):
    """Each expression leaf adds num_docs x its distinct leaf columns to num_entries_scanned_in_filter."""
    seg, dev = segs[4]
    n = seg.num_docs
    base = _query([Aggregation("COUNT")], _where("g = 3"))
    b0 = pm.execute_segments([dev], base)[0]
    for text, extra in (("g = 3 AND i > j", 2 * n), ("g = 3 AND i + i * j > 0 AND d - f < 0", 2 * n + 2 * n),
                        ("g = 3 OR l * j * l > 0", 2 * n)):
        q = _query([Aggregation("COUNT")], _where(text))
        b = pm.execute_segments([dev], q)[0]
        matched = int(np.count_nonzero(matching_docs(oracle, seg, q.filter)))
        assert b.stats.num_docs_scanned == matched == int(b.longs[0][0])
        assert b.stats.num_entries_scanned_in_filter == b0.stats.num_entries_scanned_in_filter + extra, text
        sel = pm.execute_selection([dev], SelectionQuery(columns=["rid"], filter=q.filter, limit=n))[0]
        assert sel.stats.num_entries_scanned_in_filter >= extra


def test_star_tree_segment_declines(oracle, ctx, pm):
    """A segment with a star-tree over the columns: the expression leaf is no star-tree dimension, so the raw scan runs."""
    seg = _segment(oracle, 8193, 77, name="efst")
    dev = to_device(ctx, seg)
    try:
        dev.build_star_tree(["g", "inv"], [("COUNT", None), ("SUM", "i")])
        plain = sql.parse("SELECT g, COUNT(*), SUM(i) FROM t WHERE inv = 3 GROUP BY g")
        assert pm.execute_segments([dev], plain)[0].operator_kind == "STAR_TREE"   # the same query without the leaf
        for text in ("SELECT g, COUNT(*), SUM(i) FROM t WHERE i > j GROUP BY g",
                     "SELECT g, COUNT(*), SUM(i) FROM t WHERE inv = 3 AND i > j GROUP BY g",
                     "SELECT COUNT(*), SUM(i) FROM t WHERE g - inv > 0"):
            q = sql.parse(text)
            b = pm.execute_segments([dev], q)[0]
            assert b.operator_kind != "STAR_TREE", text
            _check_groups(oracle, [seg], dev, q, b, text)
    finally:
        dev.destroy()


def test_datatable_and_cli(oracle, ctx, pm, segs, tmp_path, capsys):
    from datatable_util import parse as parse_datatable
    from segment_dir_util import write_segment_dir
    seg, dev = segs[3]
    q = sql.parse("SELECT g, COUNT(*), SUM(i) FROM t WHERE l - i <= 100 GROUP BY g")
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        dt = parse_datatable(pm.to_datatable(dev, q, b))
    finally:
        b.release(ctx)
    ref = _ref_groups(oracle, [seg], q.filter, ["g"])
    assert {(row[0],): (int(row[1]), int(round(float(row[2])))) for row in dt["rows"]} == ref
    # the CLI: bytes_out > bytes_in, per segment and merged on the device
    data = []
    for k in range(2):
        rng = np.random.default_rng(40 + k)
        n = 3000 + 11 * k
        data.append(oracle.build_segment(f"efcli{k}", {"k": rng.integers(0, 25, size=n).astype(np.int32),
                                                         "bytes_out": rng.integers(0, 5000, size=n).astype(np.int64),
                                                         "bytes_in": rng.integers(0, 5000, size=n).astype(np.int32)}))
    dirs = [str(write_segment_dir(tmp_path / f"s{k}", s)) for k, s in enumerate(data)]
    flt = _where("bytes_out > bytes_in")
    want = {}
    for s in data:
        docs = np.nonzero(matching_docs(oracle, s, flt))[0]
        for key in column_values(oracle, s, "k", docs):
            want[int(key)] = want.get(int(key), 0) + 1
    for extra in ([], ["--merge-on-device"]):
        argv = ["SELECT k, COUNT(*) FROM t WHERE bytes_out > bytes_in GROUP BY k ORDER BY k LIMIT 100", "--json"]
        for d in dirs:
            argv += ["--segment-dir", d]
        capsys.readouterr()
        assert cli.main(argv + extra) == 0
        out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
        assert {int(k): int(c) for k, c in out["rows"]} == want, extra


def test_loopback_two_ranks(oracle):
    """A group-by merged over a domain with an expression filter combines across two ranks on one GPU like any other."""
    from loopback_dist import run_ranks, values
    from pinot_b200.distributed import execute_and_combine, global_domain
    world = 2
    hosts = [[_segment(oracle, 2000 + 101 * r + 7 * k, 800 + 10 * r + k, name=f"efl{r}_{k}") for k in range(1 + r)] for r in range(world)]
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [[to_device(c, h) for h in hs] for c, hs in zip(ctxs, hosts)]
    try:
        doms = values(run_ranks(world, lambda dist: global_domain(ctxs[dist.get_rank()], devs[dist.get_rank()], ["g"], dist)))
        everything = [h for hs in hosts for h in hs]
        for text in ("SELECT g, COUNT(*), SUM(i) FROM t WHERE i > j GROUP BY g", "SELECT COUNT(*), SUM(i) FROM t WHERE d - f BETWEEN -3 AND 3"):
            q = sql.parse(text)
            got = values(run_ranks(world, lambda dist: execute_and_combine(B200PlanMaker(ctxs[dist.get_rank()]), devs[dist.get_rank()], q, dist)))
            assert all(g is None for g in got[1:])
            _check_groups(oracle, everything, devs[0][0], q, got[0], text)
        for d in doms:
            d.release()
    finally:
        for ds in devs:
            for d in ds:
                d.destroy()
        for c in ctxs:
            c.close()


def test_doc_mask_entry_point(ctx, segs):
    """pb200_expr_doc_masks directly: one mask per (predicate, segment), released with pb200_doc_mask_free, and its
    argument checks."""
    import ctypes as C

    from pinot_b200 import _lib
    L = ctx.lib
    devs = [dev for _, dev in segs[:3]]
    ops = (_lib.TransformOp * 3)(_lib.TransformOp(0, 0, devs[0].column_index("i"), 0.0),
                                 _lib.TransformOp(0, 0, devs[0].column_index("j"), 0.0), _lib.TransformOp(4, 0, 0, 0.0))
    vals = (C.c_double * 2)(0.0, 7.0)
    preds = (_lib.ExprPredicate * 2)(_lib.ExprPredicate(_lib.ExprProgram(3, 0, ops), _lib.EXPR_OPS["RANGE"], 1 | 8, 0.0, 1e300, 0, 0, None),
                                     _lib.ExprPredicate(_lib.ExprProgram(3, 0, ops), _lib.EXPR_OPS["IN"], 0, 0.0, 0.0, 2, 0, vals))
    handles = (C.c_void_p * 3)(*[L.pb200h_segment_device(d.handle) for d in devs])
    out = (C.c_void_p * 6)()
    assert L.pb200_expr_doc_masks(ctx.handle, 2, preds, handles, 3, out) == 0
    assert all(out[k] for k in range(6)) and len({out[k] for k in range(6)}) == 6
    for k in range(6):
        L.pb200_doc_mask_free(ctx.handle, out[k])
    bad = (_lib.ExprPredicate * 1)(_lib.ExprPredicate(_lib.ExprProgram(3, 0, ops), 9, 0, 0.0, 0.0, 0, 0, None))
    assert L.pb200_expr_doc_masks(ctx.handle, 1, bad, handles, 1, out) == E_INVALID
    eq_two = (_lib.ExprPredicate * 1)(_lib.ExprPredicate(_lib.ExprProgram(3, 0, ops), _lib.EXPR_OPS["EQ"], 0, 0.0, 0.0, 2, 0, vals))
    assert L.pb200_expr_doc_masks(ctx.handle, 1, eq_two, handles, 1, out) == E_INVALID
    one_leaf = (_lib.TransformOp * 3)(_lib.TransformOp(0, 0, devs[0].column_index("i"), 0.0), _lib.TransformOp(1, 0, 2, 0.0),
                                      _lib.TransformOp(5, 0, 0, 0.0))
    single = (_lib.ExprPredicate * 1)(_lib.ExprPredicate(_lib.ExprProgram(3, 0, one_leaf), _lib.EXPR_OPS["RANGE"], 2, 0.0, 0.0, 0, 0, None))
    assert L.pb200_expr_doc_masks(ctx.handle, 1, single, handles, 1, out) == E_UNSUPPORTED


def test_refusals(pm, segs):
    seg, dev = segs[3]
    for text in ("SELECT COUNT(*) FROM t WHERE s - i > 0",                          # a STRING leaf
                 "SELECT COUNT(*) FROM t WHERE plus(datetrunc('DAY', l), i) > 0",   # a time function inside
                 "SELECT COUNT(*) FROM t WHERE REGEXP_LIKE(i * j, 'x')",
                 "SELECT COUNT(*) FROM t WHERE i + j LIKE '1%'",
                 "SELECT COUNT(*) FROM t WHERE i * j = 'x'",
                 "SELECT COUNT(*) FROM t WHERE " + "plus(" * 8 + "i" + ",j)" * 8 + " > 0",
                 "SELECT COUNT(*) FROM t GROUP BY i * j"):
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], sql.parse(text))
    with pytest.raises(UnsupportedQueryError):   # selection columns stay single-column
        pm.execute_selection([dev], sql.parse_selection("SELECT i * j FROM t WHERE i > j LIMIT 3"))
    with pytest.raises(Pb200Error):
        pm.execute_segments([dev], sql.parse("SELECT COUNT(*) FROM t WHERE i * nosuch > 0"))
    # one column used twice stays a derived column, which refuses it as before
    with pytest.raises(UnsupportedQueryError):
        pm.execute_segments([dev], sql.parse("SELECT COUNT(*) FROM t WHERE i > i"))
    # a single-column expression predicate is unchanged
    q = sql.parse("SELECT COUNT(*) FROM t WHERE i * 2 > 10")
    assert pm.execute_segments([dev], q)[0].operator_kind in ("AGGREGATION", "NON_SCAN_AGGREGATION")

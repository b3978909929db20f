"""-m gpu: star-tree answers held to the exact reference (tests/exact_ref.py) over the base segment's rows.

Every case asserts that the star-tree answered (operator_kind STAR_TREE: a silent fall-back to the scan would pass
otherwise) and runs the same query with use_star_tree=False; both answers must pass.  The bar is the scan's:

* Trees built on the device (IndexSegment.build_star_tree): COUNT and the AVG count equal; SUM / AVG over INT
  float(exact int64 sum) bit for bit, also where a group's sum passes 2^53; LONG / FLOAT / DOUBLE sums within
  gamma_n * sum|x| of the exact sum (n = the group's rows); MIN / MAX bit-exact.
* Trees built by oracle/startree_builder.py and attached (the reader path): the same, except SUM / AVG over INT.  A
  Pinot-built tree stores each star doc's SUM as a double, so those are held to gamma_n * sum|x| over the base rows
  (sum_within_bound with n = the group's rows), as LONG / FLOAT / DOUBLE sums are.

Filters reach every branch of StarTree::traverse (host/star_tree.cpp); GROUP BY runs on every table route of the star
docs segment; segments carry two trees, or none; the traversal cache evicts; DataTable bytes and the CLI close the path.
Fixtures live here, not in conftest.py."""
import json
import re

import numpy as np
import pytest

import datatable_util
from exact_ref import ExactSum, assert_exact, check_sum, reference, same_double
from gpu_util import gpu_table, to_device, tuned
from oracle import startree_builder as stb
from pinot_b200 import cli, sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker
from segment_dir_util import write_segment_dir

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
F32_MAX, F32_TINY = float(np.finfo(np.float32).max), float(np.float32(1e-45))
F64_MAX, F64_TINY = float(np.finfo(np.float64).max), 5e-324
LIMIT = 1_000_000

DIMS = ["di", "ds", "dl", "df", "dd", "dr", "dw"]   # INT, STRING, LONG, FLOAT, DOUBLE, raw INT (synthesised), 17 bits
METRICS = ["mi", "ml", "mf", "md", "mq"]            # dictionary columns; "<m>_r": the same values stored raw
ATTACHED_DIMS = [d for d in DIMS if d != "dr"]      # the oracle's builder takes dictionary dimensions only
PAIRS = [("COUNT", None)] + [(fn, c) for m in METRICS for c in (m, m + "_r") for fn in ("SUM", "MIN", "MAX")]


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def _kinds_columns(rng, n, ds_values=40):
    di = rng.integers(0, 40, n).astype(np.int32)
    df = (rng.integers(0, 9, n) / 4).astype(np.float32)
    df[di == 39] = 0.0                               # di = 39 AND df = 0.25 matches no row, each leaf matches some
    dw = rng.integers(0, 66_000, n).astype(np.int32)
    dw[:66_000] = np.arange(66_000)                  # every value occurs: 17 bits
    vals = {
        "mi": rng.choice(np.array([INT_MIN, INT_MIN + 1, -1, 0, 1, 12_345, INT_MAX - 1, INT_MAX], dtype=np.int64), n).astype(np.int32),
        "ml": rng.choice(np.array([1 << 62, -(1 << 62), (1 << 53) + 1, (1 << 53) - 1, -((1 << 53) + 1), 7, -3], dtype=np.int64), n),
        "mf": rng.choice(np.array([F32_MAX, -F32_MAX, F32_TINY, -F32_TINY, 0.5, -3.25], dtype=np.float32), n),
        # DOUBLE extremes for MIN / MAX (two +max rows would overflow a SUM), and a DOUBLE column for SUMs
        "md": rng.choice(np.array([F64_MAX, -F64_MAX, F64_TINY, -F64_TINY, 1.5, -2.25]), n),
        "mq": rng.choice(np.array([1e300, -1e300, F64_TINY, 0.1, -7.0, 123.456]), n),
    }
    cols = {"di": di, "ds": np.array([f"v{i:03d}" for i in rng.integers(0, ds_values, n)]).astype("S"),
            "dl": rng.integers(0, 12, n).astype(np.int64) * 10_000_000_000, "df": df,
            "dd": rng.integers(0, 7, n).astype(np.float64) / 8 - 0.5, "dr": rng.integers(0, 25, n).astype(np.int32) * 3, "dw": dw}
    cols.update(vals)
    cols.update({m + "_r": v.copy() for m, v in vals.items()})
    cols["a_mi"] = np.abs(vals["mi"].astype(np.int64))   # sum |x| of the INT metric: the gamma_n bound of attached trees
    return cols


def _attach(dev, st):
    nd = len(st.dimensions)
    dev.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                         [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])


@pytest.fixture(scope="module")
def kinds(oracle, ctx):
    """70 000 rows, every dimension kind, every metric type at its extremes; one device copy with a tree built on the
    device, one with the oracle's tree attached (without the raw dimension), one without a tree."""
    rng = np.random.default_rng(20)
    n = 70_000
    raw = ["dr"] + [m + "_r" for m in METRICS]
    seg = oracle.build_segment("kinds", _kinds_columns(rng, n), raw=raw)
    built, attached, plain = to_device(ctx, seg), to_device(ctx, seg), to_device(ctx, seg)
    built.build_star_tree(DIMS, PAIRS, max_leaf_records=10)
    _attach(attached, stb.build_star_tree(seg, ATTACHED_DIMS, PAIRS, max_leaf_records=10))
    yield {"seg": seg, "built": built, "attached": attached, "plain": plain}
    built.destroy(); attached.destroy(); plain.destroy()


def _bounded_int_sums(oracle, seg, q, text, ref):
    """Attached trees: SUM / AVG over INT as ExactSum("approx") with A = sum |x| (the exact LONG sum of a_mi)."""
    int_cols = [i for i, a in enumerate(q.aggregations)
                if a.function in ("SUM", "AVG") and a.column in ("mi", "mi_r")]
    if not int_cols:
        return ref
    qa = sql.parse(re.sub(r"(SUM|AVG)\(mi(_r)?\)", r"\1(a_mi)", text), num_groups_limit=LIMIT)
    ra = reference(oracle, [seg], qa)
    out = {}
    for key, vals in ref.items():
        vals = list(vals)
        for i in int_cols:
            vals[i] = ExactSum("approx", vals[i].s, ra[key][i].s, vals[i].n)
        out[key] = vals
    return out


def check(oracle, pm, seg, dev, text, attached=False, star=True, ref=None):
    """The star-tree answer and the scan's, both against the exact reference; returns the star block."""
    q = sql.parse(text, num_groups_limit=LIMIT)
    block = pm.execute_segments([dev], q)[0]
    assert (block.operator_kind == "STAR_TREE") == star, (text, block.operator_kind)
    scan = pm.execute_segments([dev], sql.parse(text, use_star_tree=False, num_groups_limit=LIMIT))[0]
    assert scan.operator_kind != "STAR_TREE", text
    ref = reference(oracle, [seg], q) if ref is None else ref
    assert_exact(q, gpu_table(seg, q, scan, dev), ref, "scan " + text)
    if attached:
        ref = _bounded_int_sums(oracle, seg, q, text, ref)
    assert_exact(q, gpu_table(seg, q, block, dev), ref, ("attached " if attached else "built ") + text)
    return block


# ---------------------------------------------------------------------------------------------------- metric types
@pytest.mark.parametrize("source", ["built", "attached"])
@pytest.mark.parametrize("stored", ["dict", "raw"])
def test_metric_types_at_their_extremes(oracle, pm, kinds, source, stored):
    """INT at INT_MIN / INT_MAX, LONG at +-2^62 and 2^53 +- 1, FLOAT / DOUBLE at +-max and the smallest subnormal;
    dictionary columns and raw columns with a dictionary synthesised at load."""
    seg, dev = kinds["seg"], kinds[source]
    sfx = "" if stored == "dict" else "_r"
    shapes = [("", ""), (" WHERE di < 20", " GROUP BY ds"), ("", " GROUP BY di, dl"), (" WHERE dd > 0", " GROUP BY dw")]
    for flt, gb in shapes:
        for m in ("mi", "ml", "mf", "mq"):
            c = m + sfx
            check(oracle, pm, seg, dev, f"SELECT COUNT(*), SUM({c}), MIN({c}), MAX({c}), AVG({c}) FROM t{flt}{gb}", source == "attached")
        c = "md" + sfx
        # SUM(mq) keeps the unfiltered MIN / MAX off the answer from dictionary metadata
        check(oracle, pm, seg, dev, f"SELECT MIN({c}), MAX({c}), COUNT(*), SUM(mq{sfx}) FROM t{flt}{gb}", source == "attached")


# ---------------------------------------------------------------------------------------------------- dimension kinds
@pytest.mark.parametrize("source", ["built", "attached"])
def test_dimension_kinds(oracle, pm, kinds, source):
    """GROUP BY and predicates on INT, STRING, LONG, FLOAT, DOUBLE, a raw INT column with a synthesised dictionary and a
    dimension of 17 bits."""
    seg, dev = kinds["seg"], kinds[source]
    # a built tree's INT SUM reads three 32-bit limb columns: its queries keep the star docs' rows narrow enough for the
    # scan's shared-memory pipeline (wider ones go to the base scan)
    sel_int, sel = "SELECT COUNT(*), SUM(mi), AVG(mi) FROM t", "SELECT COUNT(*), SUM(ml), MIN(mi), AVG(mq) FROM t"
    fits = lambda text: source == "built" or "dr" not in text   # noqa: E731
    for d in DIMS:
        for s in (sel_int, sel):
            check(oracle, pm, seg, dev, f"{s} GROUP BY {d}", source == "attached", fits(d))
    for flt in (" WHERE ds = 'v007'", " WHERE ds > 'v030'", " WHERE dl = 30000000000", " WHERE dl < 25000000000.5",
                " WHERE df > 0.3", " WHERE df <= 1.1", " WHERE dd BETWEEN -0.3 AND 0.2", " WHERE dr IN (3, 9, 30)",
                " WHERE dr > 40.5", " WHERE dw < 30000", " WHERE dw = 65999", " WHERE dw > 1000 AND dl != 0"):
        for s, gb in ((sel_int, ""), (sel_int, " GROUP BY dl"), (sel, " GROUP BY ds, dr")):
            check(oracle, pm, seg, dev, s + flt + gb, source == "attached", fits(flt + gb))


# ---------------------------------------------------------------------------------------------------- traversal branches
FILTERS = [
    " WHERE di = 7", " WHERE di != 7", " WHERE di IN (2, 3)", " WHERE di NOT IN (2, 3)",
    " WHERE di < 12", " WHERE df > 0.6", " WHERE dd < -0.05",                         # RANGE, fractional literals
    " WHERE di < 25 AND di IN (3, 7, 30)", " WHERE di IN (1, 2, 3, 4) AND di != 2",  # two predicates, one dimension
                                                                                     # (two ranges would merge into one)
    " WHERE dw = 17", " WHERE dw < 300", " WHERE dd = 0.25 AND dw > 50000",          # deeper dimensions only: remaining
    " WHERE di IN (0, 1, 2, 3, 4, 5, 6, 7, 8, 9)",                                   # size * 10 > nchild: scan the children
    " WHERE di IN (" + ", ".join(str(i) for i in range(40)) + ")",                   # every child but the star node
    " WHERE di IN (" + ", ".join(str(i) for i in range(1, 40)) + ")",                # every child but one
]
EMPTY_FILTERS = [" WHERE di = 39 AND df = 0.25", " WHERE di IN (1, 2) AND di > 10"]   # each leaf matches, no row does


@pytest.mark.parametrize("source", ["built", "attached"])
def test_filter_branches(oracle, pm, kinds, source):
    seg, dev = kinds["seg"], kinds[source]
    for flt in FILTERS:
        for gb in ("", " GROUP BY ds", " GROUP BY di, dd"):
            check(oracle, pm, seg, dev, "SELECT COUNT(*), SUM(mi), MIN(mi), MAX(ml), AVG(mi) FROM t" + flt + gb, source == "attached")


@pytest.mark.parametrize("source", ["built", "attached"])
def test_empty_aggregation_only_result(oracle, pm, kinds, source):
    """A filter that matches no row while no leaf folds to EMPTY: COUNT 0, SUM 0.0, MIN +inf, MAX -inf, AVG count 0."""
    seg, dev = kinds["seg"], kinds[source]
    for flt in EMPTY_FILTERS:
        text = "SELECT COUNT(*), SUM(mi), MIN(mi), MAX(mf), AVG(mi) FROM t" + flt
        q = sql.parse(text)
        block = check(oracle, pm, seg, dev, text, source == "attached")
        assert block.stats.num_docs_scanned == 0, text
        (count, s, mn, mx, avg), = gpu_table(seg, q, block, dev).values()
        assert count == 0 and same_double(s, 0.0) and mn == float("inf") and mx == float("-inf") and avg[1] == 0, text
        check(oracle, pm, seg, dev, text + " GROUP BY dl", source == "attached")


# ---------------------------------------------------------------------------------------------------- group-by routes
@pytest.mark.parametrize("knobs", [{}, {"smem_groups": 0}, {"dense_max": 1}, {"pack_count": 0}],
                         ids=["default", "global_table", "hash_table", "no_count_carrier"])
def test_group_by_routes_on_the_star_docs(oracle, ctx, pm, kinds, knobs):
    """The star docs segment's GROUP BY on each table route (the pinned view block of try_star_tree) and aggregation-only
    queries (its plain result vectors)."""
    seg = kinds["seg"]
    with tuned(ctx, **knobs):
        for source in ("built", "attached"):
            for text in ("SELECT SUM(mi), COUNT(*) FROM t GROUP BY di", "SELECT AVG(mi), MAX(ml) FROM t WHERE dl > 0 GROUP BY ds, df",
                         "SELECT SUM(mi_r), MIN(mf_r), COUNT(*) FROM t WHERE di < 30 GROUP BY dw",
                         "SELECT SUM(mi), COUNT(*), AVG(mq) FROM t WHERE di < 30", "SELECT SUM(ml), MIN(mi) FROM t"):
                check(oracle, pm, seg, kinds[source], text, source == "attached")


# ---------------------------------------------------------------------------------------------------- trees and segments
def test_two_trees_on_one_segment(oracle, ctx, pm, kinds):
    """The first tree fits some queries; others only the second (its dimensions, its function-column pairs)."""
    seg = kinds["seg"]
    dev = to_device(ctx, seg)
    try:
        dev.build_star_tree(["di", "ds"], [("COUNT", None), ("SUM", "mi")], max_leaf_records=5)
        dev.build_star_tree(["dl", "df", "di"], [("COUNT", None), ("SUM", "mi"), ("MIN", "ml"), ("MAX", "mq")], max_leaf_records=5)
        assert dev.num_star_trees() == 2
        for text in ("SELECT COUNT(*), SUM(mi) FROM t WHERE di < 9 GROUP BY ds",       # first tree
                     "SELECT COUNT(*), SUM(mi), AVG(mi) FROM t GROUP BY dl",            # second tree: dimension
                     "SELECT MIN(ml), MAX(mq) FROM t WHERE di = 4",                      # second tree: pairs
                     "SELECT SUM(mi), MIN(ml) FROM t WHERE df > 0.5 GROUP BY di"):
            check(oracle, pm, seg, dev, text)
        check(oracle, pm, seg, dev, "SELECT COUNT(*), MAX(ml) FROM t GROUP BY ds", star=False)   # neither tree fits
    finally:
        dev.destroy()


def test_one_call_over_segments_with_and_without_trees(oracle, ctx, pm, kinds):
    """One non-merged call: a segment with a tree, one without, and one whose filter folds to EMPTY (no 'v003' in its
    STRING dictionary); each block against its own segment's reference.  merge=True uses no tree and equals the merged
    reference."""
    seg = kinds["seg"]
    other = oracle.build_segment("kinds_x", _kinds_columns(np.random.default_rng(21), 70_000, ds_values=3),   # v000..v002
                                 raw=["dr"] + [m + "_r" for m in METRICS])
    dev_other = to_device(ctx, other)
    try:
        for text in ("SELECT COUNT(*), SUM(mi), MIN(ml), AVG(mi) FROM t WHERE ds = 'v003'",
                     "SELECT COUNT(*), SUM(mi), MAX(mf) FROM t WHERE ds = 'v003' GROUP BY di"):
            q = sql.parse(text, num_groups_limit=LIMIT)
            blocks = pm.execute_segments([kinds["built"], kinds["plain"], dev_other], q)
            assert [b.operator_kind for b in blocks][0] == "STAR_TREE" and blocks[1].operator_kind != "STAR_TREE"
            assert blocks[2].operator_kind == "EMPTY", blocks[2].operator_kind
            for s, d, b in ((seg, kinds["built"], blocks[0]), (seg, kinds["plain"], blocks[1]), (other, dev_other, blocks[2])):
                assert_exact(q, gpu_table(s, q, b, d), reference(oracle, [s], q), f"{s.name}: {text}")
            merged = pm.execute_segments([kinds["built"], kinds["plain"]], q, merge=True)
            assert len(merged) == 1 and merged[0].operator_kind != "STAR_TREE"
            assert_exact(q, gpu_table(seg, q, merged[0], kinds["built"]), reference(oracle, [seg, seg], q), "merged " + text)
    finally:
        dev_other.destroy()


# ---------------------------------------------------------------------------------------------------- traversal cache
def test_traversal_cache_eviction(oracle, ctx, pm, kinds):
    """Ten distinct predicate sets (the cache holds eight), then the first again; one predicate set under two GROUP BY
    masks.  A fresh tree, so the cache starts empty."""
    seg = kinds["seg"]
    dev = to_device(ctx, seg)
    try:
        dev.build_star_tree(["di", "dl", "dd"], [("COUNT", None), ("SUM", "mi"), ("MAX", "mi")], max_leaf_records=10)
        texts = [f"SELECT COUNT(*), SUM(mi), MAX(mi) FROM t WHERE di = {k} GROUP BY dl" for k in range(10)]
        for text in texts + texts[:1]:
            check(oracle, pm, seg, dev, text)
        for gb in (" GROUP BY dl", " GROUP BY dd", "", " GROUP BY dl"):
            check(oracle, pm, seg, dev, "SELECT COUNT(*), SUM(mi), AVG(mi) FROM t WHERE di IN (3, 4) AND dd > -0.2" + gb)
    finally:
        dev.destroy()


# ---------------------------------------------------------------------------------------------------- DataTable bytes
@pytest.mark.parametrize("source", ["built", "attached"])
def test_datatable_bytes_of_a_star_result(oracle, ctx, pm, kinds, source):
    seg, dev = kinds["seg"], kinds[source]
    text = "SELECT COUNT(*), AVG(mi), SUM(ml), MIN(mf) FROM t WHERE di < 25 GROUP BY ds"
    q = sql.parse(text, num_groups_limit=LIMIT)
    block = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        assert block.operator_kind == "STAR_TREE"
        dt = datatable_util.parse(pm.to_datatable(dev, q, block))
    finally:
        block.release(ctx)
    ref = reference(oracle, [seg], q)
    if source == "attached":
        ref = _bounded_int_sums(oracle, seg, q, text, ref)
    assert dt["column_types"] == ["STRING", "LONG", "OBJECT", "DOUBLE", "DOUBLE"]
    got = {(r[0],): r[1:] for r in dt["rows"]}
    assert set(got) == set(ref), text
    for key, (count, avg, s, mn) in ref.items():
        g = got[key]
        assert g[0] == count and g[1][1] == avg.n and check_sum(g[1][0], avg), (key, g, count, avg)
        assert check_sum(g[2], s) and same_double(g[3], float(mn)), (key, g, s, mn)


# ---------------------------------------------------------------------------------------------------- CLI
def test_cli_star_tree_over_two_segment_directories(oracle, tmp_path, capsys):
    rng = np.random.default_rng(31)
    dirs = []
    for i in range(2):
        n = 20_000 + 7 * i
        seg = oracle.build_segment(f"stcli{i}", {"k": rng.integers(0, 9, n).astype(np.int32), "j": rng.integers(0, 30, n).astype(np.int32),
                                                 "v": rng.choice(np.array([INT_MIN, INT_MAX, -1, 5], dtype=np.int64), n).astype(np.int32)})
        dirs.append(write_segment_dir(str(tmp_path / f"seg{i}"), seg, "v3" if i else "v1"))
    config = json.dumps({"dimensionsSplitOrder": ["k", "j"], "functionColumnPairs": ["COUNT__*", "SUM__v", "MIN__v", "MAX__v"],
                         "maxLeafRecords": 4})
    for text in ("SELECT COUNT(*), SUM(v), MIN(v), MAX(v), AVG(v) FROM t WHERE j < 20 GROUP BY k LIMIT 50",
                 "SELECT SUM(v), AVG(v) FROM t WHERE k IN (1, 2, 3)"):
        rows = []
        for extra in ([], ["--star-tree", config]):
            assert cli.main([text, "--json"] + [x for d in dirs for x in ("--segment-dir", d)] + extra) == 0
            rows.append(json.loads(capsys.readouterr().out.strip().splitlines()[-1])["rows"])
        assert rows[0] == rows[1], text


# ---------------------------------------------------------------------------------------------------- INT sums past 2^53
@pytest.fixture(scope="module")
def big(oracle, ctx):
    """10 M rows of odd INT values within 2 000 of INT_MAX: d1 (2 values) holds groups of about 5 M rows, whose sums
    pass 2^53 (4.2 M rows do); d2 (150 values) splits each into star docs of about 33 000 rows.  One tree with a star
    node on d2, one without (skip-star), on two device copies."""
    rng = np.random.default_rng(53)
    n = 10_000_000
    seg = oracle.build_segment("big", {"d1": rng.integers(0, 2, n).astype(np.int32), "d2": rng.integers(0, 150, n).astype(np.int32),
                                       "d3": rng.integers(0, 8, n).astype(np.int32),
                                       "v": (INT_MAX - 2 * rng.integers(0, 1000, n)).astype(np.int32)})
    star, skip = to_device(ctx, seg), to_device(ctx, seg)
    pairs = [("COUNT", None), ("SUM", "v"), ("MAX", "v")]
    star.build_star_tree(["d1", "d2", "d3"], pairs, max_leaf_records=1000)
    skip.build_star_tree(["d1", "d2", "d3"], pairs, max_leaf_records=1000, skip_star_for=["d2"])
    yield seg, star, skip
    star.destroy(); skip.destroy()


@pytest.mark.parametrize("tree", ["star", "skip_star"])
def test_int_sums_past_2_53(oracle, pm, big, tree):
    """Each group sums many star docs and passes 2^53 on the way: a predicate that keeps 140 or 148 of d2's children, or,
    in the skip-star tree, a predicate on d3 below a d2 without a star node.  SUM and AVG must be float(exact sum)."""
    seg, star, skip = big
    dev = star if tree == "star" else skip
    texts = ["SELECT SUM(v), AVG(v) FROM t WHERE d2 < 140 GROUP BY d1", "SELECT SUM(v), COUNT(*), AVG(v) FROM t WHERE d2 < 140",
             "SELECT SUM(v), MAX(v) FROM t WHERE d2 NOT IN (7, 8) GROUP BY d1"]
    if tree == "skip_star":
        texts += ["SELECT SUM(v), AVG(v) FROM t WHERE d3 != 1 GROUP BY d1", "SELECT SUM(v), AVG(v) FROM t WHERE d3 != 1",
                  "SELECT SUM(v), COUNT(*) FROM t GROUP BY d1"]
    for text in texts:
        q = sql.parse(text)
        ref = reference(oracle, [seg], q)
        assert any(isinstance(x, ExactSum) and x.s > (1 << 53) for vals in ref.values() for x in vals), text
        check(oracle, pm, seg, dev, text, ref=ref)

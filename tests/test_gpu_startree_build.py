"""-m gpu: star-trees built on the device (pb200h_startree_build) against the oracle's builder on the same segment, and
queries through them against the raw scan, the oracle and an oracle-built tree attached to the same data."""
import numpy as np
import pytest

from gpu_util import assert_tables_equal, gpu_table, oracle_table, to_device, tuned
from oracle import startree_builder as stb
from pinot_b200 import _lib, sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker
from startree_canon import assert_equivalent, canonical
from test_oracle_startree import FILTERS, GROUPS

pytestmark = pytest.mark.gpu

PAIRS = [("COUNT", None), ("SUM", "m"), ("MAX", "m"), ("MIN", "m")]


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


def _check_tree(dev, seg, dims, pairs, max_leaf=10, skip=(), tolerance=None):
    info = dev.build_star_tree(dims, pairs, max_leaf_records=max_leaf, skip_star_for=skip)
    st = stb.build_star_tree(seg, dims, pairs, max_leaf_records=max_leaf, skip_star_for=skip)
    got = dev.read_star_tree(dev.num_star_trees() - 1)
    assert info["num_star_docs"] == st.num_docs and got["num_docs"] == st.num_docs
    names = list(got["columns"])
    gdims = np.stack([got["columns"][d] for d in dims], axis=1)
    gmets = [got["columns"][n] for n in names[len(dims):]]
    assert names[len(dims):] == [st.metric_name(i) for i in range(len(pairs))]
    want = canonical(st.tree, st.dim_dict_ids, st.metrics)
    assert_equivalent(canonical(got["tree"], gdims, gmets), want, tolerance, what=f"{dims} leaf={max_leaf} skip={skip}")
    assert info["num_nodes"] == len(want["nodes"])
    return info, st


def _columns(rng, n, cards=(100, 50, 7)):
    cols = {f"d{i + 1}": rng.integers(0, c, size=n).astype(np.int32) for i, c in enumerate(cards)}
    cols["m"] = rng.integers(-500, 1000, size=n).astype(np.int32)
    return cols


@pytest.mark.parametrize("n", [1, 2, 31, 1000, 30_000, 100_003])
def test_sizes(oracle, ctx, n):
    seg = oracle.build_segment("s", _columns(np.random.default_rng(n), n))
    dev = to_device(ctx, seg)
    try:
        _check_tree(dev, seg, ["d1", "d2", "d3"], PAIRS, max_leaf=10)
    finally:
        dev.destroy()


@pytest.mark.parametrize("max_leaf", [1, 10, 1000, 1_000_000])
@pytest.mark.parametrize("skip", [(), ("d1",), ("d2",), ("d1", "d2", "d3")])
def test_max_leaf_and_skip_star(oracle, ctx, max_leaf, skip):
    seg = oracle.build_segment("s", _columns(np.random.default_rng(max_leaf), 30_000))
    dev = to_device(ctx, seg)
    try:
        _check_tree(dev, seg, ["d1", "d2", "d3"], PAIRS, max_leaf=max_leaf, skip=skip)
    finally:
        dev.destroy()


def test_dimension_kinds_and_counts(oracle, ctx):
    rng = np.random.default_rng(3)
    n = 20_000
    cols = {"s": np.array([f"v{i:03d}" for i in rng.integers(0, 40, n)]).astype("S"), "x": rng.integers(0, 9, n).astype(np.float64) / 4,
            "l": rng.integers(0, 12, n).astype(np.int64) * 10_000_000_000, "i": rng.integers(0, 30, n).astype(np.int32),
            "m": rng.integers(0, 1000, n).astype(np.int32)}
    seg = oracle.build_segment("k", cols)
    dev = to_device(ctx, seg)
    try:
        for dims in (["s"], ["x", "s"], ["l", "i", "x"], ["s", "x", "l", "i"]):
            _check_tree(dev, seg, dims, PAIRS, max_leaf=5)
    finally:
        dev.destroy()


def test_split_order_beyond_64_bits(oracle, ctx):
    """5 dimensions of cardinality 8 193 (14 bits each, 70 in all): one stable sort pass per dimension."""
    rng = np.random.default_rng(70)
    n = 40_000
    cols = {f"k{j}": rng.integers(0, 8193, n).astype(np.int32) for j in range(5)}
    for j in range(5):
        cols[f"k{j}"][:8193] = np.arange(8193)  # every value occurs: 14 bits
    cols["k0"][8193:20000] = 7                 # long runs in the leading dimension
    cols["m"] = rng.integers(0, 100, n).astype(np.int32)
    seg = oracle.build_segment("w", cols)
    dev = to_device(ctx, seg)
    try:
        assert all(dev.column_info(f"k{j}")["bits"] == 14 for j in range(5))
        _check_tree(dev, seg, [f"k{j}" for j in range(5)], PAIRS, max_leaf=3)
    finally:
        dev.destroy()


def test_metric_sources(oracle, ctx):
    """Metrics over dictionary, synthesised-raw and streamed-raw columns of every numeric type."""
    rng = np.random.default_rng(11)
    n = 30_000
    vals = {"mi": rng.integers(-2**31, 2**31 - 1, n, dtype=np.int64).astype(np.int32),
            "ml": rng.integers(-2**30, 2**30, n).astype(np.int64) * 1024,
            "mf": (rng.integers(-1000, 1000, n) / 8).astype(np.float32),
            "md": rng.integers(-10**6, 10**6, n).astype(np.float64) / 16,
            "mq": rng.standard_normal(n) * 1e3}
    dims = {"d1": rng.integers(0, 60, n).astype(np.int32), "d2": rng.integers(0, 9, n).astype(np.int32)}
    pairs = [("COUNT", None)] + [(fn, c) for c in vals for fn in ("SUM", "MIN", "MAX")]
    total_abs = {c: float(np.abs(v.astype(np.float64)).sum()) for c, v in vals.items()}
    gamma = n * 2.0 ** -53 / (1 - n * 2.0 ** -53)
    tol = [None] + [2 * gamma * total_abs[c] if (fn == "SUM" and c == "mq") else None for fn, c in pairs[1:]]
    raw = {**dims, **{c + "_r": v for c, v in vals.items()}}
    dict_seg = oracle.build_segment("dict", {**dims, **vals})
    raw_seg = oracle.build_segment("raw", raw, raw=[c + "_r" for c in vals])
    raw_pairs = [(fn, c if c is None else c + "_r") for fn, c in pairs]
    dev = to_device(ctx, dict_seg)
    dev_raw = to_device(ctx, raw_seg)                      # raw columns: dictionaries synthesised at load
    with tuned(ctx, raw_dict_max=0):
        stream_seg = oracle.build_segment("stream", {**dims, "mi_r": vals["mi"], "mf_r": vals["mf"]}, raw=["mi_r", "mf_r"])
        dev_stream = to_device(ctx, stream_seg)            # raw INT / FLOAT streamed as 32-bit values
    try:
        _check_tree(dev, dict_seg, ["d1", "d2"], pairs, max_leaf=4, tolerance=tol)
        _check_tree(dev_raw, raw_seg, ["d1", "d2"], raw_pairs, max_leaf=4, tolerance=tol)
        sp = [("COUNT", None), ("SUM", "mi_r"), ("MIN", "mi_r"), ("MAX", "mi_r"), ("SUM", "mf_r"), ("MAX", "mf_r")]
        _check_tree(dev_stream, stream_seg, ["d1", "d2"], sp, max_leaf=4)
        with pytest.raises(_lib.UnsupportedQueryError):
            dev_stream.build_star_tree(["mi_r"], [("COUNT", None)])   # no dictIds: not a dimension
    finally:
        dev.destroy(); dev_raw.destroy(); dev_stream.destroy()


def test_query_parity(oracle, ctx):
    """Every filter x group-by shape of the oracle's star-tree test: built tree == raw scan == oracle == attached tree."""
    rng = np.random.default_rng(7)
    n = 50_000
    cols = {"d1": rng.integers(0, 100, n).astype(np.int32), "d2": rng.integers(0, 100, n).astype(np.int32) * 2,
            "d3": rng.integers(0, 7, n).astype(np.int32), "m": rng.integers(0, 1000, n).astype(np.int32)}
    seg = oracle.build_segment("p", cols)
    built, attached = to_device(ctx, seg), to_device(ctx, seg)
    pm = B200PlanMaker(ctx)
    try:
        built.build_star_tree(["d1", "d2", "d3"], PAIRS, max_leaf_records=10)
        st = stb.build_star_tree(seg, ["d1", "d2", "d3"], PAIRS, max_leaf_records=10)
        nd = len(st.dimensions)
        attached.attach_star_tree(st.tree, st.num_docs, st.dimensions, [st.segment.columns[j].fwd for j in range(nd)],
                                  [(fn, col, st.segment.columns[nd + i].fwd) for i, (fn, col) in enumerate(st.function_pairs)])
        for flt in FILTERS:
            for gb in GROUPS:
                text = "SELECT COUNT(*), SUM(m), MAX(m), MIN(m), AVG(m) FROM t" + flt + gb
                q = sql.parse(text)
                star = pm.execute_segments([built], q)[0]
                other = pm.execute_segments([attached], q)[0]
                scan = pm.execute_segments([built], sql.parse(text, use_star_tree=False))[0]
                assert star.operator_kind == other.operator_kind, text
                want = oracle_table(seg, q, oracle.execute(seg, q))
                assert_tables_equal(q, gpu_table(seg, q, scan), want, "scan " + text)
                if star.operator_kind != "STAR_TREE" or (not gb and scan.stats.num_docs_scanned == 0):
                    continue
                got = gpu_table(seg, q, star)
                assert_tables_equal(q, got, want, "star " + text)
                assert got == gpu_table(seg, q, other), text
                if not flt:
                    assert star.stats.num_docs_scanned < scan.stats.num_docs_scanned
    finally:
        built.destroy(); attached.destroy()


def test_float_edges(oracle, ctx):
    """NaN, -0.0, 0.0 and +-inf in metric columns: star-tree SUM / MIN / MAX == the raw scan's."""
    rng = np.random.default_rng(13)
    n = 20_000
    edges = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.5, -2.25])
    d = edges[rng.integers(0, len(edges), n)]
    d[rng.random(n) < 0.7] = 0.5
    cols = {"d1": rng.integers(0, 40, n).astype(np.int32), "d2": rng.integers(0, 5, n).astype(np.int32),
            "md": d, "mf": d.astype(np.float32), "z": np.where(rng.random(n) < 0.5, -0.0, 0.0)}
    seg = oracle.build_segment("f", cols, raw=["md", "mf", "z"])   # dictionaries synthesised at load: -0.0 apart from 0.0
    dev = to_device(ctx, seg)
    pm = B200PlanMaker(ctx)
    try:
        pairs = [("COUNT", None)] + [(fn, c) for c in ("md", "mf", "z") for fn in ("SUM", "MIN", "MAX")]
        dev.build_star_tree(["d1", "d2"], pairs, max_leaf_records=3)
        for flt in ("", " WHERE d1 < 20", " WHERE d2 = 3"):
            for gb in ("", " GROUP BY d1", " GROUP BY d2", " GROUP BY d1, d2"):
                text = ("SELECT COUNT(*), SUM(md), MIN(md), MAX(md), SUM(mf), MIN(mf) FROM t" + flt + gb)
                for t in (text, "SELECT MAX(mf), SUM(z), MIN(z), MAX(z) FROM t" + flt + gb):
                    star = pm.execute_segments([dev], sql.parse(t))[0]
                    scan = pm.execute_segments([dev], sql.parse(t, use_star_tree=False))[0]
                    assert star.operator_kind in ("STAR_TREE", "NON_SCAN_AGGREGATION"), t
                    a, b = gpu_table(seg, sql.parse(t), star), gpu_table(seg, sql.parse(t), scan)
                    assert a.keys() == b.keys(), t
                    for k in b:
                        for x, y in zip(a[k], b[k]):
                            assert np.array(x, dtype=np.float64).tobytes() == np.array(y, dtype=np.float64).tobytes() or \
                                (np.isnan(x) and np.isnan(y)), (t, k, x, y)
    finally:
        dev.destroy()


def test_refusals(oracle, ctx):
    rng = np.random.default_rng(2)
    n = 1000
    seg = oracle.build_segment("r", {"d": rng.integers(0, 10, n).astype(np.int32), "s": np.array([f"s{i % 7}" for i in range(n)]).astype("S"),
                                     "m": rng.integers(0, 10, n).astype(np.int32)})
    dev = to_device(ctx, seg)
    try:
        with pytest.raises(_lib.Pb200Error) as e:
            dev.build_star_tree(["nope"], [("COUNT", None)])
        assert e.value.code == _lib.E_INVALID
        with pytest.raises(_lib.Pb200Error) as e:
            dev.build_star_tree(["d"], [("SUM", "nope")])
        assert e.value.code == _lib.E_INVALID
        with pytest.raises(_lib.UnsupportedQueryError):
            dev.build_star_tree(["d"], [("SUM", "s")])          # STRING metric
        dev.derive("plus(m,'1')")
        with pytest.raises(_lib.UnsupportedQueryError):
            dev.build_star_tree(["plus(m,'1')"], [("COUNT", None)])
        with pytest.raises(_lib.UnsupportedQueryError):
            dev.build_star_tree(["d"], [("SUM", "plus(m,'1')")])
        assert dev.num_star_trees() == 0                       # a failure attaches nothing
    finally:
        dev.destroy()

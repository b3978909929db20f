"""Device star-tree build, the parts that need no GPU: StarTreeIndexConfig parsing (Python and CLI), the library's
refusals of a configuration before it looks at a segment, and the test-side canonical comparison of two trees."""
import ctypes as C
import json

import numpy as np
import pytest

from oracle import startree_builder as stb
from pinot_b200 import _lib, cli
from pinot_b200.plan_maker import parse_star_tree_config, star_tree_config
from startree_canon import assert_equivalent, canonical, tree_nodes


def test_parse_function_column_pairs():
    cfg = parse_star_tree_config(json.dumps({
        "dimensionsSplitOrder": ["d1", "d2"], "skipStarNodeCreationForDimensions": ["d2"],
        "functionColumnPairs": ["COUNT__*", "SUM__m", "max__m", "SUM__m"], "maxLeafRecords": 7}))
    assert cfg == {"dimensions": ["d1", "d2"], "function_pairs": [("COUNT", None), ("SUM", "m"), ("MAX", "m")],
                   "max_leaf_records": 7, "skip_star_for": ["d2"]}


def test_parse_aggregation_configs_and_defaults():
    cfg = parse_star_tree_config({"dimensionsSplitOrder": ["d"],
                                  "aggregationConfigs": [{"columnName": "m", "aggregationFunction": "MIN"},
                                                         {"columnName": "*", "aggregationFunction": "count"}]})
    assert cfg["function_pairs"] == [("MIN", "m"), ("COUNT", None)]
    assert cfg["max_leaf_records"] == 10000 and cfg["skip_star_for"] == []


@pytest.mark.parametrize("bad", [
    "{not json", "[1]", {"functionColumnPairs": ["COUNT__*"]}, {"dimensionsSplitOrder": [], "functionColumnPairs": ["COUNT__*"]},
    {"dimensionsSplitOrder": ["d"]}, {"dimensionsSplitOrder": ["d"], "functionColumnPairs": ["SUMm"]},
    {"dimensionsSplitOrder": ["d"], "functionColumnPairs": ["COUNT__*"], "maxLeafRecords": "10"},
    {"dimensionsSplitOrder": ["d"], "aggregationConfigs": [{"columnName": "m"}]},
    {"dimensionsSplitOrder": ["d"], "functionColumnPairs": ["COUNT__*"], "skipStarNodeCreationForDimensions": "d"},
])
def test_parse_refuses_malformed(bad):
    with pytest.raises(ValueError):
        parse_star_tree_config(bad)


def test_cli_refuses_a_malformed_star_tree_before_loading(capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(["--segment-dir", "/nonexistent", "--star-tree", '{"dimensionsSplitOrder": []}', "SELECT COUNT(*) FROM t"])
    assert e.value.code == 2
    assert "dimensionsSplitOrder" in capsys.readouterr().err


def _build_rc(dims, pairs, max_leaf=10, skip=()):
    L = _lib.load()
    cfg, _keep = star_tree_config(dims, pairs, max_leaf, skip)
    return L.pb200h_startree_build(None, None, C.byref(cfg), None)


@pytest.mark.parametrize("dims,pairs,max_leaf,skip,code", [
    ([], [("COUNT", None)], 10, (), _lib.E_INVALID),                          # empty split order
    (["a", "b", "a"], [("COUNT", None)], 10, (), _lib.E_INVALID),             # repeated dimension
    (["a", "b"], [("COUNT", None)], 10, ("c",), _lib.E_INVALID),              # skip dimension outside the split order
    (["a"], [("COUNT", None)], 0, (), _lib.E_INVALID),                        # maxLeafRecords < 1
    (["a"], [], 10, (), _lib.E_INVALID),                                      # no pairs
    (["a"], [("SUM", None)], 10, (), _lib.E_INVALID),                         # SUM without a column
    ([f"d{i}" for i in range(31)], [("COUNT", None)], 10, (), _lib.E_UNSUPPORTED),  # more than 30 dimensions
    (["a"], [("AVG", "m")], 10, (), _lib.E_UNSUPPORTED),                      # no star-tree metric for AVG here
    (["a"], [("DISTINCTCOUNTHLL", "m")], 10, (), _lib.E_UNSUPPORTED),
    (["a"], [("COUNT", None), ("SUM", "m")], 10, (), _lib.E_INVALID),         # a valid config, but no segment
])
def test_library_refuses_configs_without_a_segment(dims, pairs, max_leaf, skip, code):
    assert _build_rc(dims, pairs, max_leaf, skip) == code


def _oracle_tree(oracle, max_leaf=3):
    rng = np.random.default_rng(5)
    n = 400
    seg = oracle.build_segment("c", {"a": rng.integers(0, 5, n).astype(np.int32), "b": rng.integers(0, 4, n).astype(np.int32),
                                     "c": rng.integers(0, 3, n).astype(np.int32), "m": rng.integers(0, 100, n).astype(np.int32)})
    return stb.build_star_tree(seg, ["a", "b", "c"], [("COUNT", None), ("SUM", "m"), ("MAX", "m")], max_leaf_records=max_leaf)


def _tree_bytes(st, nodes):
    b = np.asarray(st.tree, dtype=np.uint8).tobytes()
    root = len(b) - 28 * len(nodes)
    return np.frombuffer(b[:root] + nodes.astype("<i4").tobytes(), dtype=np.uint8).copy()


def test_canonical_form_ignores_doc_numbering(oracle):
    st = _oracle_tree(oracle)
    base = canonical(st.tree, st.dim_dict_ids, st.metrics)
    nodes = tree_nodes(st.tree)
    # renumber: the docs inside every leaf in reverse order
    perm = np.arange(st.num_docs)
    leaves = [(s, e) for s, e, fc in zip(nodes[:, 2], nodes[:, 3], nodes[:, 5]) if fc == -1 and s >= 0]
    for s, e in leaves:
        perm[s:e] = perm[s:e][::-1]   # a leaf's docs in another order (its range stays a range)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    new_nodes = nodes.copy()
    agg = new_nodes[:, 4]
    new_nodes[:, 4] = np.where(agg >= 0, perm[np.maximum(agg, 0)], agg)
    assert_equivalent(base, canonical(_tree_bytes(st, new_nodes), st.dim_dict_ids[inv], [m[inv] for m in st.metrics]), what="renumbered")
    # aggregated docs appended in another order
    k = st.num_docs
    ranged = np.zeros(k, dtype=bool)
    for s, e in zip(nodes[:, 2], nodes[:, 3]):
        if s >= 0:
            ranged[s:e] = True
    free = np.nonzero(~ranged)[0]          # aggregated-only docs: any numbering among themselves
    perm2 = np.arange(k)
    perm2[free] = free[::-1]
    inv2 = np.empty_like(perm2)
    inv2[perm2] = np.arange(k)
    n2 = nodes.copy()
    n2[:, 4] = np.where(n2[:, 4] >= 0, perm2[np.maximum(n2[:, 4], 0)], n2[:, 4])
    assert_equivalent(base, canonical(_tree_bytes(st, n2), st.dim_dict_ids[inv2], [m[inv2] for m in st.metrics]), what="aggregated docs")


def test_canonical_form_detects_changes(oracle):
    st = _oracle_tree(oracle)
    base = canonical(st.tree, st.dim_dict_ids, st.metrics)
    nodes = tree_nodes(st.tree)
    # one metric value of one doc
    mets = [m.copy() for m in st.metrics]
    mets[1][int(nodes[5, 2])] += 1
    with pytest.raises(AssertionError):
        assert_equivalent(base, canonical(st.tree, st.dim_dict_ids, mets))
    # one node's range one doc shorter
    n2 = nodes.copy()
    i = int(np.nonzero((n2[:, 3] - n2[:, 2] > 1) & (n2[:, 2] >= 0))[0][-1])
    n2[i, 3] -= 1
    with pytest.raises(AssertionError):
        assert_equivalent(base, canonical(_tree_bytes(st, n2), st.dim_dict_ids, st.metrics))
    # one child fewer: the parent's last child dropped from the list
    n3 = nodes.copy()
    p = int(np.nonzero(n3[:, 6] > n3[:, 5])[0][0])
    n3[p, 6] -= 1
    with pytest.raises(AssertionError):
        assert_equivalent(base, canonical(_tree_bytes(st, n3), st.dim_dict_ids, st.metrics))
    # one child's value
    n4 = nodes.copy()
    n4[int(n4[0, 6]), 1] += 1
    with pytest.raises(AssertionError):
        assert_equivalent(base, canonical(_tree_bytes(st, n4), st.dim_dict_ids, st.metrics))

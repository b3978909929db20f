"""Canonical form of a star-tree, independent of how its docs are numbered.

Two builds of one tree may number their star docs differently (the oracle appends in DFS order, a level-by-level build
does not).  What the traversal reads is the same in both: the node array (breadth first, children sorted) without its
start / end / aggregated-doc fields, and per node the docs of its range and its aggregated doc.  Within a node's range
every doc has a distinct dimension tuple, so sorting the range by (node, dimensions) pairs the docs of two builds."""
from __future__ import annotations

import struct

import numpy as np


def tree_nodes(tree: np.ndarray) -> np.ndarray:
    """[num_nodes, 7] int32: dim, value, start, end, agg, first child, last child (OffHeapStarTree layout)."""
    b = np.asarray(tree, dtype=np.uint8).tobytes()
    root = struct.unpack_from("<i", b, 12)[0]
    num = struct.unpack_from("<i", b, root - 4)[0]
    return np.frombuffer(b, dtype="<i4", offset=root, count=7 * num).reshape(num, 7).astype(np.int64)


def canonical(tree: np.ndarray, dims: np.ndarray, metrics) -> dict:
    """dims [docs, D] dictIds, metrics: one array per function-column pair."""
    nodes = tree_nodes(tree)
    starts, ends = nodes[:, 2], nodes[:, 3]
    lens = np.where(starts >= 0, ends - starts, 0)
    owner = np.repeat(np.arange(len(nodes)), lens)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    docs = np.arange(int(lens.sum())) - np.repeat(offs, lens) + np.repeat(np.maximum(starts, 0), lens)
    dims = np.asarray(dims).reshape(len(dims), -1)
    order = np.lexsort([dims[docs, j] for j in reversed(range(dims.shape[1]))] + [owner])
    docs, owner = docs[order], owner[order]
    agg = nodes[:, 4]
    return {"nodes": nodes[:, [0, 1, 5, 6]], "counts": lens, "owner": owner, "dims": dims[docs],
            "metrics": [np.asarray(m)[docs] for m in metrics], "agg_dims": dims[agg],
            "agg_metrics": [np.asarray(m)[agg] for m in metrics]}


def _bits(x: np.ndarray) -> np.ndarray:
    if x.dtype.kind != "f":
        return x.astype(np.int64)
    x = x.astype(np.float64)
    return np.where(np.isnan(x), np.float64("nan"), x).view(np.int64)  # one NaN; -0.0 apart from 0.0


def assert_equivalent(a: dict, b: dict, tolerance=None, what: str = ""):
    """Equal canonical forms.  tolerance[m] (absolute) replaces bit equality for metric m, else bits must match."""
    assert a["nodes"].shape == b["nodes"].shape, f"{what}: {len(a['nodes'])} vs {len(b['nodes'])} nodes"
    assert np.array_equal(a["nodes"], b["nodes"]), f"{what}: node arrays differ"
    assert np.array_equal(a["counts"], b["counts"]), f"{what}: doc counts differ"
    assert np.array_equal(a["owner"], b["owner"]) and np.array_equal(a["dims"], b["dims"]), f"{what}: node docs differ"
    assert np.array_equal(a["agg_dims"], b["agg_dims"]), f"{what}: aggregated docs' dimensions differ"
    for m, (x, y, ax, ay) in enumerate(zip(a["metrics"], b["metrics"], a["agg_metrics"], b["agg_metrics"])):
        tol = None if tolerance is None else tolerance[m]
        for u, v, where in ((x, y, "docs"), (ax, ay, "aggregated docs")):
            if tol is None:
                bad = np.nonzero(_bits(u) != _bits(v))[0]
            else:
                bad = np.nonzero(np.abs(u.astype(np.float64) - v.astype(np.float64)) > tol)[0]
            assert len(bad) == 0, f"{what}: metric {m} differs in {len(bad)} {where}, first {u[bad[0]]} vs {v[bad[0]]}"
